"""GPU parity of the ideal-MHD build where the floors fire and the field degenerates (helpers.mhd_floor_state: near-vacuum, cold
magnetised, magnetically dominated, field-free and field-aligned regions; helpers.fill_mhd_floor_cells on AMR trees) under the
RAMSES floors (smallr = smallc = 1e-10) and raised ones (smallr = 1e-3, smallc = 1e-2), through the C-ABI.  On these states
ctoprim's pressure floor, the density / pressure clamps of the traced states, the cmpdt floors, the HLLD degenerate star state,
Roe's bt = 0 branch and the smallc floor of the 2-D HLLD Alfven speeds are all taken, and the branch-free division and square
root of the device see zero numerators, tiny fields and near-vacuum densities; every run equals the oracle bit for bit."""
import numpy as np
import pytest

from helpers import FLOORS, MhdCase, mhd_floor_counts, mhd_floor_state

pytestmark = pytest.mark.gpu

NSTEP = 5
SOLVERS = [("llf", "llf"), ("hll", "hll"), ("hlld", "hlld"), ("roe", "llf"), ("roe", "roe"), ("hlld", "hlla"),
           ("upwind", "upwind"), ("hydro", "llf")]               # test_gpu_mhd.SOLVERS


def _floor_case(floors, riemann, riemann2d, slope_type, slope_mag_type=-1, coarse=(1, 1, 1), level=4, bound=(0,) * 6, seed=7):
    """MhdCase holding an mhd_floor_state under FLOORS[floors]; asserts that the floors fire and that field-free and
    field-aligned (vA > c_s) cells are present"""
    smallr, smallc = FLOORS[floors]
    c = MhdCase(level, riemann=riemann, riemann2d=riemann2d, slope_type=slope_type, slope_mag_type=slope_mag_type, bound=bound,
                coarse=coarse, boxlen=float(coarse[0]), order=2, seed=3, smallr=smallr, smallc=smallc)
    d0 = mhd_floor_state(c.mesh.extent(level), seed, smallr, smallc, slab_vt=0.3 if riemann2d == "hlla" else 0.0)
    nrho, npr, nfree, nfast = mhd_floor_counts(d0, smallr, smallc)
    assert min(nrho, npr) >= 0.02 * d0[0].size and nfree > 0 and nfast > 0, (nrho, npr, nfree, nfast)
    c.init_dense(d0)
    return c


def _oracle_steps(c, nstep=NSTEP):
    ref, dts = c.oracle_steps(nstep, nthreads=8)
    assert np.isfinite(ref).all() and np.isfinite(dts).all() and (dts > 0).all()
    return ref, dts


def _check(c, a, dts, ref, dts_ref):
    act = c.active_cells()
    assert np.array_equal(dts, dts_ref), (dts, dts_ref)
    got, exp = a.uold[:, act], ref.reshape(11, -1)[:, act]
    assert np.isfinite(got).all()
    assert np.array_equal(got, exp), float(np.abs(got - exp).max())


def _level_steps(c, nstep=NSTEP):
    from ramses_b200.hydro import HydroGPU
    a = c.amr_commons()
    h = HydroGPU(a)
    h.bind_level(c.level)
    h.upload_state(c.level)
    dts, _ = h.level_steps(c.level, nstep)
    h.download_state(c.level)
    info = h.level_info(c.level)
    h.finalize()
    return a, np.asarray(dts), info


@pytest.mark.parametrize("floors", ["default", "raised"])
@pytest.mark.parametrize("slope_type", [0, 1, 2])
@pytest.mark.parametrize("riemann,riemann2d", SOLVERS)
def test_mhd_level_steps_at_the_floors(floors, riemann, riemann2d, slope_type):
    """rgpu_level_steps, 5 fused steps on a periodic 16^3 mhd_floor_state: state and dt history equal the oracle's"""
    c = _floor_case(floors, riemann, riemann2d, slope_type)
    ref, dts_ref = _oracle_steps(c)
    a, dts, info = _level_steps(c)
    assert info.dense == 1
    _check(c, a, dts, ref, dts_ref)


@pytest.mark.parametrize("floors", ["default", "raised"])
@pytest.mark.parametrize("riemann,riemann2d,slope_type,slope_mag_type,coarse,level", [
    ("hlld", "hlld", 3, 1, (1, 1, 1), 4), ("roe", "llf", 7, 2, (1, 1, 1), 4), ("hlld", "roe", 2, 1, (3, 2, 1), 3)])
def test_mhd_slope_variants_and_box_shape_at_the_floors(floors, riemann, riemann2d, slope_type, slope_mag_type, coarse, level):
    """slope_type 3 / 7 with slope_mag_type 1 / 2, and a 24 x 16 x 8 domain of 3 x 2 x 1 coarse cells: 5 steps equal the oracle"""
    c = _floor_case(floors, riemann, riemann2d, slope_type, slope_mag_type, coarse=coarse, level=level)
    ref, dts_ref = _oracle_steps(c)
    a, dts, _ = _level_steps(c)
    _check(c, a, dts, ref, dts_ref)


@pytest.mark.parametrize("floors", ["default", "raised"])
@pytest.mark.parametrize("bound", [(2, 2, 0, 0, 0, 0), (1, 1, 2, 2, 0, 0), (2, 1, 1, 2, 1, 1)])
@pytest.mark.parametrize("riemann,riemann2d,slope_type", [("roe", "llf", 0), ("hlld", "hlld", 1)])
def test_mhd_boundaries_at_the_floors(floors, bound, riemann, riemann2d, slope_type):
    """the zero-gradient / reflexive boxes of test_mhd_tube_boundaries_bitwise holding an mhd_floor_state: make_boundary_hydro
    (mhd_boundary_kernel, whose outflow branch floors the density of ekin) and 5 steps equal the oracle, boundary octs included"""
    c = _floor_case(floors, riemann, riemann2d, slope_type, bound=bound)
    ref, dts_ref = _oracle_steps(c)
    a, dts, _ = _level_steps(c)
    _check(c, a, dts, ref, dts_ref)
    assert np.array_equal(a.uold, ref.reshape(11, -1))


@pytest.mark.parametrize("floors", ["default", "raised"])
@pytest.mark.parametrize("riemann,riemann2d,slope_type", [("hlld", "hlld", 1), ("roe", "llf", 2)])
def test_mhd_courant_split_sequence_and_level0_at_the_floors(orc, floors, riemann, riemann2d, slope_type):
    """rgpu_courant_fine alone (dt bit for bit, the mass / kinetic / internal / magnetic energy sums to 1e-12; the internal energy
    of a cold magnetised cell is negative), then the split sequence courant_fine -> set_unew -> godunov_fine_dev -> set_uold ->
    make_boundary_hydro for 4 steps, then Level-0 godunov_fine on host arrays: equal the oracle"""
    from ramses_b200.hydro import HydroGPU
    from test_gpu_mhd import run_gpu
    c = _floor_case(floors, riemann, riemann2d, slope_type)
    dt0, sums0 = c.oracle_courant()
    a = c.amr_commons()
    h = HydroGPU(a)
    h.bind_level(c.level)
    h.upload_state(c.level)
    a.dtnew[c.level] = a.boxlen / a.smallc
    assert h.courant_fine(c.level) == dt0
    h.finalize()
    got = np.array([a.mass_tot, a.ekin_tot, a.eint_tot, a.emag_tot])
    assert np.all(np.abs(got - sums0) <= 1e-12 * np.abs(sums0).max()), (got, sums0)
    ref, dts_ref = _oracle_steps(c, 4)
    a, dts, _, _ = run_gpu(c, 4, fused=False)
    _check(c, a, dts, ref, dts_ref)
    exp = c.oracle_godunov(dt0, nthreads=8).reshape(11, -1)
    assert np.isfinite(exp).all()
    a = c.amr_commons()
    a.unew[:, :] = a.uold
    a.dtnew[c.level] = dt0
    h = HydroGPU(a)
    h.bind_level(c.level)
    h.godunov_fine(c.level)
    h.finalize()
    act = c.active_cells()
    assert np.array_equal(a.unew[:, act], exp[:, act])


@pytest.mark.parametrize("ndim,r1,r2,slope_type,field_scale,floors,resident", [
    (1, "hlld", "llf", 1, 1.0, "default", False), (1, "roe", "llf", 2, 1.0, "raised", True), (1, "hydro", "llf", 1, 0.0, "default", True),
    (2, "hlld", "hlld", 2, 1.0, "raised", False), (2, "roe", "llf", 1, 1.0, "raised", True), (2, "hlld", "hlld", 2, 0.0, "raised", True),
    (3, "hlld", "hlld", 2, 1.0, "raised", False), (3, "roe", "llf", 1, 0.0, "raised", True)])
def test_mhd_amr_mode_at_the_floors(orc, ndim, r1, r2, slope_type, field_scale, floors, resident):
    """AMR mode on the imhd-tube (1-D), Orszag-Tang (2-D) and nested 3-D meshes with every cell holding floor-state draws
    (fill_mhd_floor_cells; field_scale = 0: field-free trees), host-driven and through rgpu_amr_steps: one coarse step equals the
    oracle's amr_step bit for bit.  The 2-D and 3-D trees run under raised floors only: under the RAMSES floors the oracle's own
    update of those trees is not finite."""
    from helpers import fill_mhd_floor_cells
    from test_gpu_mhd import _mhd_amr_gpu_vs_oracle
    fill = lambda r: fill_mhd_floor_cells(r, floors, 41 + ndim, field_scale)
    if ndim == 1:
        from oracle.amr_mhd import MhdAmrRun
        from test_oracle_golden import IMHD
        r = MhdAmrRun(5, 9, (2, 2, 0, 0, 0, 0), 3.5, nsubcycle=[1, 1, 2, 2], riemann=r1, slope_type=slope_type, gamma=1.6666667,
                      courant_factor=0.8, err_grad_d=0.01, err_grad_u=0.05, err_grad_p=0.05, interpol_type=2, regions=IMHD,
                      tout=[1e9], ngridmax=10000)
        r.run(max_coarse=10)
        _mhd_amr_gpu_vs_oracle(r, 1, r1, r2, slope_type, 1, resident, fill=fill)
    elif ndim == 2:
        from oracle.amr_mhd import MhdAmrRun2D
        r = MhdAmrRun2D(4, 6, 1.0, nsubcycle=[1, 2], riemann=r1, riemann2d=r2, slope_type=slope_type, gamma=1.6666667,
                        courant_factor=0.8, err_grad_p=0.1, interpol_type=2, tout=[1e9], nexpand=1, ngridmax=20000)
        r.run(max_coarse=6)
        _mhd_amr_gpu_vs_oracle(r, 2, r1, r2, slope_type, 1, resident, fill=fill)
    else:
        from test_device_numerics_host import _mhd3_static_run
        r = _mhd3_static_run(r1, r2, slope_type)
        nlev = _mhd_amr_gpu_vs_oracle(r, 3, r1, r2, slope_type, 1, resident, regrid=False, fill=fill)
        assert nlev[2:] == [64, 64, 64]
    if field_scale == 0:
        assert (r.uold.reshape(11, -1)[5:] == 0).all()
