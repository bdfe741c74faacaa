"""GPU parity where the floors fire: near-vacuum and cold hypersonic states (helpers.floor_state) under the RAMSES floors
(smallr = smallc = 1e-10) and raised ones (smallr = 1e-3, smallc = 1e-2), through the C-ABI.  On these states ctoprim's density
and internal-energy floors, the face-density resets of the predictor, the pressure / density floors of cmpdt, the gravity
source's d_old = max(uold, smallr) and the passive-scalar fix of set_uold all take their floor branch; every run is compared with
the oracle on the same arrays, bit for bit ('exact': 1e-12, CUDA pow vs libm pow)."""
import contextlib
import ctypes as C

import numpy as np
import pytest

from helpers import FLOORS, Case, floor_counts, floor_state, max_rel_err

pytestmark = pytest.mark.gpu

NSTEP = 5


@pytest.fixture(scope="module")
def gpu():
    from ramses_b200 import lib
    lib.load()
    return lib


def _floor_case(ndim, level, coarse, floors, riemann="hllc", slope_type=1, bound=(0,) * 6, order=1, seed=3, nscalar=0):
    """Case on `coarse` domain cells (dx = 2^-level) holding a floor_state under the floors FLOORS[floors]; asserts that the
    ctoprim floors fire on it"""
    smallr, smallc = FLOORS[floors]
    c = Case(ndim, level, riemann=riemann, slope_type=slope_type, bound=bound, coarse=coarse, boxlen=float(coarse[0]), order=order,
             seed=seed, smallr=smallr, smallc=smallc, nvar=ndim + 2 + nscalar)
    d0 = floor_state(ndim, c.mesh.extent(level), seed, smallr, smallc, nscalar=nscalar)
    nrho, neint = floor_counts(d0, ndim, smallr, smallc)
    assert min(nrho, neint) >= max(2, 0.02 * d0[0].size), (nrho, neint)
    c.init_dense(d0)
    return c


def _oracle_steps(c, nstep=NSTEP):
    ref, dts = c.oracle_steps(nstep, nthreads=8)
    assert np.isfinite(ref).all() and np.isfinite(dts).all() and (dts > 0).all()
    return ref, dts


def _check(c, got, dts, ref, dts_ref, exact=False):
    idx = c.active_cells()
    ref = ref.reshape(c.nvar, -1)
    assert np.abs(ref[:, idx] - c.u.reshape(c.nvar, -1)[:, idx]).max() > 1e-4
    assert np.isfinite(got[:, idx]).all()
    if exact:
        assert np.allclose(dts, dts_ref, rtol=1e-12, atol=0)
        assert max_rel_err(got[:, idx], ref[:, idx]) <= 1e-12
    else:
        assert np.array_equal(dts, dts_ref), (dts, dts_ref)
        assert np.array_equal(got[:, idx], ref[:, idx]), float(np.abs(got[:, idx] - ref[:, idx]).max())


def _level_steps(c, nstep=NSTEP, force=None, **attrs):
    from ramses_b200.hydro import HydroGPU
    a = c.amr_commons()
    for k, v in attrs.items():
        setattr(a, k, v)
    h = HydroGPU(a)
    h.bind_level(c.level)
    info = h.level_info(c.level)
    h.upload_state(c.level)
    if force is not None:
        h.upload_force(force)
    dts, _ = h.level_steps(c.level, nstep)
    h.download_state(c.level)
    h.finalize()
    return a, np.asarray(dts), info


@pytest.mark.parametrize("floors", ["default", "raised"])
@pytest.mark.parametrize("sweep,coarse,level,riemann,slope_type", [
    (None, (2, 1, 1), 4, "hllc", 1), (None, (1, 2, 1), 4, "exact", 2), (None, (1, 1, 2), 4, "llf", 8),
    (None, (2, 1, 1), 4, "acoustic", 2), (None, (1, 2, 1), 4, "hll", 1),
    ("old", (2, 1, 1), 4, "hllc", 2), ("old", (1, 1, 2), 4, "exact", 1)])
def test_level_steps_3d_at_the_floors(gpu, monkeypatch, floors, sweep, coarse, level, riemann, slope_type):
    """rgpu_level_steps on a 32x16x16 floor_state, with the default 3-D kernel (sweep3_kernel) and with the round-1 kernel
    (RGPU_SWEEP=old at bind): state and dt history of 5 steps equal the oracle's"""
    if sweep:
        monkeypatch.setenv("RGPU_SWEEP", sweep)
    c = _floor_case(3, level, coarse, floors, riemann, slope_type)
    ref, dts_ref = _oracle_steps(c)
    a, dts, info = _level_steps(c)
    assert info.dense == 1 and (info.sweep_variant == 0) == (sweep == "old")
    _check(c, a.uold, dts, ref, dts_ref, exact=riemann == "exact")


@pytest.mark.parametrize("floors", ["default", "raised"])
@pytest.mark.parametrize("ndim,coarse,level,bound,riemann,slope_type", [
    (1, (4, 1, 1), 5, (1, 1, 0, 0, 0, 0), "hllc", 2),          # 128 cells between reflexive walls
    (1, (4, 1, 1), 5, (2, 2, 0, 0, 0, 0), "exact", 1),         # outflow ends
    (2, (2, 1, 1), 5, (0, 0, 1, 1, 0, 0), "llf", 8),           # 64 x 32, walls in y
    (2, (1, 2, 1), 5, (2, 2, 0, 0, 0, 0), "hll", 1),           # 32 x 64, outflow x
])
def test_level_steps_1d_2d_at_the_floors(gpu, floors, ndim, coarse, level, bound, riemann, slope_type):
    """the 1-D and 2-D sweep_dense_kernel on a floor_state with a wall or outflow on one axis: 5 fused steps equal the oracle"""
    c = _floor_case(ndim, level, coarse, floors, riemann, slope_type, bound=bound, order=2)
    ref, dts_ref = _oracle_steps(c)
    a, dts, info = _level_steps(c)
    assert info.dense == 1
    _check(c, a.uold, dts, ref, dts_ref, exact=riemann == "exact")


@pytest.mark.parametrize("floors", ["default", "raised"])
@pytest.mark.parametrize("riemann", ["hllc", "exact"])
def test_split_sequence_and_courant_at_the_floors(gpu, floors, riemann):
    """rgpu_courant_fine alone (dt and the mass / kinetic / internal energy sums; the internal energy of a cold hypersonic cell is
    negative), then the split sequence courant_fine -> set_unew -> godunov_fine_dev -> set_uold -> make_boundary_hydro for 4
    steps: equal the oracle's"""
    from oracle import orc
    from ramses_b200.hydro import HydroGPU
    c = _floor_case(3, 4, (2, 1, 1), floors, riemann, 1)
    dt0, sums0 = c.oracle_courant()
    L = orc.lib()
    u, unew, dts_ref = c.u.copy(), np.zeros_like(c.u), []
    for _ in range(4):
        dt = L.orc_courant_fine(C.byref(c.p), c.mesh.ptr, c.level, c.p.boxlen / c.p.smallc, orc.dptr(u), orc.dptr(np.zeros(3)))
        L.orc_set_unew(C.byref(c.p), c.mesh.ptr, c.level, orc.dptr(u), orc.dptr(unew))
        L.orc_godunov_fine(C.byref(c.p), c.mesh.ptr, c.level, dt, orc.dptr(u), orc.dptr(unew), 8)
        L.orc_set_uold(C.byref(c.p), c.mesh.ptr, c.level, orc.dptr(u), orc.dptr(unew))
        L.orc_make_boundary_hydro(C.byref(c.p), c.mesh.ptr, c.level, orc.dptr(u))
        dts_ref.append(dt)
    assert np.isfinite(u).all()
    a = c.amr_commons()
    h = HydroGPU(a)
    h.bind_level(c.level)
    h.upload_state(c.level)
    a.dtnew[c.level] = a.boxlen / a.smallc
    a.mass_tot = a.ekin_tot = a.eint_tot = 0.0
    dt_g = h.courant_fine(c.level)
    assert dt_g == dt0
    for got, ref in ((a.mass_tot, sums0[0]), (a.ekin_tot, sums0[1])):
        assert abs(got - ref) <= 1e-13 * abs(ref), (got, ref)
    assert abs(a.eint_tot - sums0[2]) <= 1e-13 * (abs(sums0[1]) + abs(sums0[2])), (a.eint_tot, sums0[2])
    dts = []
    for _ in range(4):
        a.dtnew[c.level] = a.boxlen / a.smallc
        dts.append(h.courant_fine(c.level))
        h.set_unew(c.level); h.godunov_fine_dev(c.level); h.set_uold(c.level); h.make_boundary_hydro(c.level)
    h.download_state(c.level)
    h.finalize()
    _check(c, a.uold, np.array(dts), u, np.array(dts_ref), exact=riemann == "exact")


@pytest.mark.parametrize("floors", ["default", "raised"])
def test_level0_godunov_fine_at_the_floors(gpu, floors):
    """rgpu_godunov_fine on host arrays (Level 0) of a 64x32x32 floor_state: unew equals orc_godunov_fine's"""
    from ramses_b200.hydro import HydroGPU
    c = _floor_case(3, 5, (2, 1, 1), floors, "hllc", 2)
    dt, _ = c.oracle_courant()
    ref = c.oracle_godunov(dt, nthreads=8).reshape(c.nvar, -1)
    assert np.isfinite(ref).all()
    a = c.amr_commons()
    h = HydroGPU(a)
    h.bind_level(c.level)
    assert h.level_info(c.level).dense == 1
    a.dtnew[c.level] = dt
    a.unew[:, :] = a.uold
    h.godunov_fine(c.level)
    h.finalize()
    idx = c.active_cells()
    assert np.array_equal(a.unew[:, idx], ref[:, idx])


@pytest.mark.parametrize("floors", ["default", "raised"])
@pytest.mark.parametrize("ndim,coarse,level,riemann,slope_type", [(1, (4, 1, 1), 5, "hllc", 2), (2, (2, 1, 1), 5, "llf", 1),
                                                                  (3, (2, 1, 1), 4, "hllc", 1), (3, (1, 2, 1), 4, "exact", 2)])
def test_poisson_level_steps_at_the_floors(gpu, floors, ndim, coarse, level, riemann, slope_type):
    """poisson on the dense sweep with rgpu_upload_force and an acceleration strong enough to move floored densities: the
    predictor, the source term with d_old = max(uold, smallr) and the gravity-limited Courant scan give the oracle's state and
    dt history over 5 steps"""
    from test_gpu_gravity_dense import Gravity, force_field
    c = _floor_case(ndim, level, coarse, floors, riemann, slope_type)
    f = force_field(ndim, c.mesh.s.ncell, 200.0, 9 + ndim)
    with Gravity(f):
        ref, dts_ref = _oracle_steps(c)
    a, dts, info = _level_steps(c, force=f, poisson=True)
    assert info.dense == 1
    _check(c, a.uold, dts, ref, dts_ref, exact=riemann == "exact")


@pytest.mark.parametrize("floors", ["default", "raised"])
@pytest.mark.parametrize("dense,nscalar,poisson", [("0", 0, False), ("1", 0, False), ("1", 0, True), ("0", 2, False)])
def test_amr_mode_at_the_floors(gpu, monkeypatch, floors, dense, nscalar, poisson):
    """AMR mode (rgpu_set_amr) on a 3x2x1 domain refined to level 3 holding a floor_state, swept by the oct-batch kernel
    (RGPU_AMR_DENSE=0) and by the dense AMR variant, with poisson, and with two passive scalars whose cells cross smallr in
    both directions (amr_scalar_floor_kernel, godunov_fine.f90:176-190): 3 level steps in amr_step order equal the oracle.
    level_info reports which kernel swept the level."""
    from ramses_b200.hydro import HydroGPU
    from test_gpu_gravity_dense import Gravity, force_field
    monkeypatch.setenv("RGPU_AMR_DENSE", dense)
    level = 3
    c = _floor_case(3, level, (3, 2, 1), floors, "hllc", 2, order=2, nscalar=nscalar)
    f = force_field(3, c.mesh.s.ncell, 200.0, 5) if poisson else None
    with Gravity(f) if poisson else contextlib.nullcontext():
        ref, dts_ref = _oracle_steps(c, 3)
        if nscalar:
            dt, _ = c.oracle_courant()
            one = c.oracle_godunov(dt, nthreads=8).reshape(c.nvar, -1)[0]
            old = c.u.reshape(c.nvar, -1)[0]
            idx = c.active_cells()
            up = (old[idx] < c.p.smallr) & (one[idx] > old[idx])
            down = (one[idx] < c.p.smallr) & (old[idx] > one[idx])
            assert up.sum() > 0 and down.sum() > 0
    a = c.amr_commons()
    a.poisson = poisson
    h = HydroGPU(a, amr_mode=True)
    for l in range(1, level + 1):
        h.bind_level(l)
    info = h.level_info(level)
    if nscalar == 0:
        assert info.dense == int(dense)
    h.upload_state(0)
    if poisson:
        h.upload_force(f)
    h.make_boundary_hydro(level)
    dts = []
    for _ in range(3):
        a.dtnew[level] = a.boxlen / a.smallc
        dts.append(h.courant_fine(level))
        h.set_unew(level); h.godunov_fine_dev(level); h.set_uold(level); h.make_boundary_hydro(level)
    h.download_state(0)
    h.finalize()
    _check(c, a.uold, np.array(dts), ref, dts_ref)


@pytest.mark.parametrize("ndim,gravity,resident,floors", [
    (1, True, False, "default"), (1, True, False, "raised"), (2, True, False, "default"), (2, True, True, "raised"),
    (3, True, False, "raised"), (3, False, True, "raised")])
def test_refined_mesh_pressure_fix_at_the_floors(gpu, ndim, gravity, resident, floors):
    """pressure_fix (and poisson) on an adaptively refined mesh -- coarse-fine faces refluxed, ghost octs prolongated from floored
    father cells -- every cell of which holds a floor_state cell: one sub-cycled coarse step, host-driven and through
    rgpu_amr_steps, gives the oracle's state, divu, enew and dtnew bit for bit.  At the cold hypersonic cells E/rho - ekin is
    below smalle, where enew, add_pdv_source_terms and the energy switch decide the new energy.  (The 3-D mesh under the RAMSES
    floors is left out: with pressure_fix the oracle itself gives non-finite values in a few cells of that step.)"""
    from test_gpu_amr import BOUND_2D_WALLS_X_OUTFLOW_Y, SOD, run_case
    kw = dict(gravity=gravity, pressure_fix=True, device_resident=resident, floors=floors)
    if ndim == 1:
        got, ref, dtnew, r, nlev = run_case(1, 3, 8, (1, 1, 0, 0, 0, 0), SOD, "hllc", 2, 6, 2, [1, 1, 1, 2], **kw)
    elif ndim == 2:
        regs = [dict(type="square", x_center=0.5, y_center=0.5, length_x=10, length_y=10, exp_region=10, d=1.0, p=0.1),
                dict(type="square", x_center=0.3, y_center=0.4, length_x=0.3, length_y=0.25, exp_region=2, d=2.0, u=0.3, v=-0.2, p=1.0)]
        got, ref, dtnew, r, nlev = run_case(2, 3, 5, (1, 1, 2, 2, 0, 0), regs, "hllc", 2, 2, 2, [1, 2],
                                            bound_regions=BOUND_2D_WALLS_X_OUTFLOW_Y, **kw)
    else:
        regs = [dict(type="square", x_center=0.5, y_center=0.5, z_center=0.5, length_x=10, length_y=10, length_z=10, exp_region=10,
                     d=1.0, p=1e-5),
                dict(type="square", x_center=0.4, y_center=0.45, z_center=0.55, length_x=0.3, length_y=0.3, length_z=0.3, exp_region=2,
                     d=1.5, p=2.0)]
        got, ref, dtnew, r, nlev = run_case(3, 3, 4, (0,) * 6, regs, "hllc", 1, 1, 1, [2, 2], **kw)
    assert sum(1 for n in nlev[r.levelmin:] if n > 0) >= 1
    assert np.isfinite(ref).all()
    assert dtnew[r.levelmin] == r.dtnew[r.levelmin]
    assert np.array_equal(got, ref), float(np.abs(got - ref).max())
    dk, do, ek, eo = r.pfix_cmp
    assert np.array_equal(dk, do) and np.array_equal(ek, eo)
    assert np.abs(do).max() > 0


@pytest.mark.parametrize("floors", ["default", "raised"])
def test_fast_mode_at_the_floors(gpu, floors):
    """rgpu_params.fast = 1 on a 32x16x16 floor_state: FMA contraction may flip a branch next to a floor, so the 1e-12 bound of the
    strict kernels does not apply; the fast run differs from the strict one, stays finite with positive time steps, keeps the
    and stays within 1e-9 of the strict run (measured on one H100: 3.6e-12 with the RAMSES floors, 1.1e-15 with raised ones);
    the deviation is printed"""
    c = _floor_case(3, 4, (2, 1, 1), floors, "hllc", 1)
    (as_, dts_s, _), (af, dts_f, info) = _level_steps(c), _level_steps(c, fast=True)
    idx = c.active_cells()
    us, uf = as_.uold[:, idx], af.uold[:, idx]
    assert info.sweep_variant != 0
    assert np.isfinite(uf).all() and np.isfinite(dts_f).all() and (dts_f > 0).all()
    assert not np.array_equal(uf, us)
    assert max_rel_err(uf, us) <= 1e-9
    print(f"fast vs strict ({floors} floors): max rel. deviation {max_rel_err(uf, us):.3e}, "
          f"dt {np.abs(dts_f / dts_s - 1).max():.3e}")
