"""GPU parity away from the suite's one namelist point, through the C-ABI: gamma, courant_factor, slope_theta, niter_riemann,
the box scale boxlen / nx, beta_fix and the refinement thresholds.  The parameter sets are those of tests/test_parameters_host.py,
and each test family here shows on the oracle, on its own states and meshes, that setting any one parameter of its set back to
the suite's value changes the compared result.  Beyond the emulated kernels, these
runs check the routes only the device build has: the constants rgpu_init derives from gamma and courant_factor (smalle, smallp,
entho, gamma6, cfl_k, ...), the kernel arguments passed one by one (the pdV pass, the energy switch, hydro_flag, the Courant caps
courant_factor dx / smallc and boxlen / smallc) and the cell size of every level.  Every comparison is bit for bit ('exact': 1e-12,
CUDA pow vs libm pow)."""
import ctypes as C

import numpy as np
import pytest

from helpers import Case, MhdCase, box_state, max_rel_err, mhd_box_state
from test_parameters_host import (BETA_FIX, H1, H2, HSETS, M1, MSUITE, SUITE, THRESHOLDS, _assert_each_parameter_matters, _flag_state,
                                  _scaled, _src_oracle, mhd_amr_oracle)

pytestmark = pytest.mark.gpu

NSTEP = 4
SOLVERS = ["llf", "exact", "acoustic", "hllc", "hll"]


@pytest.fixture(scope="module")
def gpu():
    from ramses_b200 import lib
    lib.load()
    return lib


def _case(ndim, level, coarse, ps, riemann, slope_type=8, bound=(0,) * 6, order=1, seed=3):
    """Case on `coarse` domain cells of size ps['scale'] with a box_state at the set's gamma and a pressure-100 blast in it"""
    c = Case(ndim, level, riemann=riemann, slope_type=slope_type, bound=bound, coarse=coarse, boxlen=ps["scale"] * coarse[0], order=order,
             seed=seed, gamma=ps["gamma"], courant_factor=ps["courant_factor"], slope_theta=ps["slope_theta"],
             niter_riemann=ps["niter_riemann"])
    d = box_state(ndim, c.mesh.extent(level), gamma=ps["gamma"])
    blast = np.zeros(d[0].shape, dtype=bool)
    blast[tuple(slice(s // 3, s // 3 + max(1, s // 8)) for s in d[0].shape)] = True
    d[ndim + 1][blast] += 100.0 / (ps["gamma"] - 1)
    c.init_dense(d)
    return c


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


@pytest.mark.parametrize("pset", ["H1", "H2"])
@pytest.mark.parametrize("riemann", SOLVERS)
def test_level_steps_3d_at_parameter_sets(gpu, pset, riemann):
    """rgpu_level_steps on a 32x16x16 periodic box of scale 0.75 / 3, slope_type 8, at the set's gamma, courant_factor,
    slope_theta and niter_riemann: state and dt history of 4 steps equal the oracle's"""
    c = _case(3, 4, (2, 1, 1), HSETS[pset], riemann)
    ref, dts_ref = c.oracle_steps(NSTEP, nthreads=8)
    a, dts, info = _level_steps(c)
    assert info.dense == 1
    _check(c, a.uold, dts, ref, dts_ref, exact=riemann == "exact")
    if riemann == "exact":
        _assert_each_parameter_matters(lambda q: _case(3, 4, (2, 1, 1), q, riemann).oracle_steps(NSTEP, nthreads=8), HSETS[pset], SUITE)


def test_fast_mode_at_h1(gpu):
    """rgpu_params.fast = 1 at H1 (slope_type 8): the fast run differs from the strict one, which equals the oracle, and stays
    within the FAST tolerance of 1e-12 of both, time steps included; the deviation is printed"""
    c = _case(3, 4, (2, 1, 1), H1, "hllc")
    (as_, dts_s, _), (af, dts_f, info) = _level_steps(c), _level_steps(c, fast=True)
    ref, dts_ref = c.oracle_steps(NSTEP, nthreads=8)
    _check(c, as_.uold, dts_s, ref, dts_ref)
    idx = c.active_cells()
    us, uf, ur = as_.uold[:, idx], af.uold[:, idx], ref.reshape(c.nvar, -1)[:, idx]
    assert info.sweep_variant != 0
    assert not np.array_equal(uf, us)
    print(f"fast vs strict at H1: max rel. deviation {max_rel_err(uf, us):.3e}, dt {np.abs(dts_f / dts_s - 1).max():.3e}")
    assert max_rel_err(uf, us) <= 1e-12 and max_rel_err(uf, ur) <= 1e-12
    assert np.allclose(dts_f, dts_ref, rtol=1e-12, atol=0)


@pytest.mark.parametrize("pset", ["H1", "H2"])
@pytest.mark.parametrize("ndim,coarse,level,bound,riemann", [
    (1, (4, 1, 1), 5, (1, 1, 0, 0, 0, 0), "exact"), (1, (4, 1, 1), 5, (2, 2, 0, 0, 0, 0), "hllc"),
    (2, (2, 1, 1), 5, (0, 0, 1, 1, 0, 0), "exact"), (2, (1, 2, 1), 5, (2, 2, 0, 0, 0, 0), "llf")])
def test_level_steps_1d_2d_at_parameter_sets(gpu, pset, ndim, coarse, level, bound, riemann):
    """the 1-D and 2-D sweep_dense_kernel with walls or outflow on one axis, at box scale 0.75 / 3 and the set's parameters:
    4 fused steps equal the oracle's"""
    c = _case(ndim, level, coarse, HSETS[pset], riemann, bound=bound, order=2)
    ref, dts_ref = c.oracle_steps(NSTEP, nthreads=8)
    a, dts, info = _level_steps(c)
    assert info.dense == 1
    _check(c, a.uold, dts, ref, dts_ref, exact=riemann == "exact")
    if riemann == "exact":
        _assert_each_parameter_matters(lambda q: _case(ndim, level, coarse, q, riemann, bound=bound, order=2).oracle_steps(NSTEP, nthreads=8),
                                       HSETS[pset], SUITE)


@pytest.mark.parametrize("pset", ["H1", "H2"])
@pytest.mark.parametrize("riemann", ["hllc", "exact"])
def test_split_sequence_at_parameter_sets(gpu, pset, riemann):
    """courant_fine -> set_unew -> godunov_fine_dev -> set_uold -> make_boundary_hydro for 4 steps at the set's parameters: dt of
    every step (the Courant cap courant_factor dx / smallc and the derived cfl_k) and the state equal the oracle's"""
    from oracle import orc
    from ramses_b200.hydro import HydroGPU
    c = _case(3, 4, (2, 1, 1), HSETS[pset], riemann, bound=(1, 1, 2, 2, 0, 0), order=2)
    L = orc.lib()
    u, unew, dts_ref = c.u.copy(), np.zeros_like(c.u), []
    for _ in range(NSTEP):
        dt = L.orc_courant_fine(C.byref(c.p), c.mesh.ptr, c.level, c.p.boxlen / c.p.smallc, orc.dptr(u), orc.dptr(np.zeros(3)))
        L.orc_set_unew(C.byref(c.p), c.mesh.ptr, c.level, orc.dptr(u), orc.dptr(unew))
        L.orc_godunov_fine(C.byref(c.p), c.mesh.ptr, c.level, dt, orc.dptr(u), orc.dptr(unew), 8)
        L.orc_set_uold(C.byref(c.p), c.mesh.ptr, c.level, orc.dptr(u), orc.dptr(unew))
        L.orc_make_boundary_hydro(C.byref(c.p), c.mesh.ptr, c.level, orc.dptr(u))
        dts_ref.append(dt)
    a = c.amr_commons()
    h = HydroGPU(a)
    h.bind_level(c.level)
    h.upload_state(c.level)
    dts = []
    for _ in range(NSTEP):
        a.dtnew[c.level] = a.boxlen / a.smallc
        dts.append(h.courant_fine(c.level))
        h.set_unew(c.level); h.godunov_fine_dev(c.level); h.set_uold(c.level); h.make_boundary_hydro(c.level)
    h.download_state(c.level)
    h.finalize()
    _check(c, a.uold, np.array(dts), u, np.array(dts_ref), exact=riemann == "exact")
    if riemann == "exact":     # orc_run_uniform is this call sequence
        _assert_each_parameter_matters(lambda q: _case(3, 4, (2, 1, 1), q, riemann, bound=(1, 1, 2, 2, 0, 0), order=2).oracle_steps(NSTEP),
                                       HSETS[pset], SUITE)


@pytest.mark.parametrize("pset", ["H1", "H2"])
def test_level0_godunov_fine_at_parameter_sets(gpu, pset):
    """rgpu_godunov_fine on host arrays (Level 0) at the set's parameters: unew equals orc_godunov_fine's"""
    from ramses_b200.hydro import HydroGPU
    c = _case(3, 4, (2, 1, 1), HSETS[pset], "hllc")
    dt, _ = c.oracle_courant()
    ref = c.oracle_godunov(dt, nthreads=8).reshape(c.nvar, -1)
    a = c.amr_commons()
    h = HydroGPU(a)
    h.bind_level(c.level)
    a.dtnew[c.level] = dt
    a.unew[:, :] = a.uold
    h.godunov_fine(c.level)
    h.finalize()
    idx = c.active_cells()
    assert np.array_equal(a.unew[:, idx], ref[:, idx])

    def run(q):
        c2 = _case(3, 4, (2, 1, 1), q, "hllc")
        return (c2.oracle_godunov(dt, nthreads=8),)
    _assert_each_parameter_matters(run, HSETS[pset], SUITE, ("gamma", "slope_theta", "scale"))


@pytest.mark.parametrize("pset", ["H1", "H2"])
@pytest.mark.parametrize("ndim,coarse,level,riemann", [(1, (4, 1, 1), 5, "hllc"), (2, (2, 1, 1), 5, "exact"), (3, (2, 1, 1), 4, "hllc")])
def test_poisson_level_steps_at_parameter_sets(gpu, pset, ndim, coarse, level, riemann):
    """poisson on the dense sweep at box scale 0.75 / 3: the gravity term of the Courant scan reads dx; state and dt history of 4
    steps equal the oracle's"""
    from test_gpu_gravity_dense import Gravity, force_field
    c = _case(ndim, level, coarse, HSETS[pset], riemann)
    f = force_field(ndim, c.mesh.s.ncell, 20.0, 7 + ndim)
    with Gravity(f):
        ref, dts_ref = c.oracle_steps(NSTEP, nthreads=8)
    a, dts, info = _level_steps(c, force=f, poisson=True)
    _check(c, a.uold, dts, ref, dts_ref, exact=riemann == "exact")
    if riemann == "exact":
        def run(q):
            with Gravity(f):
                return _case(ndim, level, coarse, q, riemann).oracle_steps(NSTEP, nthreads=8)
        _assert_each_parameter_matters(run, HSETS[pset], SUITE)


# ---- AMR mode --------------------------------------------------------------------------------------------------------------------
SOD = [dict(type="square", x_center=0.25, length_x=0.5, d=1.0, p=10.0), dict(type="square", x_center=0.75, length_x=0.5, d=0.125, p=1e-4)]
REG2 = [dict(type="square", x_center=0.5, y_center=0.5, length_x=10, length_y=10, exp_region=10, d=1.0, p=1e-3),
        dict(type="square", x_center=0.3, y_center=0.4, length_x=0.3, length_y=0.25, exp_region=2, d=2.0, u=0.3, v=-0.2, p=1.0)]
REG3 = [dict(type="square", x_center=0.5, y_center=0.5, z_center=0.5, length_x=10, length_y=10, length_z=10, exp_region=10, d=1.0, p=1e-3),
        dict(type="square", x_center=0.4, y_center=0.45, z_center=0.55, length_x=0.3, length_y=0.3, length_z=0.3, exp_region=2, d=1.5, u=0.2,
             p=2.0)]


def _amr(ndim, ps, riemann="hllc", ncoarse=3, **kw):
    """run_case at the set's parameters on the meshes of tests/test_gpu_amr.py, placed in a box of the set's scale"""
    from test_gpu_amr import BOUND_2D_WALLS_X_OUTFLOW_Y, run_case
    prm = dict(gamma=ps["gamma"], courant_factor=ps["courant_factor"], slope_theta=ps["slope_theta"], niter_riemann=ps["niter_riemann"],
               boxlen=ps["scale"], ncoarse=ncoarse)
    prm.update(kw)
    if ndim == 1:
        return run_case(1, 3, 7, (1, 1, 0, 0, 0, 0), _scaled(SOD, ps["scale"]), riemann, 8, 4, 2, [1, 1, 2], **prm)
    if ndim == 2:
        return run_case(2, 3, 5, (1, 1, 2, 2, 0, 0), _scaled(REG2, ps["scale"]), riemann, 8, 2, 2, [1, 2],
                        bound_regions=BOUND_2D_WALLS_X_OUTFLOW_Y, **prm)
    return run_case(3, 3, 4, (0,) * 6, _scaled(REG3, ps["scale"]), riemann, 8, 1, 1, [2, 2], **prm)


def _amr_oracle(r, q):
    """set_unew + godunov_fine and courant_fine of every populated level of the frozen mesh and state of run r (after its compared
    steps) with the parameters q: what the AMR comparisons look at"""
    from oracle import orc
    L = orc.lib()
    p = orc.make_params(ndim=r.ndim, nvar=r.nvar, riemann=r.p.riemann, slope_type=r.p.slope_type, gamma=q["gamma"],
                        courant_factor=q["courant_factor"], boxlen=q["scale"], nvector=r.p.nvector, slope_theta=q["slope_theta"],
                        niter_riemann=q["niter_riemann"])
    out = []
    for l in range(r.levelmin, r.nlevelmax + 1):
        if len(r.active[l]) == 0:
            continue
        unew = np.zeros_like(r.uold)
        L.orc_set_unew(C.byref(p), r.mp, l, orc.dptr(r.uold), orc.dptr(unew))
        L.orc_godunov_fine(C.byref(p), r.mp, l, 0.4 * r.dtnew[r.levelmin] / 2 ** (l - r.levelmin), orc.dptr(r.uold), orc.dptr(unew), 8)
        dt = L.orc_courant_fine(C.byref(p), r.mp, l, q["scale"] / p.smallc, orc.dptr(r.uold), orc.dptr(np.zeros(3)))
        out += [unew, np.array([dt])]
    return tuple(out)


def _check_amr(got, ref, dtnew, r, exact=False):
    lm = r.levelmin
    assert np.isfinite(got).all()
    if exact:
        assert abs(dtnew[lm] / r.dtnew[lm] - 1) <= 1e-12
        assert (np.abs(got - ref) / np.abs(ref).max(axis=1, keepdims=True)).max() <= 1e-12
    else:
        assert dtnew[lm] == r.dtnew[lm], (dtnew[lm], r.dtnew[lm])
        assert np.array_equal(got, ref), float(np.abs(got - ref).max())


@pytest.mark.parametrize("pset", ["H1", "H2"])
@pytest.mark.parametrize("ndim,riemann,resident,dense", [(1, "hllc", False, "0"), (1, "exact", True, "0"), (2, "hllc", True, "0"),
                                                        (2, "exact", False, "0"), (3, "hllc", False, "0"), (3, "exact", True, "0"),
                                                        (3, "hllc", True, "1"), (3, "llf", False, "1")])
def test_amr_mode_at_parameter_sets(gpu, monkeypatch, pset, ndim, riemann, resident, dense):
    """three sub-cycled coarse steps of a refined mesh in a box of scale 0.75 / 3 at the set's parameters, slope_type 8,
    host-driven and through rgpu_amr_steps (its CUDA graph is replayed from the second coarse step on), with the oct-batch
    kernel and with the dense base box + patches (RGPU_AMR_DENSE): state and dtnew equal the oracle's"""
    monkeypatch.setenv("RGPU_AMR_DENSE", dense)
    got, ref, dtnew, r, nlev = _amr(ndim, HSETS[pset], riemann, device_resident=resident)
    assert sum(1 for n in nlev[r.levelmin:] if n > 0) >= 1
    if ndim == 3:                # the fully refined base level: the dense AMR variant, or the oct-batch kernel
        assert r.dev_info[r.levelmin].dense == int(dense)
    _check_amr(got, ref, dtnew, r, exact=riemann == "exact")
    if riemann == "exact":
        _assert_each_parameter_matters(lambda q: _amr_oracle(r, q), HSETS[pset], SUITE)


@pytest.mark.parametrize("ndim,ivar", [(1, 1), (2, 2), (3, 1), (3, 2)])
def test_amr_interpol_var_at_h2(gpu, ndim, ivar):
    """interpol_var 1 and 2 (the ghost prolongation and upload_fine through the internal energy, gamma-dependent) at H2"""
    got, ref, dtnew, r, nlev = _amr(ndim, H2, "hllc", ncoarse=2, interpol_var=ivar)
    _check_amr(got, ref, dtnew, r)
    _assert_each_parameter_matters(lambda q: _amr_oracle(r, q), H2, SUITE, ("gamma", "slope_theta", "scale"))


@pytest.mark.parametrize("beta_fix", BETA_FIX)
@pytest.mark.parametrize("pset,ndim,resident", [("H1", 1, False), ("H2", 2, True), ("H1", 3, True), ("H2", 3, False)])
def test_amr_poisson_pressure_fix_at_parameter_sets(gpu, pset, ndim, resident, beta_fix):
    """poisson and pressure_fix on refined meshes of scale 0.75 / 3 at beta_fix 0, 0.5 and 4: the pdV pass (dx_loc, 1.5 dx_loc),
    the energy switch (beta_fix, dx) and the gravity-limited Courant step give the oracle's state, divu, enew and dtnew"""
    got, ref, dtnew, r, nlev = _amr(ndim, HSETS[pset], "hllc", ncoarse=2, gravity=True, pressure_fix=True, beta_fix=beta_fix,
                                    device_resident=resident)
    _check_amr(got, ref, dtnew, r)
    dk, do, ek, eo = r.pfix_cmp
    assert np.array_equal(dk, do) and np.array_equal(ek, eo)
    assert np.abs(do).max() > 0
    from oracle import orc
    ps = HSETS[pset]
    force = np.ascontiguousarray(np.random.default_rng(3).standard_normal((ndim, r.ncell)) * 5.0)
    levels = [l for l in range(r.levelmin, r.nlevelmax + 1) if len(r.active[l])]

    def run(q, b):             # the passes of set_unew -> godunov_fine -> set_uold on the compared mesh and state, level by level
        return sum((_src_oracle(orc, r, l, q, b, force) for l in levels), ())
    base = run(ps, beta_fix)
    assert any(not np.array_equal(x, y) for x, y in zip(base, run(SUITE, beta_fix)))            # the scale reaches it
    if beta_fix != 0.5:
        assert any(not np.array_equal(x, y) for x, y in zip(base, run(ps, 0.5)))                # and beta_fix


@pytest.mark.parametrize("ndim", [1, 2, 3])
def test_hydro_flag_on_device_at_threshold_sets(gpu, ndim):
    """rgpu_hydro_flag at gamma 5/3 with the threshold sets of the CPU tests (distinct, each criterion alone, all off) and raised
    floors, on the developed mesh with per-cell noise (test_parameters_host._flag_state): flag1 of every active cell of every level
    below levelmax equals the oracle's hydro_flag; the raised floors and each threshold of the distinct set change the flags"""
    from oracle.amr import AmrRun
    from ramses_b200.hydro import HydroGPU
    from test_gpu_amr import BOUND_2D_WALLS_X_OUTFLOW_Y, commons_from_run
    kw = dict(gamma=H1["gamma"], riemann="hllc", slope_type=2, err_grad_d=0.05, err_grad_u=0.05, err_grad_p=0.05, tout=[1e9], ngridmax=20000)
    if ndim == 1:
        r = AmrRun(1, 3, 7, (1, 1, 0, 0, 0, 0), 0.75, nsubcycle=[1, 2], interpol_type=2, regions=_scaled(SOD, 0.75), **kw)
    elif ndim == 2:
        r = AmrRun(2, 3, 5, (1, 1, 2, 2, 0, 0), 0.75, nsubcycle=[1, 2], interpol_type=2, regions=_scaled(REG2, 0.75),
                   bound_regions=BOUND_2D_WALLS_X_OUTFLOW_Y, **kw)
    else:
        r = AmrRun(3, 3, 4, (0,) * 6, 0.75, nsubcycle=[2, 2], interpol_type=1, regions=_scaled(REG3, 0.75), **kw)
    r.flag_coarse(); r.init_refine(); r.init_refine_2()
    for i in range(r.levelmin, r.nlevelmax + 1):
        if i > r.levelmin:
            r.make_boundary_hydro(i)
        r.refine_fine(i)
    for l in range(1, r.nlevelmax + 1):
        r.make_boundary_hydro(l)
    r.uold[:] = _flag_state(r, 90 + ndim)           # relative gradients spread across the thresholds
    a = commons_from_run(r, "hllc", r.p.slope_type)
    h = HydroGPU(a, amr_mode=True, interpol_type=1)
    for l in range(1, r.nlevelmax + 1):
        if len(a.active[l]):
            h.bind_level(l)
    h.upload_state(0)
    sets = [(err, (1e-10,) * 3) for err in THRESHOLDS.values()] + [((0.03, 0.2, 0.08), (0.5, 0.8, 0.3))]
    flags = []
    for err, flo in sets:
        r.err_grad_d, r.err_grad_u, r.err_grad_p = err
        r.floor_d, r.floor_u, r.floor_p = flo
        allflags = []
        for l in range(r.levelmin, r.nlevelmax):
            if not len(a.active[l]):
                continue
            flag1 = np.zeros(a.ncell, dtype=np.int32)
            h.hydro_flag(l, flag1, err, flo)
            r.flag1[:] = 0
            r.hydro_flag(l)
            assert np.array_equal(flag1, np.asarray(r.flag1[1:], dtype=np.int32)), (err, flo, l)
            allflags.append(flag1.copy())
        flags.append(np.concatenate(allflags))
    h.finalize()
    none, distinct, raised = flags[list(THRESHOLDS).index("none")], flags[list(THRESHOLDS).index("distinct")], flags[-1]
    assert none.sum() == 0 and distinct.sum() > 0
    assert not np.array_equal(raised, distinct)              # the raised floors change the flags
    # each threshold of the distinct set, set back to the suite's 0.05 alone, changes the oracle's flags
    for k in range(3):
        err = list(THRESHOLDS["distinct"])
        err[k] = 0.05
        r.err_grad_d, r.err_grad_u, r.err_grad_p = err
        r.floor_d = r.floor_u = r.floor_p = 1e-10
        other = []
        for l in range(r.levelmin, r.nlevelmax):
            if len(a.active[l]):
                r.flag1[:] = 0
                r.hydro_flag(l)
                other.append(np.asarray(r.flag1[1:], dtype=np.int32).copy())
        assert not np.array_equal(np.concatenate(other), distinct), k


# ---- MHD -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("coarse,level,bound,riemann,riemann2d,st,smt", [
    ((1, 1, 1), 4, (0,) * 6, "hlld", "hlld", 8, 1), ((2, 1, 1), 3, (0,) * 6, "roe", "llf", 8, 2),
    ((1, 2, 1), 3, (2, 2, 0, 0, 0, 0), "llf", "roe", 2, 2), ((2, 1, 1), 3, (0, 0, 1, 1, 0, 0), "hll", "hlla", 1, 1)])
def test_mhd_dense_at_m1(gpu, coarse, level, bound, riemann, riemann2d, st, smt):
    """the dense six-pass MHD sweep at gamma 1.4, courant_factor 0.5, slope_theta 1.2 and box scale 0.75 (slope_type 8 among
    the cases): 3 fused steps give the oracle's state and dt history (the fused Courant scan), and so does the split sequence
    with courant_fine alone each step"""
    from test_gpu_mhd import run_gpu

    def case(q):
        c = MhdCase(level, riemann=riemann, riemann2d=riemann2d, slope_type=st, slope_mag_type=smt, bound=bound, coarse=coarse,
                    boxlen=q["scale"] * coarse[0], order=2, seed=3, gamma=q["gamma"], courant_factor=q["courant_factor"],
                    slope_theta=q["slope_theta"])
        d0 = mhd_box_state(c.mesh.extent(level), gamma=q["gamma"])
        d0[0] *= 1 + 0.2 * (np.random.default_rng(4).standard_normal(d0[0].shape) > 1.3)
        c.init_dense(d0)
        return c
    c = case(M1)
    ref, dts_ref = c.oracle_steps(3)
    a, dts, _, info = run_gpu(c, 3)
    assert info.dense == 1
    act = c.active_cells()
    assert np.array_equal(dts, dts_ref), (dts, dts_ref)
    assert np.array_equal(a.uold[:, act], ref.reshape(11, -1)[:, act])
    assert np.abs(ref.reshape(11, -1)[:, act] - c.u.reshape(11, -1)[:, act]).max() > 1e-4
    a2, dts2, _, _ = run_gpu(c, 3, fused=False)
    assert np.array_equal(dts2, dts_ref)
    assert np.array_equal(a2.uold[:, act], ref.reshape(11, -1)[:, act])
    keys = ("gamma", "courant_factor", "scale") + (("slope_theta",) if st == 8 else ())
    _assert_each_parameter_matters(lambda q: case(q).oracle_steps(3), M1, MSUITE, keys)


@pytest.mark.parametrize("ndim,resident", [(1, False), (1, True), (2, False), (2, True), (3, False), (3, True)])
def test_mhd_amr_at_gamma_1_4(gpu, ndim, resident):
    """MHD in AMR mode (NDIM = 1, 2, 3) at gamma 1.4 and courant_factor 0.5, host-driven and through rgpu_amr_steps: 3 coarse
    steps of the frozen mesh give the oracle's state and dtnew"""
    from test_gpu_mhd import _mhd_amr_gpu_vs_oracle
    kw = dict(gamma=M1["gamma"], courant_factor=M1["courant_factor"])
    if ndim == 1:
        from oracle.amr_mhd import MhdAmrRun
        from test_oracle_golden import IMHD
        r = MhdAmrRun(5, 9, (2, 2, 0, 0, 0, 0), 3.5, nsubcycle=[1, 1, 1, 1], riemann="hlld", slope_type=2, err_grad_d=0.01,
                      err_grad_u=0.05, err_grad_p=0.05, interpol_type=2, regions=IMHD, tout=[1e9], ngridmax=10000, **kw)
        r.run(max_coarse=6)
        _mhd_amr_gpu_vs_oracle(r, 1, "hlld", "llf", 2, 3, resident)
    elif ndim == 2:
        from oracle.amr_mhd import MhdAmrRun2D
        r = MhdAmrRun2D(4, 6, 1.0, nsubcycle=[1, 2], riemann="roe", riemann2d="llf", slope_type=1, err_grad_p=0.1, interpol_type=2,
                        tout=[1e9], nexpand=1, ngridmax=20000, **kw)
        r.run(max_coarse=6)
        _mhd_amr_gpu_vs_oracle(r, 2, "roe", "llf", 1, 3, resident)
    else:
        from test_device_numerics_host import _mhd3_static_run
        r = _mhd3_static_run("hlld", "hlld", 2)
        r.pm.gamma, r.pm.courant_factor = kw["gamma"], kw["courant_factor"]
        _mhd_amr_gpu_vs_oracle(r, 3, "hlld", "hlld", 2, 3, resident, regrid=False)
    from oracle import orc
    _assert_each_parameter_matters(lambda q: mhd_amr_oracle(orc, r, q), M1, MSUITE, ("gamma", "courant_factor"))


def test_passive_scalar_amr_at_h1(gpu):
    """one passive scalar (nvar 6) in AMR mode at H1 -- gamma 5/3, courant_factor 0.5, slope_type 8 with slope_theta 1.2,
    niter_riemann 2, `exact` -- on the 3-level nested tree of the scalar tests, boxlen 0.75: one coarse step driven by the host
    mirror of amr_step equals the oracle's amr_step (1e-12, CUDA pow); the scalar moved, and every parameter reaches the oracle's
    result"""
    from oracle.amr import AmrRun
    from test_gpu_passive_scalars import _assert_close, _nested_gpu, _nested_scalar_case
    levelmin, levelmax, nvar = 4, 6, 6

    def setup(a, q):
        a.gamma, a.courant_factor, a.slope_type, a.riemann = q["gamma"], q["courant_factor"], 8, "exact"
        a.slope_theta, a.niter_riemann, a.boxlen = q["slope_theta"], q["niter_riemann"], q["scale"]
        return a

    def oracle(q, u0, a):
        r = AmrRun(3, levelmin, levelmax, (0,) * 6, q["scale"], nsubcycle=[1, 2, 2], ngridmax=a.ngridmax, riemann="exact", slope_type=8,
                   gamma=q["gamma"], courant_factor=q["courant_factor"], interpol_type=1, interpol_var=0, tout=[1e9], nvar=nvar)
        r.p.slope_theta, r.p.niter_riemann = q["slope_theta"], q["niter_riemann"]
        r.uold[:] = u0.ravel()
        r.son[1:] = a.son; r.father[1:] = a.father; r.nbor[:, 1:] = a.nbor
        for l in range(1, levelmax + 1):
            r.active[l] = [int(g) for g in a.active[l]]
        r.push_all()
        r.static = True
        r.amr_step(levelmin, 1)
        return r.uold.reshape(nvar, -1).copy(), np.array([r.dtnew[levelmin]])

    a = setup(_nested_scalar_case(nvar, levelmin, levelmax), H1)
    u0, dts = _nested_gpu(a, levelmin, levelmax, 1, 0)
    ref, dt_ref = oracle(H1, u0, a)
    assert abs(dts[0] / dt_ref[0] - 1) <= 1e-12
    cells = np.concatenate([[a.ncoarse + ind * a.ngridmax + int(g) - 1 for g in a.active[l] for ind in range(8)] for l in range(1, levelmax + 1)])
    _assert_close(a.uold[:, cells], ref[:, cells], True)
    assert np.abs(a.uold[5:, cells] - u0[5:, cells]).max() > 1e-4
    _assert_each_parameter_matters(lambda q: oracle(q, u0, a), H1, SUITE)
