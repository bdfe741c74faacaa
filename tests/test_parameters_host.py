"""The device numerics away from the suite's one namelist point, emulated on the CPU and compared with the oracle bit for bit:
gamma, courant_factor, slope_theta, niter_riemann, the box scale boxlen / nx, beta_fix and the refinement thresholds and floors.

Every other CPU test runs hydro at gamma 1.4, courant_factor 0.8, slope_theta 1.5 (1.3 in places), niter_riemann 10, a box
scale of 1 and beta_fix 0.5, and MHD at gamma 5/3.  A kernel that hard-coded any of these values, or used the bare level factor
0.5^l where the reference uses dx = 0.5^l * boxlen / nx, would pass all of them.  The parameter sets below move every value
away from those points and from each other, so that a swapped pair changes the bits too, and each test family asserts on the
oracle that setting any one parameter back to the suite's value changes the compared result: the states of a test do reach
every parameter (the exact solver's Newton iteration, for one, is still unconverged at the niter_riemann cap).

The oracle's own gamma dependence is pinned by an independent exact Riemann solution in numpy / scipy (the golden files of
the reference hold one gamma each)."""
import ctypes as C

import numpy as np
import pytest
from scipy import optimize

from helpers import FLOORS, Case, MhdCase, box_state, level_slots, mhd_box_state
from test_device_numerics_host import (IP3, MHD_R1D, MHD_R2D, SOLVER_ID, _amr_source_terms_compare, _hydro_states,  # noqa: F401
                                       _mhd3_static_run, _mhd_amr_compare_levels, dev)
from test_passive_scalars_host import scl, sedov_runs  # noqa: F401  (fixtures)

DP = C.POINTER(C.c_double)
IP = C.POINTER(C.c_int)

# the suite's values, and two hydro sets away from them; scale = boxlen / nx (the size of a coarse cell)
SUITE = dict(gamma=1.4, courant_factor=0.8, slope_theta=1.5, niter_riemann=10, scale=1.0)
H1 = dict(gamma=5.0 / 3.0, courant_factor=0.5, slope_theta=1.2, niter_riemann=2, scale=0.75)
H2 = dict(gamma=1.2, courant_factor=0.35, slope_theta=1.9, niter_riemann=1, scale=3.0)
HSETS = {"H1": H1, "H2": H2}
# MHD: the suite runs gamma 5/3; slope_theta is read by slope_type 8 of the dense six-pass sweep only
MSUITE = dict(gamma=5.0 / 3.0, courant_factor=0.8, slope_theta=1.5, scale=1.0)
M1 = dict(gamma=1.4, courant_factor=0.5, slope_theta=1.2, scale=0.75)
BETA_FIX = (0.0, 0.5, 4.0)
# refinement thresholds (err_grad_d, err_grad_u, err_grad_p); -1 switches a criterion off
THRESHOLDS = {"distinct": (0.03, 0.2, 0.08), "d": (0.03, -1.0, -1.0), "u": (-1.0, 0.2, -1.0), "p": (-1.0, -1.0, 0.08),
              "none": (-1.0, -1.0, -1.0)}


def _differs(a, b):
    return any(not np.array_equal(x, y) for x, y in zip(a, b))


def _assert_each_parameter_matters(run, pset, suite, keys=None):
    """run(params) -> tuple of oracle arrays; with any one parameter of pset set back to the suite's value the result changes"""
    base = run(pset)
    for k in keys or pset:
        if pset[k] != suite[k]:
            assert _differs(base, run(dict(pset, **{k: suite[k]}))), f"{k} does not reach the compared result"
    return base


# ---- Riemann solvers ---------------------------------------------------------------------------------------------------------
def _oracle_riemann(orc, ndim, solver, ql, qr, gamma, smallr, smallc, niter):
    L = orc.lib()
    f = {"llf": L.orc_riemann_llf, "exact": L.orc_riemann_approx, "acoustic": L.orc_riemann_acoustic, "hllc": L.orc_riemann_hllc,
         "hll": L.orc_riemann_hll}[solver]
    f.argtypes = [C.POINTER(orc.Params), DP, DP, DP, C.c_int]
    n, nv = ql.shape
    p = orc.make_params(ndim=ndim, riemann=solver, nvector=n, niter_riemann=niter, gamma=gamma, smallr=smallr, smallc=smallc)
    qlf, qrf = np.asfortranarray(ql), np.asfortranarray(qr)
    fgf = np.zeros((n, nv + 1), order="F")
    f(C.byref(p), qlf.ctypes.data_as(DP), qrf.ctypes.data_as(DP), fgf.ctypes.data_as(DP), n)
    return fgf[:, :nv].copy(), fgf[:, nv].copy()


def _niters(solver, pset):
    return (1, 2, 3) if solver == "exact" else (pset["niter_riemann"],)


@pytest.mark.parametrize("pset", ["H1", "H2"])
@pytest.mark.parametrize("solver", ["llf", "exact", "acoustic", "hllc", "hll"])
def test_riemann_at_parameter_sets(orc, dev, solver, pset):
    """riemann_* of hydro_device.cuh and the internal-energy flux at gamma 5/3 and 1.2, `exact` at niter_riemann 1, 2 and 3:
    equal the oracle's bit for bit on 20 000 face states per dimension (strong shocks and rarefactions among them, so that
    the two-shock Newton iteration is cut by the cap)"""
    ps = HSETS[pset]
    sid = SOLVER_ID[solver]
    dev.devnum_riemann_eflux.argtypes = [C.c_int, C.c_int, C.c_int, DP, DP, DP, C.c_double, C.c_double, C.c_double, C.c_int]
    for ndim in (1, 2, 3):
        n, nv = 20000, ndim + 2
        ql, qr = _hydro_states(np.random.default_rng(300 + ndim * 10 + sid), n, ndim)
        for smallr, smallc in FLOORS.values():
            for niter in _niters(solver, ps):
                fg, fe = np.zeros((n, nv)), np.zeros(n)
                dev.devnum_riemann(ndim, sid, n, orc.dptr(ql), orc.dptr(qr), orc.dptr(fg), ps["gamma"], smallr, smallc, niter)
                dev.devnum_riemann_eflux(ndim, sid, n, orc.dptr(ql), orc.dptr(qr), orc.dptr(fe), ps["gamma"], smallr, smallc, niter)
                ref, ref_e = _oracle_riemann(orc, ndim, solver, ql, qr, ps["gamma"], smallr, smallc, niter)
                assert np.isfinite(fg).all()
                assert np.array_equal(fg, ref), (ndim, niter)
                assert np.array_equal(fe, ref_e), (ndim, niter)
                # the oracle: gamma and (exact) the cap reach the fluxes of these states
                other = _oracle_riemann(orc, ndim, solver, ql, qr, SUITE["gamma"], smallr, smallc, niter)
                assert _differs((ref, ref_e), other)
                if solver == "exact":
                    assert _differs((ref, ref_e), _oracle_riemann(orc, ndim, solver, ql, qr, ps["gamma"], smallr, smallc, 10)), niter


@pytest.mark.parametrize("pset", ["H1", "H2"])
@pytest.mark.parametrize("niter", [1, 2])
def test_vec_solvers_at_low_niter(orc, dev, niter, pset):
    """the branch-free scalar and the 3-lane forms of `exact` (hydro_vec.cuh) with the iteration cut at 1 or 2 steps: each lane
    freezes on its own, and both forms equal the oracle bit for bit on 30 000 face states"""
    ps = HSETS[pset]
    dev.devnum_riemann_vec.argtypes = [C.c_int, C.c_int, DP, DP, DP, DP, C.c_double, C.c_double, C.c_double, C.c_int]
    n = 30000
    ql, qr = _hydro_states(np.random.default_rng(900 + niter), n, 3)
    ql[100:200, 1] = 50.0; qr[100:200, 1] = 50.0
    ql[200:300, 1] = -50.0; qr[200:300, 1] = -50.0
    for smallr, smallc in FLOORS.values():
        f1, f3 = np.zeros((n, 5)), np.zeros((n, 5))
        dev.devnum_riemann_vec(1, n, orc.dptr(ql), orc.dptr(qr), orc.dptr(f1), orc.dptr(f3), ps["gamma"], smallr, smallc, niter)
        ref, _ = _oracle_riemann(orc, 3, "exact", ql, qr, ps["gamma"], smallr, smallc, niter)
        assert np.array_equal(f1, ref)
        assert np.array_equal(f3, ref)
        converged, _ = _oracle_riemann(orc, 3, "exact", ql, qr, ps["gamma"], smallr, smallc, 10)
        # lanes of one triple stop at different iterations: some rows differ from the converged flux, others do not
        same = (ref == converged).all(axis=1)
        assert 0 < same.sum() < n


# ---- cmpdt -------------------------------------------------------------------------------------------------------------------
def _cmpdt_cells(rng, n, ndim):
    u = np.zeros((n, ndim + 2))
    u[:, 0] = 10.0 ** rng.uniform(-3, 2, n)
    vel = rng.standard_normal((n, ndim)) * 3
    u[:, 1:1 + ndim] = u[:, :1] * vel
    u[:, ndim + 1] = 10.0 ** rng.uniform(-4, 2, n) + 0.5 * u[:, 0] * (vel ** 2).sum(axis=1)
    return np.ascontiguousarray(u)


def _oracle_cmpdt(orc, u, g, dx, ndim, gamma, cfl, smallr, smallc):
    L = orc.lib()
    L.orc_cmpdt.argtypes = [C.POINTER(orc.Params), DP, DP, C.c_double, DP, C.c_int]
    p = orc.make_params(ndim=ndim, nvector=1, gamma=gamma, courant_factor=cfl, smallr=smallr, smallc=smallc)
    ref = np.zeros(len(u))
    for i in range(len(u)):
        uu = u[i].copy()
        gg = None
        if g is not None:
            gg = np.zeros(3)
            gg[:ndim] = g[i]
        o = C.c_double(0.0)
        L.orc_cmpdt(C.byref(p), orc.dptr(uu), None if gg is None else orc.dptr(gg), dx, C.byref(o), 1)
        ref[i] = o.value
    return ref


@pytest.mark.parametrize("pset", ["H1", "H2"])
@pytest.mark.parametrize("ndim", [1, 2, 3])
def test_cmpdt_at_parameter_sets(orc, dev, ndim, pset):
    """cmpdt_cell with and without the gravity term at the set's gamma, courant_factor and a cell size of scale / 128: equal
    orc_cmpdt bit for bit"""
    ps = HSETS[pset]
    rng = np.random.default_rng(70 + ndim)
    n = 3000
    u = _cmpdt_cells(rng, n, ndim)
    g = rng.standard_normal((n, ndim)) * 10.0 ** rng.uniform(-3, 5, (n, 1))
    gsum = np.zeros(n)
    for d in range(ndim):
        gsum = gsum + np.abs(g[:, d])
    dx = ps["scale"] / 128
    for smallr, smallc in FLOORS.values():
        dt, dtg = np.zeros(n), np.zeros(n)
        dev.devnum_cmpdt(ndim, n, orc.dptr(u), dx, orc.dptr(dt), ps["gamma"], smallr, smallc, ps["courant_factor"])
        dev.devnum_cmpdt_grav(ndim, n, orc.dptr(u), orc.dptr(gsum), dx, orc.dptr(dtg), ps["gamma"], smallr, smallc,
                              ps["courant_factor"])

        def run(q):
            return (_oracle_cmpdt(orc, u, None, dx, ndim, q["gamma"], q["courant_factor"], smallr, smallc),
                    _oracle_cmpdt(orc, u, g, dx, ndim, q["gamma"], q["courant_factor"], smallr, smallc))
        ref, refg = _assert_each_parameter_matters(run, ps, SUITE, ("gamma", "courant_factor"))
        assert np.array_equal(dt, ref)
        assert np.array_equal(dtg, refg)


# ---- dense sweeps ------------------------------------------------------------------------------------------------------------
def _param_case(ndim, level, coarse, bound, solver, st, ps, seed=2):
    """oracle set-up on `coarse` domain coarse cells of size ps['scale'] (dx = scale 2^-level) with a box_state at the set's gamma
    and a strong blast in it (pressure ratio 100: the exact solver's iteration is unconverged at a small cap)"""
    c = Case(ndim, level, riemann=solver, slope_type=st, bound=bound, coarse=coarse, boxlen=ps["scale"] * coarse[0], order=1, seed=seed,
             gamma=ps["gamma"], courant_factor=ps["courant_factor"], slope_theta=ps["slope_theta"], niter_riemann=ps["niter_riemann"])
    ext = c.mesh.extent(level)
    d = box_state(ndim, ext, gamma=ps["gamma"])
    blast = np.zeros(d[0].shape, dtype=bool)
    blast[tuple(slice(s // 3, s // 3 + max(1, s // 8)) for s in d[0].shape)] = True
    d[ndim + 1][blast] += 100.0 / (ps["gamma"] - 1)
    c.init_dense(d)
    return c, ext


def _oracle_level_step(c):
    """dt of the state, the new state and the next dt with the mass / energy sums (the fused Courant partials)"""
    dt, _ = c.oracle_courant()
    dt *= 0.8
    unew = c.oracle_godunov(dt, nthreads=4)
    dt_next, sums = c.oracle_courant(unew)
    return dt, unew, dt_next, sums


def _dense_run(ndim, level, coarse, bound, solver, st):
    def run(q):
        c, _ = _param_case(ndim, level, coarse, bound, solver, st, q)
        dt, unew, dt_next, sums = _oracle_level_step(c)
        return np.array([dt, dt_next]), unew
    return run


def _check_level(c, uout, act, slot, unew, part, nb, dt_next, sums, dx):
    s = c.mesh.s
    T, nv = 1 << c.ndim, c.nvar
    U = unew.reshape(nv, s.ncell)
    for ind in range(T):
        cells = s.ncoarse + ind * s.ngridmax + act - 1
        assert np.array_equal(uout[:, ind, slot], U[:, cells]), (ind, float(np.abs(uout[:, ind, slot] - U[:, cells]).max()))
    p4 = part[:4 * nb].reshape(4, nb)
    assert min(p4[0].min(), c.p.boxlen / c.p.smallc) == dt_next
    vol = dx ** c.ndim
    assert abs(p4[1].sum() * vol - sums[0]) <= 1e-13 * abs(sums[0])


DENSE_CASES = [(1, (4, 1, 1), 5, (1, 1, 0, 0, 0, 0), "exact", 3), (1, (4, 1, 1), 5, (2, 2, 0, 0, 0, 0), "hllc", 2),
               (2, (2, 1, 1), 4, (0, 0, 1, 1, 0, 0), "exact", 3), (2, (1, 2, 1), 4, (2, 2, 0, 0, 0, 0), "llf", 2),
               (3, (2, 1, 1), 3, (0,) * 6, "exact", 3), (3, (1, 1, 2), 3, (0,) * 6, "acoustic", 2)]


@pytest.mark.parametrize("pset", ["H1", "H2"])
@pytest.mark.parametrize("ndim,coarse,level,bound,solver,nblocks", DENSE_CASES)
def test_dense_sweep_at_parameter_sets(orc, dev, pset, ndim, coarse, level, bound, solver, nblocks):
    """sweep_dense_kernel in 1-D, 2-D and 3-D, slope_type 8, with walls, outflow and periodic axes, at the set's parameters:
    the new state equals the oracle's level step bit for bit and the fused Courant partials give its next dt"""
    ps = HSETS[pset]
    c, ext = _param_case(ndim, level, coarse, bound, solver, 8, ps)
    dt, unew, dt_next, sums = _oracle_level_step(c)
    shell = [int(bound[2 * d] > 0) for d in range(3)]
    uin, act, slot = level_slots(c.mesh, level, c.u, ndim + 2)
    uout = np.zeros_like(uin)
    part = np.zeros(4 * 64)
    dx = ps["scale"] * 2.0 ** -level
    nb = dev.devnum_sweep_dense_box(ndim, SOLVER_ID[solver], IP3(*ext), IP3(*shell), nblocks, orc.dptr(uin), orc.dptr(uout), dt, dx, 8,
                                    ps["slope_theta"], ps["courant_factor"], ps["gamma"], 1e-10, 1e-10, ps["niter_riemann"],
                                    orc.dptr(part), 0)
    _check_level(c, uout, act, slot, unew, part, nb, dt_next, sums, dx)


@pytest.mark.parametrize("pset", ["H1", "H2"])
@pytest.mark.parametrize("ndim", [1, 2, 3])
def test_dense_sweep_parameters_are_not_vacuous(orc, pset, ndim):
    """on the exact-solver cases of the dense sweep tests, each parameter of the set, set back to the suite's value alone,
    changes the oracle's new state or time steps"""
    case = next(k for k in DENSE_CASES if k[0] == ndim and k[4] == "exact")
    _assert_each_parameter_matters(_dense_run(ndim, case[2], case[1], case[3], "exact", 8), HSETS[pset], SUITE)


@pytest.mark.parametrize("pset", ["H1", "H2"])
@pytest.mark.parametrize("solver,nblocks,by,vec", [("exact", 3, 12, 1), ("hllc", 2, 8, 0), ("exact", 2, 16, 2), ("llf", 3, 12, 12),
                                                   ("exact", 4, 12, 41), ("hll", 3, 12, 40), ("exact", 2, 8, 42)])
def test_sweep3_kernel_at_parameter_sets(orc, dev, pset, solver, nblocks, by, vec):
    """sweep3_kernel / sweep4_kernel (tile heights 8/12/16, solver forms 0/1/2/12 and the one-barrier orders 40-42) on a
    32x16x16 periodic box, slope_type 8, at the set's parameters: state and Courant partials equal the oracle's"""
    ps = HSETS[pset]
    c, ext = _param_case(3, 4, (2, 1, 1), (0,) * 6, solver, 8, ps)
    dt, unew, dt_next, sums = _oracle_level_step(c)
    uin, act, slot = level_slots(c.mesh, c.level, c.u, 5)
    uout = np.zeros_like(uin)
    part = np.zeros(4 * 64)
    nb = dev.devnum_sweep3_box(SOLVER_ID[solver], IP3(*ext), IP3(0, 0, 0), nblocks, orc.dptr(uin), orc.dptr(uout), dt,
                               ps["scale"] * 2.0 ** -c.level, 8, ps["slope_theta"], ps["courant_factor"], ps["gamma"], 1e-10, 1e-10,
                               ps["niter_riemann"], orc.dptr(part), by, vec)
    _check_level(c, uout, act, slot, unew, part, nb, dt_next, sums, ps["scale"] * 2.0 ** -c.level)


# ---- AMR mode: the dense AMR variant, the oct-batch kernel, the source terms, hydro_flag ----------------------------------------
_RUNS = {}


def _scaled(regions, scale):
    """condinit regions placed in a box of size `scale` the way they sit in the unit box"""
    keys = ("x_center", "y_center", "z_center", "length_x", "length_y", "length_z")
    return [{k: (v * scale if k in keys else v) for k, v in reg.items()} for reg in regions]


def _amr_run(ndim, ps, solver, st=8, **kw):
    """an adaptively refined mesh developed by the oracle's driver at the set's gamma and scale (boxlen = scale, one coarse cell),
    slope_theta and niter_riemann in force; cached per arguments (tests copy what they change).  The oracle's prolongation
    setting is global: it is set back to this run's (type 2 below 3-D, 1 in 3-D) whenever the run is handed out."""
    from oracle import orc
    from oracle.amr import FastAmrRun
    key = (ndim, tuple(sorted(ps.items())), solver, st, tuple(sorted(kw.items())))
    if key in _RUNS:
        orc.lib().orc_set_interpol(2 if ndim < 3 else 1, 0)
        return _RUNS[key]
    g, sc = ps["gamma"], ps["scale"]
    if ndim == 1:
        reg = [dict(type="square", x_center=0.25, length_x=0.5, d=1.0, p=10.0), dict(type="square", x_center=0.75, length_x=0.5, d=0.125, p=1e-4)]
        r = FastAmrRun(1, 3, 8, (1, 1, 0, 0, 0, 0), ps["scale"], nsubcycle=[1, 2], ngridmax=500, riemann=solver, slope_type=st, gamma=g,
                       courant_factor=ps["courant_factor"], err_grad_d=0.05, err_grad_p=0.05, interpol_type=2, regions=_scaled(reg, sc),
                       tout=[1e9], **kw)
    elif ndim == 2:
        reg = [dict(type="square", x_center=0.5, y_center=0.5, length_x=10, length_y=10, exp_region=10, d=1.0, p=1e-3),
               dict(type="square", x_center=0.3, y_center=0.4, length_x=0.3, length_y=0.25, exp_region=2, d=2.0, u=0.3, v=-0.2, p=10.0)]
        from test_gpu_amr import BOUND_2D_WALLS_X_OUTFLOW_Y
        r = FastAmrRun(2, 3, 5, (1, 1, 2, 2, 0, 0), ps["scale"], nsubcycle=[1, 2], ngridmax=20000, riemann=solver, slope_type=st,
                       gamma=g, courant_factor=ps["courant_factor"], err_grad_d=0.05, err_grad_u=0.05, err_grad_p=0.05, interpol_type=2,
                       regions=_scaled(reg, sc), tout=[1e9], bound_regions=BOUND_2D_WALLS_X_OUTFLOW_Y, **kw)
    else:
        reg = [dict(type="square", x_center=0.5, y_center=0.5, z_center=0.5, length_x=10, length_y=10, length_z=10, exp_region=10, d=1.0,
                    p=1e-3),
               dict(type="point", x_center=0.5, y_center=0.5, z_center=0.5, p=0.4)]
        r = FastAmrRun(3, 3, 5, (0,) * 6, ps["scale"], nsubcycle=[1, 2], ngridmax=4000, riemann=solver, slope_type=st, gamma=g,
                       courant_factor=ps["courant_factor"], err_grad_p=0.1, interpol_type=1, regions=_scaled(reg, sc), tout=[1e9], **kw)
    r.p.slope_theta, r.p.niter_riemann = ps["slope_theta"], ps["niter_riemann"]
    r.run(max_coarse=3)
    _RUNS[key] = r
    return r


def _level_dt(r, l):
    return 0.4 * r.dtnew[r.levelmin] / 2 ** (l - r.levelmin)


def _oct_batch_oracle(orc, r, l, q, dt):
    """set_unew + godunov_fine of level l with the parameters q in force (the mesh and state of r)"""
    L = orc.lib()
    p = orc.make_params(ndim=r.ndim, riemann=r.p.riemann, slope_type=r.p.slope_type, gamma=q["gamma"], courant_factor=q["courant_factor"],
                        boxlen=q["scale"], nvector=r.p.nvector,
                        slope_theta=q["slope_theta"], niter_riemann=q["niter_riemann"])
    unew = np.zeros_like(r.uold)
    L.orc_set_unew(C.byref(p), r.mp, l, orc.dptr(r.uold), orc.dptr(unew))
    L.orc_godunov_fine(C.byref(p), r.mp, l, dt, orc.dptr(r.uold), orc.dptr(unew), 1)
    return unew


OCT_CASES = [("H1", 1, s) for s in ("llf", "exact", "acoustic", "hllc", "hll")] + \
    [(ps, 2, "exact") for ps in ("H1", "H2")] + [("H2", 2, "hllc"), ("H1", 3, "exact"), ("H2", 3, "exact"), ("H2", 3, "llf")]


@pytest.mark.parametrize("pset,ndim,solver", OCT_CASES)
def test_oct_batch_kernel_at_parameter_sets(orc, dev, pset, ndim, solver):
    """amr_godfine_kernel, slope_type 8, on adaptively refined meshes at the set's gamma, slope_theta, niter_riemann and box
    scale (dx = scale 2^-l): the update of every level equals godfine1 of the oracle bit for bit; the exact-solver cases also
    show that every parameter reaches the oracle's update"""
    ps = HSETS[pset]
    r = _amr_run(ndim, ps, solver)
    m = r.m
    T, nvar = 1 << ndim, ndim + 2
    son = np.ascontiguousarray(r.son[1:], dtype=np.int32)
    father = np.ascontiguousarray(r.father[1:], dtype=np.int32)
    nbor = np.ascontiguousarray(r.nbor[:, 1:], dtype=np.int32)
    itype = 2 if ndim < 3 else 1
    nlev = 0
    for l in range(r.levelmin, r.nlevelmax + 1):
        act = np.ascontiguousarray(r.active[l], dtype=np.int32)
        if len(act) == 0:
            continue
        dt = _level_dt(r, l)
        dx = 0.5 ** l * r.p.boxlen / (m.icoarse_max - m.icoarse_min + 1)
        assert dx == ps["scale"] * 0.5 ** l
        unew_o = _oct_batch_oracle(orc, r, l, ps, dt)
        unew_k = np.zeros_like(r.uold)
        orc.lib().orc_set_unew(C.byref(r.p), r.mp, l, orc.dptr(r.uold), orc.dptr(unew_k))
        rflux = np.zeros(len(act) * 2 * ndim * (T // 2) * nvar)
        dev.devnum_amr_godfine(ndim, SOLVER_ID[solver], r.ncoarse, r.ngridmax, m.nx, m.ny, m.nz, orc.iptr(son), orc.iptr(father),
                               orc.iptr(nbor), orc.iptr(act), len(act), l, orc.dptr(r.uold), orc.dptr(unew_k), orc.dptr(rflux), dt, dx,
                               itype, 8, ps["slope_theta"], ps["gamma"], r.p.smallr, r.p.smallc, ps["niter_riemann"], 0.0)
        assert np.isfinite(unew_o).all()
        Uo, Uk = unew_o.reshape(nvar, r.ncell), unew_k.reshape(nvar, r.ncell)
        for ind in range(T):
            c = r.ncoarse + ind * r.ngridmax + act.astype(np.int64) - 1
            assert np.array_equal(Uk[:, c], Uo[:, c]), (l, ind)
        nlev += 1
    assert nlev >= 2
    if solver == "exact":
        levels = [l for l in range(r.levelmin, r.nlevelmax + 1) if len(r.active[l])]
        _assert_each_parameter_matters(lambda q: tuple(_oct_batch_oracle(orc, r, l, q, _level_dt(r, l)) for l in levels), ps, SUITE,
                                       ("gamma", "slope_theta", "niter_riemann", "scale"))


def _src_oracle(orc, r, l, q, beta_fix, force):
    """set_unew -> godunov_fine -> set_uold of level l with poisson and pressure_fix on, boxlen = q['scale'] and beta_fix"""
    L = orc.lib()
    L.orc_set_pressure_fix.argtypes = [DP, DP, C.c_double]
    L.orc_set_gravity.argtypes = [DP]
    p = orc.make_params(ndim=r.ndim, riemann=r.p.riemann, slope_type=r.p.slope_type, gamma=r.p.gamma, boxlen=q["scale"],
                        nvector=r.p.nvector, slope_theta=r.p.slope_theta, niter_riemann=r.p.niter_riemann)
    u, unew = r.uold.copy(), np.zeros_like(r.uold)
    divu, enew = np.zeros(r.ncell), np.zeros(r.ncell)
    try:
        L.orc_set_pressure_fix(orc.dptr(divu), orc.dptr(enew), beta_fix)
        L.orc_set_gravity(orc.dptr(force))
        L.orc_set_unew(C.byref(p), r.mp, l, orc.dptr(u), orc.dptr(unew))
        L.orc_godunov_fine(C.byref(p), r.mp, l, _level_dt(r, l), orc.dptr(u), orc.dptr(unew), 1)
        L.orc_set_uold(C.byref(p), r.mp, l, orc.dptr(u), orc.dptr(unew))
    finally:
        L.orc_set_pressure_fix(None, None, 0.0)
        L.orc_set_gravity(None)
    return u, divu, enew


@pytest.mark.parametrize("beta_fix", BETA_FIX)
@pytest.mark.parametrize("pset,ndim,solver", [("H1", 1, "exact"), ("H2", 1, "hllc"), ("H2", 2, "hllc"), ("H1", 2, "exact"), ("H1", 3, "hllc")])
def test_amr_source_terms_at_parameter_sets(orc, dev, pset, ndim, solver, beta_fix):
    """poisson and pressure_fix on refined meshes of box scale 0.75 and 3 at beta_fix 0, 0.5 and 4: the SRC oct-batch kernel,
    add_pdv_source_terms (dx_loc = scale 0.5^l, 1.5 dx_loc next to a coarser neighbour) and the energy switch of set_uold
    (beta_fix (|div u| dx)^2) equal the oracle's state, divu and enew bit for bit.  At beta_fix 4 the switch fires in many
    cells but not in all; the scale and beta_fix reach the oracle's result."""
    ps = HSETS[pset]
    r = _amr_run(ndim, ps, solver)
    switched, ncmp = _amr_source_terms_compare(orc, dev, ndim, solver, True, True, run=r, beta_fix=beta_fix)
    if beta_fix == 4.0:
        assert 0.005 * ncmp < switched < 0.9 * ncmp, (switched, ncmp)
    rng = np.random.default_rng(3)
    force = np.ascontiguousarray(rng.standard_normal((ndim, r.ncell)) * 5.0)
    levels = [l for l in range(r.levelmin, r.nlevelmax + 1) if len(r.active[l])]

    def run(q, b):
        return sum((_src_oracle(orc, r, l, q, b, force) for l in levels), ())
    base = run(ps, beta_fix)
    assert _differs(base, run(SUITE, beta_fix))
    if beta_fix != 0.5:
        assert _differs(base, run(ps, 0.5))


@pytest.mark.parametrize("pset", ["H1", "H2"])
@pytest.mark.parametrize("solver", ["exact", "hllc"])
def test_dense_sweep_amr_variant_at_parameter_sets(orc, dev, pset, solver):
    """sweep_dense_kernel<..., AMRV=true> on the fully refined base level of a refined 3-D mesh of box scale 0.75 / 3, slope_type 8,
    at the set's gamma, slope_theta and niter_riemann: the update accumulated into unew equals godfine1 of the oracle"""
    from oracle.amr import FastAmrRun
    ps = HSETS[pset]
    # a cold advected background with nested density steps 1 / 2 / 4 and pressure steps of 7 % (below err_grad_p: their cells stay
    # leaf cells of level 4, where slope_theta and the Newton iteration act) and a blast refined to level 5
    box = dict(type="square", x_center=0.3, y_center=0.3, z_center=0.7, exp_region=10, p=1e-3, u=0.3, v=0.2, w=-0.1)
    reg = [dict(box, x_center=0.5, y_center=0.5, z_center=0.5, length_x=10, length_y=10, length_z=10, d=1.0),
           dict(box, length_x=0.3, length_y=0.3, length_z=0.3, d=2.0, p=1.07e-3),
           dict(box, length_x=0.18, length_y=0.18, length_z=0.18, d=4.0, p=1.14e-3),
           dict(type="point", x_center=0.6, y_center=0.55, z_center=0.4, p=0.4)]
    key = ("amrv", pset, solver)
    if key not in _RUNS:
        r = FastAmrRun(3, 4, 5, (0,) * 6, ps["scale"], nsubcycle=[1, 2], ngridmax=6000, riemann=solver, slope_type=8, gamma=ps["gamma"],
                       courant_factor=ps["courant_factor"], err_grad_p=0.1, interpol_type=1, regions=_scaled(reg, ps["scale"]), tout=[1e9])
        r.p.slope_theta, r.p.niter_riemann = ps["slope_theta"], ps["niter_riemann"]
        r.run(max_coarse=2)
        _RUNS[key] = r
    r = _RUNS[key]
    orc.lib().orc_set_interpol(1, 0)
    l, N = 4, 16
    act = np.asarray(r.active[l], dtype=np.int64)
    assert len(act) == 8 ** 3 and len(r.active[5]) > 0
    dt = 0.5 * r.dtnew[l]
    ref_u = _oct_batch_oracle(orc, r, l, ps, dt)
    if solver == "exact":         # the leaf cells of level 4 hold no pressure ratio large enough to leave the iteration unconverged
        _assert_each_parameter_matters(lambda q: (_oct_batch_oracle(orc, r, l, q, dt),), ps, SUITE, ("gamma", "slope_theta", "scale"))
    start = np.zeros_like(r.uold)
    orc.lib().orc_set_unew(C.byref(r.p), r.mp, l, orc.dptr(r.uold), orc.dptr(start))
    pos = np.rint(r.xg[:, act] * 2 ** (l - 1) - 0.5).astype(np.int64)
    assert len(set(map(tuple, pos.T))) == len(act)
    h = N // 2
    slot = pos[0] + h * (pos[1] + h * pos[2])
    Uold, Ust, Uref = r.uold.reshape(5, r.ncell), start.reshape(5, r.ncell), ref_u.reshape(5, r.ncell)
    uin, uout, ref = np.zeros((5, 8, h ** 3)), np.zeros((5, 8, h ** 3)), np.zeros((5, 8, h ** 3))
    refined = np.zeros((8, h ** 3), dtype=np.uint8)
    for ind in range(8):
        c = r.ncoarse + ind * r.ngridmax + act - 1
        uin[:, ind, slot], uout[:, ind, slot], ref[:, ind, slot] = Uold[:, c], Ust[:, c], Uref[:, c]
        refined[ind, slot] = r.son[c + 1] > 0
    assert refined.sum() > 0
    dev.devnum_sweep_dense_amr.argtypes = [C.c_int, C.c_int, C.c_int, DP, DP, C.POINTER(C.c_ubyte), C.c_double, C.c_double, C.c_int,
                                           C.c_double, C.c_double, C.c_double, C.c_double, C.c_int]
    dev.devnum_sweep_dense_amr(SOLVER_ID[solver], N, 4, orc.dptr(np.ascontiguousarray(uin)), orc.dptr(uout),
                               refined.ctypes.data_as(C.POINTER(C.c_ubyte)), dt, ps["scale"] / N, 8, ps["slope_theta"], ps["gamma"],
                               1e-10, 1e-10, ps["niter_riemann"])
    assert np.abs(ref - uin).max() > 1e-5
    assert np.array_equal(uout, ref)


@pytest.mark.parametrize("solver", ["hllc", "exact"])
def test_oct_batch_kernel_with_scalars_at_h1(orc, scl, sedov_runs, solver):
    """amr_godfine_kernel with one passive scalar (NPS = 1, the instantiation launch_amr_godfine picks for nvar 6) at H1: gamma 5/3,
    slope_type 8 with slope_theta 1.2, niter_riemann 2 and box scale 0.75 (dx = 0.75 2^-l) on the 3-D refined mesh of the scalar
    tests: the update of every level, coarse refluxes included, equals the oracle's; for `exact` every parameter reaches it"""
    from test_passive_scalars_host import _godfine_compare, fill_scalars
    r = sedov_runs[6]
    uold = r.uold.copy()
    fill_scalars(r, 31)
    try:
        _godfine_compare(orc, scl, r, solver, 8, 1, 0, 6, params=H1)
        if solver == "exact":
            _assert_each_parameter_matters(lambda q: _godfine_compare(orc, scl, r, solver, 8, 1, 0, 6, params=q), H1, SUITE,
                                           ("gamma", "slope_theta", "niter_riemann", "scale"))
    finally:
        r.uold[:] = uold


# ---- hydro_flag ----------------------------------------------------------------------------------------------------------------
def _flags(orc, dev, r, err, flo, uold=None):
    """(device flags, oracle flags) of every level below the finest, for thresholds err and floors flo"""
    m = r.m
    T = 1 << r.ndim
    u = r.uold if uold is None else uold
    son = np.ascontiguousarray(r.son[1:], dtype=np.int32)
    father = np.ascontiguousarray(r.father[1:], dtype=np.int32)
    nbor = np.ascontiguousarray(r.nbor[:, 1:], dtype=np.int32)
    dev.devnum_amr_hydro_flag.argtypes = [C.c_int] * 6 + [IP, IP, IP, IP, C.c_int, C.c_int, DP, C.c_double, C.c_double, DP, DP, IP]
    saved = (r.err_grad_d, r.err_grad_u, r.err_grad_p, r.floor_d, r.floor_u, r.floor_p, r.uold.copy())
    r.err_grad_d, r.err_grad_u, r.err_grad_p = err
    r.floor_d, r.floor_u, r.floor_p = flo
    r.uold[:] = u
    got, ref = [], []
    try:
        for l in range(r.levelmin, r.nlevelmax):
            act = np.asarray(r.active[l], dtype=np.int32)
            if not len(act):
                continue
            g = np.zeros((len(act), T), dtype=np.int32)
            dev.devnum_amr_hydro_flag(r.ndim, r.ncoarse, r.ngridmax, m.nx, m.ny, m.nz, orc.iptr(son), orc.iptr(father), orc.iptr(nbor),
                                      orc.iptr(act), len(act), l, orc.dptr(r.uold), r.p.gamma, r.p.smallr, orc.dptr(np.array(err)),
                                      orc.dptr(np.array(flo)), orc.iptr(g))
            r.flag1[:] = 0
            r.hydro_flag(l)
            got.append(g)
            ref.append(np.array([[r.flag1[r.cell(ind, int(ig))] for ind in range(T)] for ig in act], dtype=np.int32))
    finally:
        r.err_grad_d, r.err_grad_u, r.err_grad_p, r.floor_d, r.floor_u, r.floor_p = saved[:6]
        r.uold[:] = saved[6]
    return np.concatenate([x.ravel() for x in got]), np.concatenate([x.ravel() for x in ref])


def _flag_state(r, seed, rho_scale=1.0, p_scale=1.0):
    """the run's state with per-cell noise in density (1 %), pressure (4 %) and velocity (0.05 c): relative gradients spread
    continuously across the thresholds; density and pressure are then scaled by rho_scale and p_scale"""
    nd, g = r.ndim, r.p.gamma
    U = r.uold.reshape(nd + 2, r.ncell).copy()
    rng = np.random.default_rng(seed)
    rho = np.maximum(U[0], 1e-10)
    v = U[1:1 + nd] / rho
    p = np.maximum((g - 1) * (U[nd + 1] - 0.5 * rho * (v ** 2).sum(axis=0)), 1e-10)
    c = np.sqrt(g * p / rho)
    rho = rho * np.exp(0.01 * rng.standard_normal(r.ncell)) * rho_scale
    p = p * np.exp(0.04 * rng.standard_normal(r.ncell)) * p_scale
    v = v + 0.05 * c * rng.standard_normal((nd, r.ncell))
    U[0] = rho
    U[1:1 + nd] = rho * v
    U[nd + 1] = p / (g - 1) + 0.5 * rho * (v ** 2).sum(axis=0)
    return U.ravel()


@pytest.mark.parametrize("ndim", [1, 2, 3])
def test_amr_hydro_flag_at_threshold_sets(orc, dev, ndim):
    """amr_hydro_flag_kernel at gamma 5/3 with distinct thresholds (d, u, p) = (0.03, 0.2, 0.08), each criterion alone with the
    other two at -1, and all three at -1 (the early return): equal the oracle's flags.  Setting any one threshold of the
    distinct set back to the suite's 0.05 changes the flags; each criterion alone flags cells, and a different set of them."""
    r = _amr_run(ndim, H1, "hllc", st=2)
    u = _flag_state(r, 90 + ndim)
    flo = (1e-10, 1e-10, 1e-10)
    refs = {}
    for name, err in THRESHOLDS.items():
        got, ref = _flags(orc, dev, r, err, flo, u)
        assert np.array_equal(got, ref), name
        refs[name] = ref
        if name == "none":
            assert ref.sum() == 0
        else:
            assert 0 < ref.sum() < ref.size, name
    for k in range(3):
        err = list(THRESHOLDS["distinct"])
        err[k] = 0.05
        assert not np.array_equal(_flags(orc, dev, r, tuple(err), flo, u)[1], refs["distinct"]), k


@pytest.mark.parametrize("ndim", [1, 2, 3])
def test_amr_hydro_flag_floors_decide(orc, dev, ndim):
    """amr_hydro_flag_kernel on a thin, cold state (density 1e-3 and pressure 1e-6 of the run's) with the criterion floors
    (floor_d, floor_u, floor_p) raised to the median density, 100 x sound speed and pressure of the tree's cells that hold gas, one
    criterion at a time with thresholds (0.015, 0.1, 0.05) near the state's noise: the
    flags equal the oracle's, and the raised floor of each criterion changes its flags against the 1e-10 floors"""
    r = _amr_run(ndim, H1, "hllc", st=2)
    u = _flag_state(r, 95 + ndim, 1e-3, 1e-6)
    U = u.reshape(ndim + 2, r.ncell)
    p = (r.p.gamma - 1) * (U[ndim + 1] - 0.5 * (U[1:1 + ndim] ** 2).sum(axis=0) / U[0])
    gas = U[0] > 1e-12                 # cells of unused octs hold zeros (floored to 1e-10, then scaled)
    raised = tuple(f * float(np.median(x[gas])) for f, x in zip((1, 100, 1), (U[0], np.sqrt(r.p.gamma * p / U[0]), p)))
    for k in range(3):
        err = tuple((0.015, 0.1, 0.05)[j] if j == k else -1.0 for j in range(3))
        flo = tuple(raised[j] if j == k else 1e-10 for j in range(3))
        got, ref = _flags(orc, dev, r, err, flo, u)
        assert np.array_equal(got, ref), k
        low = _flags(orc, dev, r, err, (1e-10,) * 3, u)[1]
        assert ref.sum() > 0 and not np.array_equal(ref, low), k


# ---- MHD ---------------------------------------------------------------------------------------------------------------------
def _mhd_case(coarse, level, bound, r1d, r2d, st, q):
    c = MhdCase(level, riemann=r1d, riemann2d=r2d, slope_type=st, slope_mag_type=1 if st == 8 else -1, bound=bound, coarse=coarse,
                boxlen=q["scale"] * coarse[0], order=2, seed=3, gamma=q["gamma"], courant_factor=q["courant_factor"],
                slope_theta=q["slope_theta"])
    ext = c.mesh.extent(level)
    d0 = mhd_box_state(ext, gamma=q["gamma"])
    d0[0] *= 1 + 0.2 * (np.random.default_rng(4).standard_normal(d0[0].shape) > 1.3)
    c.init_dense(d0)
    return c, ext


def _mhd_oracle(coarse, level, bound, r1d, r2d, st, q):
    c, _ = _mhd_case(coarse, level, bound, r1d, r2d, st, q)
    dt, sums = c.oracle_courant()
    dt *= 0.7
    return c, dt, sums, c.oracle_godunov(dt, nthreads=4)


@pytest.mark.parametrize("coarse,level,bound,r1d,r2d,st", [
    ((1, 1, 1), 4, (0,) * 6, "hlld", "hlld", 8), ((2, 1, 1), 3, (0,) * 6, "roe", "llf", 8), ((1, 2, 1), 3, (2, 2, 0, 0, 0, 0), "llf", "roe", 2),
    ((1, 1, 1), 4, (0,) * 6, "hll", "hlla", 1), ((2, 1, 1), 3, (0, 0, 1, 1, 0, 0), "hydro", "hll", 8)])
def test_mhd_six_pass_kernels_at_m1(orc, dev, coarse, level, bound, r1d, r2d, st):
    """the six MHD passes of the dense sweep at gamma 1.4, courant_factor 0.5, slope_theta 1.2 and box scale 0.75, slope_type 8
    among them: the new state equals the oracle's, and gamma, slope_theta (slope_type 8) and the scale reach it"""
    c, dt, _, unew = _mhd_oracle(coarse, level, bound, r1d, r2d, st, M1)
    ext = c.mesh.extent(level)
    shell = [int(bound[2 * d] > 0) for d in range(3)]
    uin, act, slot = level_slots(c.mesh, level, c.u, 11)
    uout = np.zeros_like(uin)
    dev.devnum_mhd_sweep_box(IP3(*ext), IP3(*shell), MHD_R1D[r1d], MHD_R2D[r2d], 0 if st == 0 else 1, orc.dptr(uin), orc.dptr(uout), dt,
                             M1["scale"] * 2.0 ** -level, M1["gamma"], c.p.smallr, c.p.smallc, st, c.p.slope_mag_type, M1["slope_theta"],
                             M1["courant_factor"])
    s = c.mesh.s
    U = unew.reshape(11, s.ncell)
    for ind in range(8):
        cells = s.ncoarse + ind * s.ngridmax + act - 1
        assert np.array_equal(uout[:, ind, slot], U[:, cells]), ind
    keys = ("gamma", "scale") + (("slope_theta",) if st == 8 else ())
    _assert_each_parameter_matters(lambda q: (_mhd_oracle(coarse, level, bound, r1d, r2d, st, q)[3],), M1, MSUITE, keys)


@pytest.mark.parametrize("coarse,level,bound,nblocks", [((1, 1, 1), 4, (0,) * 6, 3), ((3, 2, 1), 3, (2, 2, 0, 0, 0, 0), 5)])
def test_mhd_courant_kernel_at_m1(orc, dev, coarse, level, bound, nblocks):
    """mhd_courant_kernel at gamma 1.4, courant_factor 0.5 and a cell size of 0.75 2^-level: the time step equals the oracle's
    bit for bit, the sums agree to 1e-12; gamma, courant_factor and the scale reach the oracle's time step"""
    c, ext = _mhd_case(coarse, level, bound, "hlld", "hlld", 1, M1)
    dt_ref, sums = c.oracle_courant()
    uin, _, _ = level_slots(c.mesh, level, c.u, 11)
    shell = [int(bound[2 * d] > 0) for d in range(3)]
    part = np.zeros(5 * nblocks)
    dx = M1["scale"] * 2.0 ** -level
    dev.devnum_mhd_courant.argtypes = [IP3, IP3, C.c_int, DP, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, DP]
    dev.devnum_mhd_courant(IP3(*ext), IP3(*shell), nblocks, orc.dptr(np.ascontiguousarray(uin)), dx, c.p.gamma, c.p.smallr, c.p.smallc,
                           c.p.courant_factor, orc.dptr(part))
    p5 = part.reshape(5, nblocks)
    assert min(p5[0].min(), c.p.courant_factor * dx / c.p.smallc, c.p.boxlen / c.p.smallc) == dt_ref
    got = p5[1:].sum(axis=1) * dx ** 3
    assert np.all(np.abs(got - sums) <= 1e-12 * np.abs(sums).max()), (got, sums)

    def run(q):
        c2, _ = _mhd_case(coarse, level, bound, "hlld", "hlld", 1, q)
        return (np.array([c2.oracle_courant()[0]]),)
    _assert_each_parameter_matters(run, M1, MSUITE, ("gamma", "courant_factor", "scale"))


def _mhd_amr_run(ndim):
    """the MHD AMR runs of the emulated-kernel tests at gamma 1.4 and courant_factor 0.5"""
    kw = dict(gamma=M1["gamma"], courant_factor=M1["courant_factor"])
    if ndim == 1:
        from oracle.amr_mhd import MhdAmrRun
        from test_oracle_golden import IMHD
        r = MhdAmrRun(5, 10, (2, 2, 0, 0, 0, 0), 3.5, nsubcycle=[1, 1, 1, 1], riemann="hlld", slope_type=2, err_grad_d=0.01,
                      err_grad_u=0.05, err_grad_p=0.05, interpol_type=2, regions=IMHD, tout=[1e9], ngridmax=10000, **kw)
        r.run(max_coarse=12)
    elif ndim == 2:
        from oracle.amr_mhd import MhdAmrRun2D
        r = MhdAmrRun2D(4, 6, 1.0, nsubcycle=[1], riemann="roe", riemann2d="llf", slope_type=1, err_grad_p=0.1, interpol_type=2,
                        tout=[1e9], nexpand=1, ngridmax=20000, **kw)
        r.run(max_coarse=16)
    else:
        r = _mhd3_static_run("hlld", "hlld", 2)
        r.pm.gamma, r.pm.courant_factor = kw["gamma"], kw["courant_factor"]
    return r


@pytest.mark.parametrize("ndim", [1, 2, 3])
def test_mhd_amr_kernels_at_gamma_1_4(orc, dev, ndim):
    """the MHD AMR kernels (godunov_fine with the Euler and EMF refluxes, upload_fine, the leaf-cell Courant step, the 1-D
    boundaries) at gamma 1.4 and courant_factor 0.5 on the refined meshes of the emulated-kernel tests: equal the oracle bit for
    bit on every level; gamma and courant_factor each reach the oracle's update or time step"""
    r = _mhd_amr_run(ndim)
    assert r.pm.gamma == M1["gamma"] and r.pm.courant_factor == M1["courant_factor"]
    L = orc.lib()
    if ndim == 1:
        nlev, nrefl, moved = _mhd_amr_compare_levels(orc, dev, r, 1, "hlld", "llf", 2, 2, L.orc_mhd1_godunov_fine, L.orc_mhd1_upload_fine,
                                                     L.orc_mhd1_courant_fine, boundary=L.orc_mhd1_make_boundary_hydro)
    elif ndim == 2:
        nlev, nrefl, moved = _mhd_amr_compare_levels(orc, dev, r, 2, "roe", "llf", 1, 2, L.orc_mhd2_godunov_fine, L.orc_mhdn_upload_fine,
                                                     L.orc_mhdn_courant_fine)
    else:
        nlev, nrefl, moved = _mhd_amr_compare_levels(orc, dev, r, 3, "hlld", "hlld", 2, 2, L.orc_mhd3_godunov_fine, L.orc_mhdn_upload_fine,
                                                     L.orc_mhdn_courant_fine)
    assert nlev >= 2 and nrefl > 0 and moved > 1e-6
    _assert_each_parameter_matters(lambda q: mhd_amr_oracle(orc, r, q), M1, MSUITE, ("gamma", "courant_factor"))


def mhd_amr_oracle(orc, r, q):
    """godunov_fine and courant_fine of every populated level of the MHD AMR run r with gamma and courant_factor of q: the results
    the MHD AMR comparisons look at"""
    L = orc.lib()
    godunov = {1: L.orc_mhd1_godunov_fine, 2: L.orc_mhd2_godunov_fine, 3: L.orc_mhd3_godunov_fine}[r.ndim]
    courant = L.orc_mhd1_courant_fine if r.ndim == 1 else L.orc_mhdn_courant_fine
    saved = (r.pm.gamma, r.pm.courant_factor)
    out = []
    try:
        r.pm.gamma, r.pm.courant_factor = q["gamma"], q["courant_factor"]
        for l in range(r.levelmin, r.nlevelmax + 1):
            if len(r.active[l]) == 0:
                continue
            dt = 0.5 * r.dtnew[r.levelmin] / 2 ** (l - r.levelmin)
            unew = np.zeros_like(r.uold)
            L.orc_mhdn_set_unew(r.mp, l, orc.dptr(r.uold), orc.dptr(unew))
            godunov(C.byref(r.pm), r.mp, l, r.levelmin, r.nvector, dt, orc.dptr(r.uold), orc.dptr(unew))
            out += [unew, np.array([courant(C.byref(r.pm), r.mp, l, r.p.boxlen / r.p.smallc, orc.dptr(r.uold))])]
    finally:
        r.pm.gamma, r.pm.courant_factor = saved
    return tuple(out)


# ---- the oracle's gamma dependence against an exact Riemann solution -------------------------------------------------------------
def exact_riemann(x, t, left, right, gamma, x0=0.5):
    """the self-similar solution of the 1-D Riemann problem left = (rho, u, p), right = (rho, u, p) at x0 and time t: the star
    pressure is the root of the pressure function (Toro, Riemann Solvers and Numerical Methods, sec. 4.2-4.5) found to 1e-14;
    returns rho, u, p at x"""
    g = gamma
    (rl, ul, pl), (rr, ur, pr) = left, right
    cl, cr = np.sqrt(g * pl / rl), np.sqrt(g * pr / rr)

    def f(p, rk, pk, ck):
        if p > pk:
            a, b = 2.0 / ((g + 1) * rk), (g - 1) / (g + 1) * pk
            return (p - pk) * np.sqrt(a / (p + b))
        return 2 * ck / (g - 1) * ((p / pk) ** ((g - 1) / (2 * g)) - 1)

    ps = optimize.brentq(lambda p: f(p, rl, pl, cl) + f(p, rr, pr, cr) + ur - ul, 1e-12, 10 * max(pl, pr), xtol=1e-14 * max(pl, pr),
                         rtol=4 * np.finfo(float).eps, maxiter=500)
    us = 0.5 * (ul + ur) + 0.5 * (f(ps, rr, pr, cr) - f(ps, rl, pl, cl))
    s = (np.asarray(x) - x0) / t
    rho, u, p = np.empty_like(s), np.empty_like(s), np.empty_like(s)
    for i, si in enumerate(s):
        if si <= us:       # left of the contact
            rk, uk, pk, ck, sg = rl, ul, pl, cl, -1.0
        else:
            rk, uk, pk, ck, sg = rr, ur, pr, cr, 1.0
        if ps > pk:        # shock
            rs = rk * (ps / pk + (g - 1) / (g + 1)) / ((g - 1) / (g + 1) * ps / pk + 1)
            sk = uk + sg * ck * np.sqrt((g + 1) / (2 * g) * ps / pk + (g - 1) / (2 * g))
            inside = si * sg < sk * sg
            rho[i], u[i], p[i] = (rs, us, ps) if inside else (rk, uk, pk)
        else:              # rarefaction
            rs = rk * (ps / pk) ** (1 / g)
            cs = ck * (ps / pk) ** ((g - 1) / (2 * g))
            head, tail = uk + sg * ck, us + sg * cs
            if si * sg >= head * sg:
                rho[i], u[i], p[i] = rk, uk, pk
            elif si * sg <= tail * sg:
                rho[i], u[i], p[i] = rs, us, ps
            else:
                uf = 2 / (g + 1) * (-sg * ck + (g - 1) / 2 * uk + si)
                cf = 2 / (g + 1) * ck - sg * (g - 1) / (g + 1) * (uk - si)
                rho[i] = rk * (cf / ck) ** (2 / (g - 1))
                u[i], p[i] = uf, pk * (cf / ck) ** (2 * g / (g - 1))
    return rho, u, p


SOD = ((1.0, 0.0, 1.0), (0.125, 0.0, 0.1))


def _sod_l1(riemann, level, gamma_run, gamma_ref, tend=0.2):
    """L1 errors (rho, u, p) of the oracle's Sod tube at gamma_run on 2^level cells against the exact solution at gamma_ref, at
    the time the run reached"""
    from helpers import SOD_REGIONS
    c = Case(1, level, riemann=riemann, slope_type=2, bound=(1, 1, 0, 0, 0, 0), gamma=gamma_run)
    c.init_regions(SOD_REGIONS)
    u, t = c.u.copy(), 0.0
    while t < tend:
        u, dts = c.oracle_steps(1, u)
        t += dts[0]
    d = c.dense(u)
    rho = d[0, 0, 0]
    vel = d[1, 0, 0] / rho
    p = (gamma_run - 1) * (d[2, 0, 0] - 0.5 * rho * vel ** 2)
    n = 1 << level
    x = (np.arange(n) + 0.5) / n
    ra, ua, pa = exact_riemann(x, t, *SOD, gamma_ref)
    return np.abs(rho - ra).mean(), np.abs(vel - ua).mean(), np.abs(p - pa).mean()


def test_exact_riemann_reference_reproduces_the_sod_star_state():
    """the numpy reference solution: at gamma 1.4 the Sod star state is the textbook one (p* = 0.30313, u* = 0.92745), and the
    solution conserves mass between the walls of the waves"""
    x = np.linspace(0.0, 1.0, 20001)
    rho, u, p = exact_riemann(x, 0.2, *SOD, 1.4)
    mid = np.abs(x - 0.7) < 1e-3                       # between the contact (0.685) and the shock (0.850) at t = 0.2
    assert np.allclose(p[mid], 0.30313, atol=1e-5) and np.allclose(u[mid], 0.92745, atol=1e-5)
    assert abs(np.trapezoid(rho, x) - 0.5625) < 1e-4


@pytest.mark.parametrize("gamma", [5.0 / 3.0, 1.2])
@pytest.mark.parametrize("riemann", ["llf", "hllc", "exact", "acoustic", "hll"])
def test_oracle_sod_tube_at_other_gammas_vs_exact_solution(orc, riemann, gamma):
    """the oracle's uniform 1024-cell Sod tube at gamma 5/3 and 1.2 against the exact solution at the same gamma: L1 errors of
    a few 1e-3, like the gamma-1.4 pin against the reference's analytic file; the same run against the exact solution at gamma
    1.4 is off by far more"""
    tol = {"exact": 2.5e-3, "hllc": 2.5e-3, "acoustic": 2.5e-3, "hll": 3e-3, "llf": 4e-3}[riemann]
    er, eu, ep = _sod_l1(riemann, 10, gamma, gamma)
    assert er < tol and eu < 2 * tol and ep < tol, (er, eu, ep)
    wrong = _sod_l1(riemann, 10, gamma, 1.4)
    assert max(wrong) > 4 * tol, wrong


@pytest.mark.parametrize("gamma", [5.0 / 3.0, 1.2])
def test_oracle_sod_tube_at_other_gammas_converges(orc, gamma):
    """the L1 density error against the exact solution drops at first order from 256 to 1024 cells"""
    errs = [_sod_l1("hllc", lev, gamma, gamma)[0] for lev in (8, 9, 10)]
    assert errs[1] < 0.7 * errs[0] and errs[2] < 0.7 * errs[1], errs


def test_oracle_sod_tube_at_gamma_1_4_is_not_the_5_3_solution(orc):
    """the sanity check of the reference solution: the oracle run at gamma 1.4 fails the gamma-5/3 tolerance"""
    assert max(_sod_l1("hllc", 10, 1.4, 5.0 / 3.0)) > 1e-2
