"""Passive scalars (NVAR = NDIM+2+NPS, NDIM = 3, NPS = 1, 2; AMR mode) on the CPU, bit for bit against the oracle: the NX forms of
the five Riemann solvers, the NPS = 0, 1, 2 instantiations of the oct-batch kernel (picked by the same selection as
launch_amr_godfine), the set_uold floor fix, upload_fine and the physical boundaries with nvar = 6, 7, and the drop-in flow of a
3-D adaptive run whose godunov_fine is the device code.  The device code is compiled for the host by tests/host_numerics
(devnum_scalars.cpp) and run by its emulated launch.  One CPU test pins the oracle itself: on a uniform flow the scalars of one
step equal an independent numpy statement of the MUSCL-Hancock step."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from helpers import FLOORS

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_numerics")
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "ramses_b200", "csrc")
DP, IP = C.POINTER(C.c_double), C.POINTER(C.c_int)
SOLVER_ID = {"llf": 0, "exact": 1, "acoustic": 2, "hllc": 3, "hll": 4}
ORC_RIEMANN = {"llf": "orc_riemann_llf", "exact": "orc_riemann_approx", "acoustic": "orc_riemann_acoustic", "hllc": "orc_riemann_hllc",
               "hll": "orc_riemann_hll"}


@pytest.fixture(scope="module")
def scl():
    """devnum_scalars.cpp (devnum.cpp's emulated launch + the passive-scalar entry points) built for the host like devnum.cpp"""
    lib = os.path.join(HERE, "libdevnum_scalars_host.so")
    srcs = [os.path.join(HERE, f) for f in ("devnum_scalars.cpp", "devnum.cpp", os.path.join("stub", "cuda_runtime.h"))] + \
        [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    if not os.path.exists(lib) or os.path.getmtime(lib) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fno-fast-math", "-std=c++17", "-fPIC", "-shared", "-pthread",
                               "-fvisibility=hidden", "-fvisibility-inlines-hidden", "-Wl,-Bsymbolic",
                               "-I" + os.path.join(HERE, "stub"), "-I" + CSRC, "-I" + HERE, "-o", lib,
                               os.path.join(HERE, "devnum_scalars.cpp")])
    L = C.CDLL(lib, mode=os.RTLD_LOCAL | os.RTLD_NOW)
    L.devnum_riemann_nx.argtypes = [C.c_int, C.c_int, C.c_int, DP, DP, DP, DP, C.c_double, C.c_double, C.c_double, C.c_int]
    L.devnum_amr_godfine_nps.argtypes = [C.c_int] * 7 + [IP, IP, IP, IP, C.c_int, C.c_int, DP, DP, DP, C.c_double, C.c_double] + \
        [C.c_int] * 3 + [C.c_double] * 3 + [C.c_int, C.c_int]
    L.devnum_amr_godunov_nps.argtypes = [C.c_int] * 7 + [IP, IP, IP, IP, C.c_int, C.c_int, DP, DP, C.c_double, C.c_double] + \
        [C.c_int] * 3 + [C.c_double] * 3 + [C.c_int] * 3
    L.devnum_amr_list_pass.argtypes = [C.c_int] * 7 + [IP, IP, IP, IP, C.c_int, C.c_int, DP, DP, C.c_double, C.c_int, C.c_int, DP]
    return L


# ---- the Riemann solvers with NX = 1, 2 ------------------------------------------------------------------------------------------
def _scalar_face_states(nx, seed):
    """_hydro_states of the 3-D hydro tests (smooth pairs, strong shocks, both floors, cold rarefactions) plus nx scalars in [-1, 2],
    and rows where the upwinding of the scalars ties: ustar = 0 (equal pressures at rest, density jump), a zero mass flux with
    sgnm = +1 (exact / acoustic pick the left state at ustar = 0) and exactly mirrored states"""
    from test_device_numerics_host import _hydro_states
    rng = np.random.default_rng(seed)
    n = 8000
    h_l, h_r = _hydro_states(rng, n, 3)
    ql, qr = np.zeros((n + 300, 5 + nx)), np.zeros((n + 300, 5 + nx))
    ql[:n, :5], qr[:n, :5] = h_l, h_r
    ql[:, 5:], qr[:, 5:] = rng.uniform(-1.0, 2.0, (n + 300, nx)), rng.uniform(-1.0, 2.0, (n + 300, nx))
    t = slice(n, n + 100)                                  # contact at rest: ul = ur = 0, pl = pr, rho jumps
    ql[t, 0], qr[t, 0] = 10.0 ** rng.uniform(-3, 2, 100), 10.0 ** rng.uniform(-3, 2, 100)
    ql[t, 2] = qr[t, 2] = 10.0 ** rng.uniform(-3, 2, 100)
    ql[t, 3:5], qr[t, 3:5] = rng.standard_normal((100, 2)), rng.standard_normal((100, 2))
    t = slice(n + 100, n + 200)                            # identical states at rest
    ql[t, :5] = np.c_[10.0 ** rng.uniform(-3, 2, 100), np.zeros(100), 10.0 ** rng.uniform(-3, 2, 100), rng.standard_normal((100, 2))]
    qr[t, :5] = ql[t, :5]
    t = slice(n + 200, n + 300)                            # mirrored states: ul = -ur, the same rho and P -> ustar = 0
    ql[t, :5] = np.c_[10.0 ** rng.uniform(-3, 2, 100), rng.standard_normal(100), 10.0 ** rng.uniform(-3, 2, 100), rng.standard_normal((100, 2))]
    qr[t, :5] = ql[t, :5] * np.array([1, -1, 1, 1, 1])
    return np.ascontiguousarray(ql), np.ascontiguousarray(qr)


@pytest.mark.parametrize("nx", [1, 2])
@pytest.mark.parametrize("solver", ["llf", "exact", "acoustic", "hllc", "hll"])
def test_riemann_with_scalars_equals_oracle(orc, scl, nx, solver):
    """riemann<3, RS, NX> (fg of all 5+nx variables and the internal-energy flux fe) == the oracle's solver with nvar = 5+nx, bit
    for bit under both floor settings; the scalar fluxes are not all zero, and the tie rows give finite fluxes"""
    ql, qr = _scalar_face_states(nx, 10 * nx + SOLVER_ID[solver])
    n, nv = ql.shape
    f = getattr(orc.lib(), ORC_RIEMANN[solver])
    f.argtypes = [C.POINTER(orc.Params), DP, DP, DP, C.c_int]
    for smallr, smallc in FLOORS.values():
        fg, fe = np.zeros((n, nv)), np.zeros(n)
        assert scl.devnum_riemann_nx(SOLVER_ID[solver], nx, n, orc.dptr(ql), orc.dptr(qr), orc.dptr(fg), orc.dptr(fe), 1.4, smallr,
                                     smallc, 10) == 0
        p = orc.make_params(ndim=3, nvar=nv, riemann=solver, nvector=n, niter_riemann=10, smallr=smallr, smallc=smallc)
        qlf, qrf = np.asfortranarray(ql), np.asfortranarray(qr)
        fgf = np.zeros((n, nv + 1), order="F")
        f(C.byref(p), qlf.ctypes.data_as(DP), qrf.ctypes.data_as(DP), fgf.ctypes.data_as(DP), n)
        assert np.isfinite(fg).all() and np.isfinite(fe).all()
        assert np.array_equal(fg, fgf[:, :nv])
        assert np.array_equal(fe, fgf[:, nv])
        assert (np.abs(fg[:, 5:]) > 0).mean() > 0.5
        # the scalar flux of every row is the mass flux times an upwind concentration (hllc / exact / acoustic) or a blend of both
        if solver in ("hllc", "exact", "acoustic"):
            up = np.where(np.isclose(fg[:, 5:], fg[:, :1] * ql[:, 5:], rtol=1e-12, atol=0), 1, 0) | \
                np.where(np.isclose(fg[:, 5:], fg[:, :1] * qr[:, 5:], rtol=1e-12, atol=0), 1, 0)
            assert up.all()


# ---- the oct-batch kernel on an adaptively refined 3-D mesh --------------------------------------------------------------------
def _cell_positions(r, l):
    """octs of level l of run r and the centres of their cells: ig [n], x [T][3][n] in units of the box (one coarse cell)"""
    ig = np.asarray(r.active[l], dtype=np.int64)
    dx = 0.5 ** l
    x = np.stack([np.stack([r.xg[d, ig] + (((ind >> d) & 1) - 0.5) * dx for d in range(3)]) for ind in range(r.T)])
    return ig, x


def fill_scalars(r, seed):
    """scalar fields on every oct cell of run r (nvar = 6 or 7): Z1 = a step in x plus a sine, Z2 = a smooth blob plus a different
    step; both span negative values and values above 1.  rho Z is written, with rho the cell's own density."""
    rng = np.random.default_rng(seed)
    U = r.uold.reshape(r.nvar, r.ncell)
    U[5:] = 0.3 * U[0]
    for l in range(1, r.nlevelmax + 1):
        if not len(r.active[l]):
            continue
        ig, x = _cell_positions(r, l)
        for ind in range(r.T):
            c = r.ncoarse + ind * r.ngridmax + ig - 1
            X, Y, Z = x[ind]
            z1 = np.where(X < 0.45, 1.5, -0.5) + 0.4 * np.sin(2 * np.pi * (X + 0.3 * Y))
            U[5, c] = U[0, c] * z1
            if r.nvar > 6:
                z2 = np.exp(-((X - 0.4) ** 2 + (Y - 0.55) ** 2 + (Z - 0.5) ** 2) / 0.02) + np.where(Z > 0.6, 0.8, -0.2)
                U[6, c] = U[0, c] * (z2 + 0.01 * rng.standard_normal(len(c)))


def _sedov_run(nvar, solver="hllc", itype=1):
    """the 3-D adaptively refined mesh of test_amr_oct_batch_kernel_emulated_on_the_cpu_equals_oracle (levels 3..5) with nvar
    variables; the scalars are filled after the flow has developed"""
    from oracle.amr import FastAmrRun
    reg = [dict(type="square", x_center=0.5, y_center=0.5, z_center=0.5, length_x=10, length_y=10, length_z=10, exp_region=10, d=1.0, p=1e-5),
           dict(type="point", x_center=0.5, y_center=0.5, z_center=0.5, p=0.4)]
    r = FastAmrRun(3, 3, 5, (0,) * 6, 1.0, nsubcycle=[1, 2], ngridmax=4000, riemann=solver, slope_type=1, err_grad_p=0.1,
                   interpol_type=itype, regions=reg, tout=[1e9], nvar=nvar)
    r.run(max_coarse=3)
    return r


def _tree_args(r):
    m = r.m
    son = np.ascontiguousarray(r.son[1:], dtype=np.int32)
    father = np.ascontiguousarray(r.father[1:], dtype=np.int32)
    nbor = np.ascontiguousarray(r.nbor[:, 1:], dtype=np.int32)
    return (r.ncoarse, r.ngridmax, m.nx, m.ny, m.nz), (son, father, nbor)


# (solver, slope_type, interpol_type, interpol_var, nvar): every solver with one and with two scalars, slope_type 0/1/2/3/7/8, and
# interpol (type, var) in {(0,0), (1,0), (2,1), (3,2), (4,2)} with scalars; two NPS = 0 rows with interpol_var 1 / 2
GODFINE_ROWS = [("hllc", 1, 0, 0, 6), ("hllc", 8, 1, 0, 7), ("llf", 2, 1, 0, 6), ("llf", 3, 2, 1, 7), ("hll", 7, 2, 1, 6),
                ("hll", 0, 3, 2, 7), ("exact", 2, 3, 2, 6), ("exact", 1, 4, 2, 7), ("acoustic", 3, 4, 2, 6), ("acoustic", 7, 0, 0, 7),
                ("hllc", 2, 2, 1, 5), ("llf", 1, 4, 2, 5)]


def _set_interpol(orc, itype, ivar):
    L = orc.lib()
    L.orc_set_interpol.argtypes = [C.c_int, C.c_int]
    L.orc_set_interpol(itype, ivar)


@pytest.fixture(scope="module")
def sedov_runs():
    return {nvar: _sedov_run(nvar) for nvar in (5, 6, 7)}


@pytest.mark.parametrize("solver,st,itype,ivar,nvar", GODFINE_ROWS)
def test_amr_oct_batch_kernel_with_scalars_equals_oracle(orc, scl, sedov_runs, solver, st, itype, ivar, nvar):
    """amr_godfine_kernel<3, RS, false, NPS> for NPS = nvar - 5 = 0, 1, 2 (chosen by amr_godfine_select, the selection
    launch_amr_godfine launches) on the 3-level adaptively refined mesh: gather, prolongation of ghost octs incl. the coupled
    interpol_var 1 / 2 and interpol_type 4 path (one thread per father cell), ctoprim q = u/rho, the slopes, the scalar trace,
    the solvers' scalar fluxes and the update of every level == set_unew + godunov_fine of the oracle, bit for bit; the outer-face
    fluxes rflux carry all nvar columns and refluxed into the coarser cells (devnum_amr_godunov_nps) equal the oracle's coarse
    cells too.  Covering set (GODFINE_ROWS): every solver with one and two scalars, slope_type 0/1/2/3/7/8, interpol
    (type, var) (0,0) (1,0) (2,1) (3,2) (4,2), and NPS = 0 with interpol_var 1 and 2."""
    r = sedov_runs[nvar]
    uold = r.uold.copy()
    if nvar > 5:
        fill_scalars(r, 7 + nvar)
    try:
        _godfine_compare(orc, scl, r, solver, st, itype, ivar, nvar)
    finally:
        r.uold[:] = uold


def _godfine_compare(orc, scl, r, solver, st, itype, ivar, nvar, dt_of=None):
    dims, (son, father, nbor) = _tree_args(r)
    L = orc.lib()
    p = orc.make_params(ndim=3, nvar=nvar, riemann=solver, slope_type=st, nvector=r.nvector, smallr=r.p.smallr, smallc=r.p.smallc)
    nlev, moved = 0, 0.0
    T, nc = 8, r.ncell
    try:
        _set_interpol(orc, itype, ivar)
        for l in range(r.levelmin, r.nlevelmax + 1):
            act = np.ascontiguousarray(r.active[l], dtype=np.int32)
            if len(act) == 0:
                continue
            dt = dt_of(l) if dt_of else 0.4 * r.dtnew[r.levelmin] / 2 ** (l - r.levelmin)
            dx = 0.5 ** l
            unew_o = np.zeros_like(r.uold)
            L.orc_set_unew(C.byref(p), r.mp, l, orc.dptr(r.uold), orc.dptr(unew_o))
            L.orc_godunov_fine(C.byref(p), r.mp, l, dt, orc.dptr(r.uold), orc.dptr(unew_o), 1)
            # uold / unew with NaN columns up to 7 variables behind the state: a kernel built for the wrong NPS (a broken selection)
            # reads and writes them and fails the comparison, instead of running past the arrays
            pad = np.full((7 - nvar) * nc, np.nan) if nvar < 7 else np.zeros(0)
            uold_k = np.concatenate([r.uold, pad])
            unew_k = np.concatenate([np.zeros_like(r.uold), pad])
            L.orc_set_unew(C.byref(p), r.mp, l, orc.dptr(r.uold), orc.dptr(unew_k))
            assert scl.devnum_amr_godunov_nps(3, SOLVER_ID[solver], *dims, orc.iptr(son), orc.iptr(father), orc.iptr(nbor), orc.iptr(act),
                                              len(act), l, orc.dptr(uold_k), orc.dptr(unew_k), dt, dx, itype, ivar, st, 1.4, r.p.smallr,
                                              r.p.smallc, 10, nvar, r.nvector) == 0
            unew_k = unew_k[:nvar * nc]
            assert np.isfinite(unew_o).all()
            assert np.array_equal(unew_k, unew_o), (l, float(np.abs(unew_k - unew_o).max()))
            cells = np.concatenate([r.ncoarse + ind * r.ngridmax + act.astype(np.int64) - 1 for ind in range(T)])
            Uo = unew_o.reshape(nvar, nc)
            moved = max(moved, float(np.abs(Uo[nvar - 1, cells] - r.uold.reshape(nvar, nc)[nvar - 1, cells]).max()))
            nlev += 1
    finally:
        _set_interpol(orc, 1, 0)
    assert nlev >= 3 and moved > 1e-6


def test_amr_oct_batch_kernel_selection_rejects_what_is_not_built(orc, scl, sedov_runs):
    """amr_godfine_select returns no kernel for three scalars (nvar = 8) and for scalars in 1-D / 2-D, so the harness, like
    launch_amr_godfine, refuses them instead of running a kernel for the wrong NPS"""
    r = sedov_runs[6]
    dims, (son, father, nbor) = _tree_args(r)
    act = np.ascontiguousarray(r.active[3], dtype=np.int32)
    u = np.zeros(8 * r.ncell)
    rf = np.zeros(len(act) * 6 * 4 * 8)
    assert scl.devnum_amr_godfine_nps(3, 3, *dims, orc.iptr(son), orc.iptr(father), orc.iptr(nbor), orc.iptr(act), len(act), 3,
                                      orc.dptr(u), orc.dptr(u.copy()), orc.dptr(rf), 1e-3, 0.125, 1, 0, 1, 1.4, 1e-10, 1e-10, 10, 8) == -1
    assert scl.devnum_amr_godfine_nps(2, 3, *dims, orc.iptr(son), orc.iptr(father), orc.iptr(nbor), orc.iptr(act), len(act), 3,
                                      orc.dptr(u), orc.dptr(u.copy()), orc.dptr(rf), 1e-3, 0.125, 1, 0, 1, 1.4, 1e-10, 1e-10, 10, 5) == -1


# ---- floor states: the oct-batch kernel and the set_uold floor fix ------------------------------------------------------------
@pytest.mark.parametrize("floors", ["default", "raised"])
@pytest.mark.parametrize("solver,nvar", [("hllc", 6), ("llf", 7), ("exact", 7)])
def test_scalar_floor_fix_at_the_floors_equals_oracle(orc, scl, sedov_runs, floors, solver, nvar):
    """every cell of the refined mesh holds a floor_state cell with scalars (helpers.fill_floor_state with nvar): per level, the
    oct-batch kernel + coarse reflux, then amr_scalar_floor_kernel, then uold = unew == the oracle's set_unew -> godunov_fine ->
    set_uold (godunov_fine.f90:176-190), bit for bit; both branches of the fix fire (inflow into a floored cell and outflow below
    the floor)"""
    from helpers import fill_floor_state
    r = sedov_runs[nvar]
    saved = (r.uold.copy(), r.p.smallr, r.p.smallc)
    try:
        smallr, smallc = fill_floor_state(r.uold, 3, nvar, r.ncell, floors, 70 + nvar)
        r.p.smallr, r.p.smallc = smallr, smallc
        d = r.uold.reshape(nvar, r.ncell)
        rho = np.maximum(d[0], smallr)
        v2 = sum((d[1 + k] / rho) ** 2 for k in range(3))
        eint = np.maximum(d[4] / rho - 0.5 * v2, smallc ** 2 / 1.4 / 0.4)
        dt_fine = 0.3 * 0.5 ** r.nlevelmax / float((np.sqrt(v2) + np.sqrt(1.4 * 0.4 * eint)).max())
        dims, (son, father, nbor) = _tree_args(r)
        L = orc.lib()
        p = orc.make_params(ndim=3, nvar=nvar, riemann=solver, slope_type=2, nvector=r.nvector, smallr=smallr, smallc=smallc)
        _set_interpol(orc, 1, 0)
        up = down = 0
        for l in range(r.levelmin, r.nlevelmax + 1):
            act = np.ascontiguousarray(r.active[l], dtype=np.int32)
            if len(act) == 0:
                continue
            dt = dt_fine * 2 ** (r.nlevelmax - l)
            cells = np.concatenate([r.ncoarse + ind * r.ngridmax + act.astype(np.int64) - 1 for ind in range(8)])
            uold_o, unew_o = r.uold.copy(), np.zeros_like(r.uold)
            L.orc_set_unew(C.byref(p), r.mp, l, orc.dptr(uold_o), orc.dptr(unew_o))
            L.orc_godunov_fine(C.byref(p), r.mp, l, dt, orc.dptr(uold_o), orc.dptr(unew_o), 1)
            L.orc_set_uold(C.byref(p), r.mp, l, orc.dptr(uold_o), orc.dptr(unew_o))
            uold_k, unew_k = r.uold.copy(), np.zeros_like(r.uold)
            L.orc_set_unew(C.byref(p), r.mp, l, orc.dptr(uold_k), orc.dptr(unew_k))
            assert scl.devnum_amr_godunov_nps(3, SOLVER_ID[solver], *dims, orc.iptr(son), orc.iptr(father), orc.iptr(nbor), orc.iptr(act),
                                              len(act), l, orc.dptr(uold_k), orc.dptr(unew_k), dt, 0.5 ** l, 1, 0, 2, 1.4, smallr, smallc,
                                              10, nvar, r.nvector) == 0
            do, dn = uold_k.reshape(nvar, -1)[0, cells], unew_k.reshape(nvar, -1)[0, cells]
            up += int(((do < smallr) & (dn > do)).sum())
            down += int(((dn < smallr) & (do > dn)).sum())
            assert scl.devnum_amr_list_pass(0, 3, *dims, orc.iptr(son), orc.iptr(father), orc.iptr(nbor), orc.iptr(act), len(act), nvar,
                                            orc.dptr(uold_k), orc.dptr(unew_k), smallr, 0, 0, None) == 0
            uold_k.reshape(nvar, -1)[:, cells] = unew_k.reshape(nvar, -1)[:, cells]
            assert np.isfinite(uold_o).all()
            assert np.array_equal(uold_k, uold_o), l
        assert up > 0 and down > 0, (up, down)
    finally:
        r.uold[:], r.p.smallr, r.p.smallc = saved


# ---- upload_fine and the physical boundaries ------------------------------------------------------------------------------------
@pytest.mark.parametrize("nvar,ivar", [(6, 0), (7, 0), (6, 1), (7, 1), (6, 2), (7, 2)])
def test_upload_with_scalars_equals_oracle(orc, scl, sedov_runs, nvar, ivar):
    """amr_upload_kernel (split cells <- mean of their sons over all nvar variables, interpol_var 1 / 2: the internal energy is
    averaged instead of the total energy) == orc_upload_fine on every level below levelmax; the split cells first hold values
    unrelated to their sons, and the scalars of some sons are negative"""
    r = sedov_runs[nvar]
    saved = r.uold.copy()
    try:
        fill_scalars(r, 3 * nvar + ivar)
        rng = np.random.default_rng(nvar + 10 * ivar)
        r.uold *= 1.0 + 0.2 * rng.random(r.uold.shape)
        dims, (son, father, nbor) = _tree_args(r)
        p = orc.make_params(ndim=3, nvar=nvar, smallr=r.p.smallr, smallc=r.p.smallc)
        L = orc.lib()
        _set_interpol(orc, 1, ivar)
        n = 0
        for l in range(1, r.nlevelmax):
            act = np.ascontiguousarray(r.active[l], dtype=np.int32)
            if len(act) == 0:
                continue
            u_o, u_k = r.uold.copy(), r.uold.copy()
            L.orc_upload_fine(C.byref(p), r.mp, l, orc.dptr(u_o))
            assert scl.devnum_amr_list_pass(1, 3, *dims, orc.iptr(son), orc.iptr(father), orc.iptr(nbor), orc.iptr(act), len(act), nvar,
                                            orc.dptr(u_k), None, r.p.smallr, ivar, 0, None) == 0
            assert np.array_equal(u_k, u_o), l
            n += int((u_o.reshape(nvar, -1)[5:] != r.uold.reshape(nvar, -1)[5:]).any(axis=0).sum())
        assert n > 100
    finally:
        _set_interpol(orc, 1, 0)
        r.uold[:] = saved


@pytest.mark.parametrize("nvar", [6, 7])
def test_boundaries_with_scalars_equal_oracle(orc, scl, nvar):
    """amr_boundary_kernel with the arguments amr_boundaries passes (reflexive walls in x, outflow in y, imposed inflow in z) ==
    orc_make_boundary_hydro on every level of a 3-D mesh, all nvar variables: the scalars are copied by walls and outflow faces
    (not mirrored) and set from boundary_var on imposed faces"""
    from helpers import Case
    c = Case(3, 3, nvar=nvar, bound=(1, 1, 2, 2, 3, 3))
    L = orc.lib()
    L.orc_set_boundary_var.argtypes = [C.c_int, DP, C.c_int]
    bvars = {4: np.array([1.2, 0.3, -0.1, 0.5, 3.0, 0.7, -0.4])[:nvar], 5: np.array([0.8, -0.2, 0.1, -0.6, 2.0, -0.3, 1.4])[:nvar]}
    rng = np.random.default_rng(nvar)
    u = rng.uniform(0.5, 2.0, nvar * c.mesh.s.ncell)
    U = u.reshape(nvar, -1)
    U[1:4] = rng.standard_normal((3, U.shape[1]))
    U[5:] = U[0] * rng.uniform(-1.0, 2.0, (nvar - 5, U.shape[1]))
    U[4] = 2.0 + 0.5 * (U[1] ** 2 + U[2] ** 2 + U[3] ** 2) / U[0]
    m, s = c.mesh, c.mesh.s
    son = np.ascontiguousarray(m.son()[1:], dtype=np.int32)
    father = np.ascontiguousarray(m.father()[1:], dtype=np.int32)
    nbor = np.ascontiguousarray(m.nbor()[:, 1:], dtype=np.int32)
    bts = m.boundary_types()
    assert sorted(bt // 10 for bt in bts) == [0, 0, 1, 1, 2, 2]
    try:
        for b, v in bvars.items():
            L.orc_set_boundary_var(b, orc.dptr(np.ascontiguousarray(v)), nvar)
        nb = 0
        for l in range(1, c.level + 1):
            u_o, u_k = u.copy(), u.copy()
            L.orc_make_boundary_hydro(C.byref(c.p), m.ptr, l, orc.dptr(u_o))
            for b in range(s.nboundary):
                ig = np.ascontiguousarray(m.bound(b, l), dtype=np.int32)
                if len(ig) == 0:
                    continue
                bv = bvars.get(b)
                assert scl.devnum_amr_list_pass(2, 3, s.ncoarse, s.ngridmax, s.nx, s.ny, s.nz, orc.iptr(son), orc.iptr(father), orc.iptr(nbor),
                                                orc.iptr(ig), len(ig), nvar, orc.dptr(u_k), None, c.p.smallr, 0, int(bts[b]),
                                                orc.dptr(np.ascontiguousarray(bv)) if bv is not None else None) == 0
                nb += len(ig)
            assert np.array_equal(u_k, u_o), l
            assert (u_o != u).reshape(nvar, -1)[5:].any()
        assert nb > 0
    finally:
        zero = np.zeros(nvar)
        for b in bvars:
            L.orc_set_boundary_var(b, orc.dptr(zero), nvar)


# ---- the drop-in flow of a 3-D adaptive run with scalars ------------------------------------------------------------------------
def scalar_blast_run(nvar, emulate=None):
    """3-D blast (levels 3..5, regridding every coarse step, periodic) whose ejecta carry Z1 = 1 and the ambient gas Z1 = 0, plus
    (nvar = 7) a smooth second scalar; the scalars are set by init_flow_fine on every level, like a condinit with scalars"""
    from oracle.amr import FastAmrRun

    class Run(FastAmrRun):
        def init_flow_fine(self, l):
            super().init_flow_fine(l)
            if self.numbtot(l) == 0:
                return
            U = self.uold.reshape(self.nvar, self.ncell)
            ig, x = _cell_positions(self, l)
            for ind in range(self.T):
                c = self.ncoarse + ind * self.ngridmax + ig - 1
                X, Y, Z = x[ind]
                r2 = (X - 0.5) ** 2 + (Y - 0.5) ** 2 + (Z - 0.5) ** 2
                U[5, c] = U[0, c] * (r2 < 0.15 ** 2)
                if self.nvar > 6:
                    U[6, c] = U[0, c] * (0.5 + 0.3 * np.sin(2 * np.pi * X) * np.cos(2 * np.pi * Y))

    reg = [dict(type="square", x_center=0.5, y_center=0.5, z_center=0.5, length_x=10, length_y=10, length_z=10, exp_region=10, d=1.0, p=0.1),
           dict(type="square", x_center=0.5, y_center=0.5, z_center=0.5, length_x=0.3, length_y=0.3, length_z=0.3, exp_region=2, d=2.0, p=3.0)]
    return Run(3, 3, 5, (0,) * 6, 1.0, nsubcycle=[1, 2], ngridmax=6000, riemann="hllc", slope_type=2, err_grad_d=0.1, err_grad_p=0.1,
               interpol_type=1, regions=reg, tout=[1e9], nvar=nvar)


@pytest.mark.parametrize("nvar", [6, 7])
def test_dropin_with_scalars_device_code_equals_oracle(orc, scl, nvar):
    """the oracle's AMR driver with godunov_fine replaced by devnum_amr_godunov_nps (the oct-batch kernel with NPS scalars + the
    coarse reflux of all nvar variables) over 2 coarse steps of the scalar blast: state, mesh and time bit-identical to the
    all-oracle run, and the scalars moved"""
    runs = []
    for emulated in (False, True):
        r = scalar_blast_run(nvar)
        calls = [0]
        if emulated:
            def c_godunov_fine(l, r=r):
                act = np.ascontiguousarray(r.active[l], dtype=np.int32)
                if len(act) == 0:
                    return
                dims, (son, father, nbor) = _tree_args(r)
                assert scl.devnum_amr_godunov_nps(3, SOLVER_ID["hllc"], *dims, orc.iptr(son), orc.iptr(father), orc.iptr(nbor), orc.iptr(act),
                                                  len(act), l, orc.dptr(r.uold), orc.dptr(r.unew), r.dtnew[l], 0.5 ** l, 1, 0, 2, r.p.gamma,
                                                  r.p.smallr, r.p.smallc, 10, nvar, r.nvector) == 0
                calls[0] += 1
            r.c_godunov_fine = c_godunov_fine
        r.run(max_coarse=2)
        runs.append(r)
    a, b = runs
    assert a.t == b.t and a.nstep == b.nstep and a.t > 0
    assert np.array_equal(a.son, b.son) and np.array_equal(a.nbor, b.nbor) and np.array_equal(a.father, b.father)
    assert np.array_equal(a.uold, b.uold)
    assert calls[0] >= 2 * 3 and len(b.active[5]) > 0
    U = b.uold.reshape(nvar, -1)
    leaf = np.concatenate([b.ncoarse + ind * b.ngridmax + np.asarray(b.active[l], dtype=np.int64) - 1 for l in range(3, 6) for ind in range(8)])
    z1 = U[5, leaf] / U[0, leaf]
    assert ((z1 > 0.01) & (z1 < 0.99)).sum() > 50            # the ejecta mixed into the ambient gas


# ---- the oracle pinned by an independent statement of the scheme --------------------------------------------------------------
def _uslope(zl, zc, zr, st):
    """uslope (hydro/umuscl.f90:970): slope_type 0 -> 0 (:1002-1005); 1 minmod, 2 monotonized central (:1012-1021 -- the same
    limiter per direction in the 3-D branch :1240): dlft = k (zc - zl), drgt = k (zr - zc), dcen = (dlft + drgt) / (2 k),
    k = min(slope_type, 2), dq = sign(dcen) min(|dlft|, |drgt|, |dcen|), 0 where dlft drgt <= 0"""
    if st == 0:
        return np.zeros_like(zc)
    k = min(st, 2)
    dl, dr = k * (zc - zl), k * (zr - zc)
    dc = 0.5 * (dl + dr) / k
    lim = np.where(dl * dr <= 0, 0.0, np.minimum(np.abs(dl), np.abs(dr)))
    return np.sign(dc) * np.minimum(lim, np.abs(dc))


def _face_flux(solver, rho, u, p, zl, zr, gamma=1.4):
    """scalar flux through a face between two identical hydro states (rho, u, p) carrying concentrations zl | zr:
    hllc (hydro/godunov_utils.f90:1194-1202), exact (riemann_approx :488-490) and acoustic (:649-651): rho u Z of the upwind side
    (ustar = u); llf (:762-816): 0.5 (rho u zl + rho u zr - cmax rho (zr - zl)), cmax = |u| + c; hll (:874-875, :924-981):
    (SR rho u zl - SL rho u zr + SR SL rho (zr - zl)) / (SR - SL), SL = min(u - c, 0), SR = max(u + c, 0)"""
    c = np.sqrt(gamma * p / rho)
    if solver in ("hllc", "exact", "acoustic"):
        return rho * u * (zl if u > 0 else zr)
    if solver == "llf":
        return 0.5 * (rho * u * zl + rho * u * zr - (abs(u) + c) * (rho * zr - rho * zl))
    sl, sr = min(u - c, 0.0), max(u + c, 0.0)
    return (sr * rho * u * zl - sl * rho * u * zr + sr * sl * (rho * zr - rho * zl)) / (sr - sl)


@pytest.mark.parametrize("nvar", [6, 7])
@pytest.mark.parametrize("st", [0, 1, 2])
@pytest.mark.parametrize("solver", ["llf", "exact", "acoustic", "hllc", "hll"])
def test_oracle_scalar_step_equals_numpy_muscl_hancock(solver, st, nvar):
    """One oracle step of a uniform flow (rho, p, u along +x or -x, v = w = 0) carrying scalars that vary along x only (nvar = 6:
    a step plus a sine; nvar = 7: a second, different profile): (a) the hydro variables are bitwise unchanged; (b) every rho Z
    equals an independent numpy MUSCL-Hancock step to 1e-13 relative: ctoprim Z = rho Z / rho (umuscl.f90:948-961), the slope of
    _uslope, the trace Z +- dZ/2 - u dZ dt / (2 dx) (trace3d :681-700) and the solver's closed-form scalar flux (_face_flux)"""
    from helpers import Case
    n, rho, p = 16, 1.3, 0.9
    x = (np.arange(n) + 0.5) / n
    profiles = [np.where((x > 0.25) & (x < 0.6), 1.7, -0.4) + 0.3 * np.sin(2 * np.pi * x),
                0.5 + 0.5 * np.cos(4 * np.pi * x) + np.where(x > 0.8, -1.0, 0.0)]
    for u in (0.45, -0.7):
        c = Case(3, 4, riemann=solver, slope_type=st, nvar=nvar)
        d = np.zeros((nvar, n, n, n))
        d[0] = rho
        d[1] = rho * u
        d[4] = p / 0.4 + 0.5 * rho * u * u
        for k in range(nvar - 5):
            d[5 + k] = rho * profiles[k][None, None, :]
        c.init_dense(d)
        dt, _ = c.oracle_courant()
        out = c.dense(c.oracle_godunov(dt, nthreads=1))
        assert np.array_equal(out[:5], d[:5]), u
        dtdx = dt * n
        for k in range(nvar - 5):
            z = profiles[k]
            zl, zr = np.roll(z, 1), np.roll(z, -1)
            dz = _uslope(zl, z, zr, st)
            qm = z + 0.5 * dz - u * dz * dtdx * 0.5          # left state of face i+1/2
            qp = z - 0.5 * dz - u * dz * dtdx * 0.5          # right state of face i-1/2
            f = np.array([_face_flux(solver, rho, u, p, qm[i], qp[(i + 1) % n]) for i in range(n)])   # flux through face i+1/2
            ref = rho * z + dtdx * (np.roll(f, 1) - f)
            got = out[5 + k]
            assert np.allclose(got, ref[None, None, :], rtol=1e-13, atol=0), (u, k, float(np.abs(got - ref[None, None, :]).max()))
            assert np.abs(ref - rho * z).max() > 1e-3
