"""pressure_fix in the dense sweep, on the CPU: the PFIX instantiations of sweep_dense_kernel's 3-D AMR variant (tmp1 / tmp2 of
every face accumulated into divu / enew next to the conservative update, without and with the gravity predictor) compiled for
the host by tests/host_numerics and run by the emulated launch, compared with set_unew + godunov_fine of the oracle under
orc_set_pressure_fix, bit for bit."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_numerics")
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "ramses_b200", "csrc")
DP = C.POINTER(C.c_double)
IP3 = C.c_int * 3
SOLVER_ID = {"llf": 0, "exact": 1, "acoustic": 2, "hllc": 3, "hll": 4}


@pytest.fixture(scope="module")
def pfix_dev():
    """devnum_pfix.cpp (devnum.cpp's emulated launch + the PFIX entry point) built for the host, the way devnum.cpp is built"""
    lib = os.path.join(HERE, "libdevnum_pfix_host.so")
    srcs = [os.path.join(HERE, f) for f in ("devnum_pfix.cpp", "devnum.cpp", os.path.join("stub", "cuda_runtime.h"))] + \
        [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    if not os.path.exists(lib) or os.path.getmtime(lib) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fno-fast-math", "-std=c++17", "-fPIC", "-shared", "-pthread",
                               "-fvisibility=hidden", "-fvisibility-inlines-hidden", "-Wl,-Bsymbolic",
                               "-I" + os.path.join(HERE, "stub"), "-I" + CSRC, "-I" + HERE, "-o", lib,
                               os.path.join(HERE, "devnum_pfix.cpp")])
    L = C.CDLL(lib, mode=os.RTLD_LOCAL | os.RTLD_NOW)
    L.devnum_sweep_dense_pfix_box.restype = C.c_int
    L.devnum_sweep_dense_pfix_box.argtypes = [C.c_int, IP3, IP3, C.c_int, DP, DP, DP, DP, C.POINTER(C.c_ubyte), C.c_double, C.c_double,
                                              C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int]
    return L


def force_field(ncell, amp, seed):
    """f[3][ncell]: a mean pull plus cell-to-cell noise on every cell of the tree (boundary octs included)"""
    rng = np.random.default_rng(seed)
    return np.ascontiguousarray(amp * (np.array([0.8, -0.5, 0.3])[:, None] + 0.4 * rng.standard_normal((3, ncell))))


CASES = [   # coarse, level, bound, solver, slope_type, nblocks, scale (boxlen / coarse[0]: 1 = power-of-two dx)
    ((3, 2, 1), 4, (0,) * 6, "hllc", 1, 5, 1.0),                 # 48 x 32 x 16, periodic, non-cubic
    ((1, 2, 3), 4, (2, 2, 0, 0, 0, 0), "exact", 2, 7, 1.0),      # 16 x 32 x 48, outflow x
    ((3, 2, 1), 3, (1, 1, 0, 0, 0, 0), "acoustic", 3, 4, 0.75),  # 24 x 16 x 8, reflexive x walls, dx not a power of two
    ((8, 4, 1), 1, (0,) * 6, "hll", 8, 3, 1.0),                  # 16 x 8 x 2: 2-cell periodic z
    ((1, 4, 2), 2, (0, 0, 0, 0, 1, 1), "llf", 7, 2, 3.0),        # 4 x 16 x 8, walls in z, dx not a power of two
    ((2, 2, 2), 3, (0,) * 6, "hllc", 2, 1, 0.75),                # one CTA
]


def _run(orc, pfix_dev, coarse, lev, bound, solver, st, nblocks, scale, gravity, floors=None, seed=8):
    """one AMR-variant sweep of level lev with about a tenth of its cells marked refined and random refluxes preloaded into the
    state, divu and enew of unew; returns (device state, divu, enew at the active cells, the same from the oracle, the starting
    divu / enew)"""
    from helpers import FLOORS, Case, box_state, fill_floor_state, level_slots
    smallr, smallc = FLOORS[floors] if floors else (1e-10, 1e-10)
    c = Case(3, lev, riemann=solver, slope_type=st, slope_theta=1.5, bound=bound, coarse=coarse, boxlen=scale * coarse[0], order=2,
             seed=seed, smallr=smallr, smallc=smallc)
    ext = c.mesh.extent(lev)
    c.init_dense(box_state(3, ext, seed=seed))
    s = c.mesh.s
    L = orc.lib()
    if floors:
        fill_floor_state(c.u, 3, 5, s.ncell, floors, 40 + seed)
        L.orc_make_boundary_hydro(C.byref(c.p), c.mesh.ptr, lev, orc.dptr(c.u))
    f = force_field(s.ncell, 20.0, 21) if gravity else None
    act = c.mesh.active(lev).astype(np.int64)
    cells = np.concatenate([s.ncoarse + ind * s.ngridmax + act for ind in range(8)])        # 1-based
    son = c.mesh.son()
    rng = np.random.default_rng(3 + seed)
    ref_cells = cells[rng.random(len(cells)) < 0.1]
    son[ref_cells] = 1
    L.orc_set_pressure_fix.argtypes = [DP, DP, C.c_double]
    L.orc_set_gravity.argtypes = [DP]
    divu, enew = np.zeros(s.ncell), np.zeros(s.ncell)
    try:
        L.orc_set_pressure_fix(orc.dptr(divu), orc.dptr(enew), 0.5)
        L.orc_set_gravity(orc.dptr(f) if gravity else None)
        dt, _ = c.oracle_courant()
        unew = np.zeros_like(c.u)
        L.orc_set_unew(C.byref(c.p), c.mesh.ptr, lev, orc.dptr(c.u), orc.dptr(unew))
        U = unew.reshape(5, s.ncell)
        live = son[cells] == 0
        U[:, cells - 1] += 1e-3 * rng.standard_normal((5, len(cells))) * live          # refluxes of a finer level
        divu[cells - 1] += 1e-3 * rng.standard_normal(len(cells)) * live
        enew[cells - 1] += 1e-3 * rng.standard_normal(len(cells)) * live
        start, pstart = unew.copy(), np.stack([divu, enew])
        L.orc_godunov_fine(C.byref(c.p), c.mesh.ptr, lev, dt, orc.dptr(c.u), orc.dptr(unew), 1)
    finally:
        L.orc_set_pressure_fix(None, None, 0.0)
        L.orc_set_gravity(None)
        son[ref_cells] = 0
    uin, act_, slot = level_slots(c.mesh, lev, c.u, 5)
    uout, _, _ = level_slots(c.mesh, lev, start, 5)
    pout, _, _ = level_slots(c.mesh, lev, pstart.ravel(), 2)
    fin = level_slots(c.mesh, lev, f.ravel(), 3)[0] if gravity else None
    refined = np.zeros(uin.shape[1:], dtype=np.uint8)
    for ind in range(8):
        refined[ind, slot] = np.isin(s.ncoarse + ind * s.ngridmax + act, ref_cells)
    assert refined.sum() == len(ref_cells) > 0
    shell = [int(bound[2 * d] > 0) for d in range(3)]
    pfix_dev.devnum_sweep_dense_pfix_box(SOLVER_ID[solver], IP3(*ext), IP3(*shell), nblocks, orc.dptr(uin), orc.dptr(uout), orc.dptr(pout),
                                         orc.dptr(fin) if gravity else None, refined.ctypes.data_as(C.POINTER(C.c_ubyte)), dt,
                                         c.p.boxlen / coarse[0] / 2 ** lev, st, 1.5, 0.8, 1.4, smallr, smallc, 10)
    got, ref, p0 = [], [], []
    for ind in range(8):
        cc = s.ncoarse + ind * s.ngridmax + act - 1
        got.append(np.concatenate([uout[:, ind, slot], pout[:, ind, slot]]))
        ref.append(np.concatenate([unew.reshape(5, -1)[:, cc], divu[None, cc], enew[None, cc]]))
        p0.append(pstart[:, cc])
    return np.concatenate(got, axis=1), np.concatenate(ref, axis=1), np.concatenate(p0, axis=1)


def _assert_equal(got, ref, p0):
    assert np.isfinite(ref).all()
    assert np.abs(ref[5]).max() > 0 and not np.array_equal(ref[6], p0[1])   # divu and enew moved: the comparison is not vacuous
    assert np.array_equal(got, ref), [float(np.abs(got[n] - ref[n]).max()) for n in range(7)]


@pytest.mark.parametrize("gravity", [False, True], ids=["pfix", "grav+pfix"])
@pytest.mark.parametrize("coarse,lev,bound,solver,st,nblocks,scale", CASES)
def test_pfix_dense_sweep_amr_variant_emulated_equals_oracle(orc, pfix_dev, coarse, lev, bound, solver, st, nblocks, scale, gravity):
    """sweep_dense_kernel<3, ..., AMRV, GRAV, PFIX> on a base level with about a tenth of its cells marked refined, unew, divu and
    enew holding a finer level's refluxes: fluxes and tmp1 / tmp2 through refined faces reset, the state, divu and enew
    accumulated in godfine1's x, y, z order -- equal set_unew + godunov_fine of the oracle under orc_set_pressure_fix (and
    orc_set_gravity), bit for bit"""
    _assert_equal(*_run(orc, pfix_dev, coarse, lev, bound, solver, st, nblocks, scale, gravity))


@pytest.mark.parametrize("solver", ["llf", "exact", "acoustic", "hllc", "hll"])
def test_pfix_dense_sweep_every_solver(orc, pfix_dev, solver):
    """every solver's internal-energy flux (tmp2) through the PFIX form, on a periodic non-cubic box with the runtime slope switch"""
    _assert_equal(*_run(orc, pfix_dev, (3, 2, 1), 3, (0,) * 6, solver, 1, 3, 1.0, False, seed=5))


@pytest.mark.parametrize("floors", ["default", "raised"])
@pytest.mark.parametrize("solver,gravity", [("hllc", False), ("llf", True), ("exact", False)])
def test_pfix_dense_sweep_at_the_floors(orc, pfix_dev, floors, solver, gravity):
    """the PFIX form on a tree whose every cell holds a floor_state cell (helpers.fill_floor_state): ctoprim's density and
    internal-energy floors and the face-density resets fire under the traced states whose normal velocities make tmp1; state,
    divu and enew equal the oracle's bit for bit"""
    _assert_equal(*_run(orc, pfix_dev, (2, 2, 1), 3, (0,) * 6, solver, 1, 3, 1.0, gravity, floors=floors, seed=6))
