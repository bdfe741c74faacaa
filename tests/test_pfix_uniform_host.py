"""pressure_fix on a levelmin=levelmax level, on the CPU: the plain PFIX instantiations of sweep_dense_kernel (1-D, 2-D and 3-D)
and the dense set_unew / set_uold passes of a level store (divu / enew initialisation, the pdV source from the face neighbours,
the energy switch) compiled for the host by tests/host_numerics and run by the emulated launch, compared with set_unew +
godunov_fine + set_uold of the oracle under orc_set_pressure_fix, bit for bit."""
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
def plain_dev():
    """devnum_pfix_plain.cpp (devnum.cpp's emulated launch + the level-step entry point) built for the host like devnum.cpp"""
    lib = os.path.join(HERE, "libdevnum_pfix_plain_host.so")
    srcs = [os.path.join(HERE, f) for f in ("devnum_pfix_plain.cpp", "devnum.cpp", os.path.join("stub", "cuda_runtime.h"))] + \
        [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    if not os.path.exists(lib) or os.path.getmtime(lib) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fno-fast-math", "-std=c++17", "-fPIC", "-shared", "-pthread",
                               "-fvisibility=hidden", "-fvisibility-inlines-hidden", "-Wl,-Bsymbolic",
                               "-I" + os.path.join(HERE, "stub"), "-I" + CSRC, "-I" + HERE, "-o", lib,
                               os.path.join(HERE, "devnum_pfix_plain.cpp")])
    L = C.CDLL(lib, mode=os.RTLD_LOCAL | os.RTLD_NOW)
    L.devnum_pfix_plain_step.restype = C.c_int
    L.devnum_pfix_plain_step.argtypes = [C.c_int, C.c_int, IP3, IP3, C.c_int, DP, DP, DP, C.c_double, C.c_double, C.c_int, C.c_double,
                                         C.c_double, C.c_double, C.c_double, C.c_double, C.c_int, C.c_double, DP]
    return L


def _oracle_step(c, beta_fix):
    """courant (dt) -> set_unew -> godunov_fine -> set_uold of the oracle; beta_fix None: without pressure_fix.  Returns dt, the new
    state and divu / enew (zeros without pressure_fix)"""
    from oracle import orc
    L = orc.lib()
    L.orc_set_pressure_fix.argtypes = [DP, DP, C.c_double]
    n = c.mesh.s.ncell
    divu, enew = np.zeros(n), np.zeros(n)
    if beta_fix is not None:
        L.orc_set_pressure_fix(orc.dptr(divu), orc.dptr(enew), beta_fix)
    try:
        dt, _ = c.oracle_courant()
        unew = c.oracle_godunov(dt, nthreads=1)
        uold = c.u.copy()
        L.orc_set_uold(C.byref(c.p), c.mesh.ptr, c.level, orc.dptr(uold), orc.dptr(unew))
    finally:
        L.orc_set_pressure_fix(None, None, 0.0)
    return dt, uold, divu, enew


def _run(orc, plain_dev, ndim, coarse, level, bound, solver, st, nblocks, scale, beta_fix=0.5, floors=None, seed=2):
    """one level step on the emulated device and on the oracle; returns (device [nvar+2][cells], oracle [nvar+2][cells], the oracle's
    state without pressure_fix [nvar][cells]) over the active cells"""
    from helpers import FLOORS, Case, box_state, fill_floor_state, level_slots
    smallr, smallc = FLOORS[floors] if floors else (1e-10, 1e-10)
    c = Case(ndim, level, riemann=solver, slope_type=st, slope_theta=1.3, bound=bound, coarse=coarse, boxlen=scale * coarse[0],
             order=1, seed=seed, smallr=smallr, smallc=smallc)
    ext = c.mesh.extent(level)
    c.init_dense(box_state(ndim, ext, seed=seed))
    s = c.mesh.s
    nv = ndim + 2
    if floors:
        fill_floor_state(c.u, ndim, nv, s.ncell, floors, 40 + seed)
        orc.lib().orc_make_boundary_hydro(C.byref(c.p), c.mesh.ptr, level, orc.dptr(c.u))
    dt, ref, divu, enew = _oracle_step(c, beta_fix)
    _, ref_plain, _, _ = _oracle_step(c, None)
    uin, act, slot = level_slots(c.mesh, level, c.u, nv)
    uout = np.zeros_like(uin)
    pfix = np.full((2,) + uin.shape[1:], np.nan)
    shell = [int(bound[2 * d] > 0) for d in range(3)]
    plain_dev.devnum_pfix_plain_step(ndim, SOLVER_ID[solver], IP3(*ext), IP3(*shell), nblocks, orc.dptr(uin), orc.dptr(uout),
                                     orc.dptr(pfix), dt, c.p.boxlen / coarse[0] / 2 ** level, st, 1.3, 0.8, 1.4, smallr, smallc, 10,
                                     beta_fix, None)
    got, want, plain = [], [], []
    R, Rp = ref.reshape(nv, -1), ref_plain.reshape(nv, -1)
    for ind in range(1 << ndim):
        cc = s.ncoarse + ind * s.ngridmax + act - 1
        got.append(np.concatenate([uout[:, ind, slot], pfix[:, ind, slot]]))
        want.append(np.concatenate([R[:, cc], divu[None, cc], enew[None, cc]]))
        plain.append(Rp[:, cc])
    return np.concatenate(got, axis=1), np.concatenate(want, axis=1), np.concatenate(plain, axis=1)


def _assert_equal(got, want):
    nv = got.shape[0] - 2
    assert np.isfinite(want).all()
    assert np.abs(want[nv]).max() > 0                        # divu moved: the comparison is not vacuous
    assert np.array_equal(got, want), [float(np.abs(got[n] - want[n]).max()) for n in range(nv + 2)]


CASES = [   # ndim, coarse, level, bound, solver, slope_type, nblocks, scale (boxlen / coarse[0]: 1 = power-of-two dx)
    (1, (5, 1, 1), 3, (0,) * 6, "hllc", 2, 1, 1.0),                  # 40 cells, periodic
    (1, (5, 1, 1), 3, (1, 1, 0, 0, 0, 0), "exact", 1, 2, 0.75),      # 40 cells between walls, dx not a power of two
    (1, (3, 1, 1), 4, (2, 2, 0, 0, 0, 0), "llf", 8, 3, 1.0),         # 48 cells, outflow
    (2, (3, 2, 1), 4, (0,) * 6, "llf", 8, 5, 1.0),                   # 48 x 32, periodic
    (2, (3, 2, 1), 4, (0, 0, 1, 1, 0, 0), "hll", 3, 3, 3.0),         # 48 x 32, walls in y
    (2, (1, 4, 1), 2, (2, 2, 0, 0, 0, 0), "acoustic", 7, 2, 1.0),    # 4 x 16, outflow x
    (2, (8, 1, 1), 1, (0,) * 6, "hllc", 1, 1, 0.75),                 # 16 x 2: 2-cell periodic y
    (3, (3, 2, 1), 3, (0,) * 6, "hllc", 7, 4, 1.0),                  # 24 x 16 x 8
    (3, (1, 2, 3), 3, (2, 2, 0, 0, 0, 0), "exact", 2, 5, 1.0),       # 8 x 16 x 24, outflow x
    (3, (8, 4, 1), 1, (0,) * 6, "hll", 8, 3, 1.0),                   # 16 x 8 x 2: 2-cell periodic z
    (3, (3, 2, 1), 3, (1, 1, 0, 0, 0, 0), "acoustic", 3, 4, 0.75),   # 24 x 16 x 8, reflexive x walls, dx not a power of two
    (3, (1, 4, 2), 2, (0, 0, 0, 0, 1, 1), "llf", 1, 2, 3.0),         # 4 x 16 x 8, walls in z
]


@pytest.mark.parametrize("ndim,coarse,level,bound,solver,st,nblocks,scale", CASES)
def test_pfix_plain_level_step_emulated_equals_oracle(orc, plain_dev, ndim, coarse, level, bound, solver, st, nblocks, scale):
    """set_unew's divu / enew, sweep_dense_kernel<..., PFIX> (plain form: the state from uin, tmp1 / tmp2 of every face into divu /
    enew), set_uold's pdV source from the face neighbours in uold (shell and periodic images included) and the energy switch on the
    new state -- equal set_unew + godunov_fine + set_uold of the oracle under orc_set_pressure_fix in state, divu and enew, bit for
    bit, on periodic boxes, walls and outflow, non-cubic domains and 2-cell periodic axes"""
    got, want, _ = _run(orc, plain_dev, ndim, coarse, level, bound, solver, st, nblocks, scale)
    _assert_equal(got, want)


@pytest.mark.parametrize("ndim", [1, 2, 3])
@pytest.mark.parametrize("solver", ["llf", "exact", "acoustic", "hllc", "hll"])
def test_pfix_plain_every_solver(orc, plain_dev, ndim, solver):
    """every solver's internal-energy flux (tmp2) through the plain PFIX form in each dimension, periodic non-cubic boxes"""
    coarse = {1: (6, 1, 1), 2: (3, 2, 1), 3: (3, 2, 1)}[ndim]
    got, want, _ = _run(orc, plain_dev, ndim, coarse, {1: 3, 2: 3, 3: 2}[ndim], (0,) * 6, solver, 1, 3, 1.0, seed=5)
    _assert_equal(got, want)


@pytest.mark.parametrize("ndim,ext_coarse,level,solver", [(1, (6, 1, 1), 3, "hllc"), (2, (2, 2, 1), 3, "llf"),
                                                          (3, (2, 2, 1), 2, "exact")])
def test_pfix_plain_at_the_raised_floors_switch_fires(orc, plain_dev, ndim, ext_coarse, level, solver):
    """a tree whose every cell holds a floor_state cell under the raised floors (cold hypersonic cells, near-vacuum neighbours):
    the energy switch replaces the total energy in some cells and keeps it in others, on the oracle and on the emulated device
    alike, bit for bit"""
    got, want, plain = _run(orc, plain_dev, ndim, ext_coarse, level, (0,) * 6, solver, 1, 2, 1.0, floors="raised", seed=6)
    _assert_equal(got, want)
    nv = ndim + 2
    assert np.array_equal(want[:nv - 1], plain[:nv - 1])     # the switch touches the total energy only
    fired = want[nv - 1] != plain[nv - 1]
    assert 0 < fired.sum() < fired.size, (int(fired.sum()), fired.size)


@pytest.mark.parametrize("ndim,coarse,level,solver", [(1, (5, 1, 1), 3, "hll"), (2, (3, 2, 1), 3, "hllc"), (3, (3, 2, 1), 2, "llf")])
def test_pfix_plain_beta_fix_zero_keeps_the_state(orc, plain_dev, ndim, coarse, level, solver):
    """beta_fix = 0: the truncation error is zero, the switch never fires on these states, and the new state equals the run
    without pressure_fix; divu and enew still equal the oracle's"""
    got, want, plain = _run(orc, plain_dev, ndim, coarse, level, (0,) * 6, solver, 2, 2, 1.0, beta_fix=0.0)
    _assert_equal(got, want)
    assert np.array_equal(got[:ndim + 2], plain)
