"""poisson in the dense sweep, on the CPU: the GRAV instantiation of sweep_dense_kernel (gravity predictor in ctoprim, the fused
add_gravity_source_terms and the gravity term of the fused Courant scan) compiled for the host by tests/host_numerics and run
by the emulated launch, compared with the oracle fed the same acceleration (orc_set_gravity) bit for bit."""
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
def grav_dev():
    """devnum_grav.cpp (devnum.cpp's emulated launch + the GRAV entry point) built for the host, the way devnum.cpp is built"""
    lib = os.path.join(HERE, "libdevnum_grav_host.so")
    srcs = [os.path.join(HERE, f) for f in ("devnum_grav.cpp", "devnum.cpp", os.path.join("stub", "cuda_runtime.h"))] + \
        [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    if not os.path.exists(lib) or os.path.getmtime(lib) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fno-fast-math", "-std=c++17", "-fPIC", "-shared", "-pthread",
                               "-fvisibility=hidden", "-fvisibility-inlines-hidden", "-Wl,-Bsymbolic",
                               "-I" + os.path.join(HERE, "stub"), "-I" + CSRC, "-I" + HERE, "-o", lib,
                               os.path.join(HERE, "devnum_grav.cpp")])
    L = C.CDLL(lib, mode=os.RTLD_LOCAL | os.RTLD_NOW)
    L.devnum_sweep_dense_grav_box.restype = C.c_int
    L.devnum_sweep_dense_grav_box.argtypes = [C.c_int, C.c_int, IP3, IP3, C.c_int, DP, DP, DP, C.c_int, C.POINTER(C.c_ubyte),
                                              C.c_double, C.c_double, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double,
                                              C.c_double, C.c_int, DP]
    return L


def force_field(ndim, ncell, amp, seed):
    """f[ndim][ncell]: a mean pull plus cell-to-cell noise on every cell of the tree (boundary octs included)"""
    rng = np.random.default_rng(seed)
    mean = np.array([0.8, -0.5, 0.3])[:ndim, None]
    return np.ascontiguousarray(amp * (mean + 0.4 * rng.standard_normal((ndim, ncell))))


class Gravity:
    """orc_set_gravity(f) for the duration of a with-block"""

    def __init__(self, f):
        from oracle import orc
        self.L, self.f = orc.lib(), f
        self.L.orc_set_gravity.argtypes = [DP]

    def __enter__(self):
        from oracle import orc
        self.L.orc_set_gravity(orc.dptr(self.f) if self.f is not None else None)

    def __exit__(self, *exc):
        self.L.orc_set_gravity(None)


def _oracle_level_step(c, f, gsrc):
    """courant (dt) -> set_unew -> godunov_fine (-> set_uold with the source term) of the oracle with acceleration f"""
    from oracle import orc
    with Gravity(f):
        dt, _ = c.oracle_courant()
        unew = c.oracle_godunov(dt, nthreads=1)
        if gsrc:
            uold = c.u.copy()
            orc.lib().orc_set_uold(C.byref(c.p), c.mesh.ptr, c.level, orc.dptr(uold), orc.dptr(unew))
            unew = uold
    return dt, unew


@pytest.mark.parametrize("ndim,coarse,level,bound,solver,st,nblocks,gsrc", [
    (1, (5, 1, 1), 3, (0,) * 6, "hllc", 2, 1, 1),                  # 40 cells, periodic
    (1, (5, 1, 1), 3, (1, 1, 0, 0, 0, 0), "exact", 1, 2, 0),       # 40 cells between walls
    (2, (3, 2, 1), 4, (0,) * 6, "llf", 8, 5, 1),                   # 48 x 32
    (2, (3, 2, 1), 4, (0, 0, 1, 1, 0, 0), "hll", 3, 3, 0),         # 48 x 32, walls in y
    (2, (1, 4, 1), 2, (0,) * 6, "acoustic", 7, 2, 1),              # 4 x 16
    (3, (3, 2, 1), 3, (0,) * 6, "hllc", 7, 4, 1),                  # 24 x 16 x 8
    (3, (1, 2, 3), 3, (2, 2, 0, 0, 0, 0), "hllc", 1, 5, 1),        # 8 x 16 x 24, outflow x
    (3, (8, 4, 1), 1, (0,) * 6, "hll", 2, 3, 1),                   # 16 x 8 x 2: 2-cell periodic z
    (3, (1, 4, 2), 2, (0,) * 6, "exact", 1, 2, 0),                 # 4 x 16 x 8: 4-cell periodic x
    (3, (3, 2, 1), 3, (1, 1, 0, 0, 0, 0), "acoustic", 3, 4, 1),    # 24 x 16 x 8, reflexive x walls
    (3, (3, 2, 1), 3, (0,) * 6, "llf", 8, 3, 0),
])
def test_gravity_dense_sweep_emulated_equals_oracle(orc, grav_dev, ndim, coarse, level, bound, solver, st, nblocks, gsrc):
    """sweep_dense_kernel<..., GRAV> on periodic boxes and boxes with a ghost shell, non-cubic domains and thin periodic axes: the
    owned cells equal set_unew + godunov_fine of the oracle with the same f (gsrc = 0: the predictor only, what
    rgpu_godunov_fine(_dev) returns), or that plus set_uold's source term (gsrc = 1, rgpu_level_steps), bit for bit.  With gsrc the
    fused Courant partials give the oracle's next dt with the gravity term, which differs from the dt without it."""
    from helpers import Case, box_state, level_slots
    c = Case(ndim, level, riemann=solver, slope_type=st, slope_theta=1.3, bound=bound, coarse=coarse, boxlen=float(coarse[0]),
             order=1, seed=2)
    ext = c.mesh.extent(level)
    c.init_dense(box_state(ndim, ext))
    s = c.mesh.s
    f = force_field(ndim, s.ncell, 40.0, 11 + ndim)
    dt, unew = _oracle_level_step(c, f, gsrc)
    _, unew_nograv = _oracle_level_step(c, None, gsrc)
    shell = [int(bound[2 * d] > 0) for d in range(3)]
    uin, act, slot = level_slots(c.mesh, level, c.u, ndim + 2)
    fin, _, _ = level_slots(c.mesh, level, f.ravel(), ndim)
    uout = np.zeros_like(uin)
    part = np.zeros(4 * 64)
    nb = grav_dev.devnum_sweep_dense_grav_box(ndim, SOLVER_ID[solver], IP3(*ext), IP3(*shell), nblocks, orc.dptr(uin), orc.dptr(uout),
                                              orc.dptr(fin), gsrc, None, dt, 2.0 ** -level, st, 1.3, 0.8, 1.4, 1e-10, 1e-10, 10,
                                              orc.dptr(part))
    T = 1 << ndim
    U, Ung = unew.reshape(ndim + 2, s.ncell), unew_nograv.reshape(ndim + 2, s.ncell)
    differs = False
    for ind in range(T):
        cells = s.ncoarse + ind * s.ngridmax + act - 1
        assert np.array_equal(uout[:, ind, slot], U[:, cells]), (ind, float(np.abs(uout[:, ind, slot] - U[:, cells]).max()))
        differs |= not np.array_equal(U[:, cells], Ung[:, cells])
    assert differs                                           # gravity changed the answer
    if gsrc:
        with Gravity(f):
            dt_next, sums = c.oracle_courant(unew)
        dt_nograv, _ = c.oracle_courant(unew)
        p4 = part[:4 * nb].reshape(4, nb)
        assert min(p4[0].min(), c.p.boxlen / c.p.smallc) == dt_next
        assert dt_next != dt_nograv
        vol = (2.0 ** -level) ** ndim
        assert abs(p4[1].sum() * vol - sums[0]) <= 1e-13 * abs(sums[0])


def test_gravity_limits_the_time_step(orc):
    """the acceleration of the cases above is strong enough that the gravity term of cmpdt, not the sound crossing, sets dt"""
    from helpers import Case, box_state
    c = Case(3, 3, riemann="hllc", slope_type=1, coarse=(3, 2, 1), boxlen=3.0, order=1, seed=2)
    c.init_dense(box_state(3, c.mesh.extent(3)))
    f = force_field(3, c.mesh.s.ncell, 40.0, 14)
    with Gravity(f):
        dt_g, _ = c.oracle_courant()
    dt_0, _ = c.oracle_courant()
    assert dt_g < 0.9 * dt_0


@pytest.mark.parametrize("coarse,bound,solver,nblocks", [((3, 2, 1), (0,) * 6, "hllc", 5), ((1, 2, 3), (2, 2, 0, 0, 0, 0), "exact", 7)])
def test_gravity_dense_sweep_amr_variant_emulated_equals_oracle(orc, grav_dev, coarse, bound, solver, nblocks):
    """sweep_dense_kernel<3, ..., AMRV, GRAV> on a base level with about a tenth of its cells marked refined: fluxes through
    refined faces reset, the update accumulated into a unew holding the finer level's refluxes, every flux with the gravity
    predictor -- equals set_unew + godunov_fine of the oracle with the same f, bit for bit"""
    from helpers import Case, box_state, level_slots
    lev = 4
    c = Case(3, lev, riemann=solver, slope_type=1, bound=bound, coarse=coarse, boxlen=float(coarse[0]), order=2, seed=8)
    ext = c.mesh.extent(lev)
    c.init_dense(box_state(3, ext))
    s = c.mesh.s
    f = force_field(3, s.ncell, 40.0, 21)
    act = c.mesh.active(lev).astype(np.int64)
    cells = np.concatenate([s.ncoarse + ind * s.ngridmax + act for ind in range(8)])        # 1-based
    son = c.mesh.son()
    rng = np.random.default_rng(3)
    ref_cells = cells[rng.random(len(cells)) < 0.1]
    son[ref_cells] = 1
    L = orc.lib()
    try:
        with Gravity(f):
            dt, _ = c.oracle_courant()
            unew = np.zeros_like(c.u)
            L.orc_set_unew(C.byref(c.p), c.mesh.ptr, lev, orc.dptr(c.u), orc.dptr(unew))
            U = unew.reshape(5, s.ncell)
            U[:, cells - 1] += 1e-3 * rng.standard_normal((5, len(cells))) * (son[cells] == 0)    # refluxes of a finer level
            start = unew.copy()
            L.orc_godunov_fine(C.byref(c.p), c.mesh.ptr, lev, dt, orc.dptr(c.u), orc.dptr(unew), 1)
    finally:
        son[ref_cells] = 0
    uin, act_, slot = level_slots(c.mesh, lev, c.u, 5)
    fin, _, _ = level_slots(c.mesh, lev, f.ravel(), 3)
    uout, _, _ = level_slots(c.mesh, lev, start, 5)
    refined = np.zeros(uin.shape[1:], dtype=np.uint8)
    for ind in range(8):
        refined[ind, slot] = np.isin(s.ncoarse + ind * s.ngridmax + act, ref_cells)
    assert refined.sum() == len(ref_cells) > 0
    shell = [int(bound[2 * d] > 0) for d in range(3)]
    grav_dev.devnum_sweep_dense_grav_box(3, SOLVER_ID[solver], IP3(*ext), IP3(*shell), nblocks, orc.dptr(uin), orc.dptr(uout),
                                         orc.dptr(fin), 0, refined.ctypes.data_as(C.POINTER(C.c_ubyte)), dt, 2.0 ** -lev, 1, 1.5,
                                         0.8, 1.4, 1e-10, 1e-10, 10, None)
    Un = unew.reshape(5, s.ncell)
    for ind in range(8):
        cc = s.ncoarse + ind * s.ngridmax + act - 1
        assert np.array_equal(uout[:, ind, slot], Un[:, cc]), (ind, float(np.abs(uout[:, ind, slot] - Un[:, cc]).max()))


@pytest.mark.parametrize("floors", ["default", "raised"])
@pytest.mark.parametrize("ndim,ext,solver,st,nblocks", [(1, (64, 1, 1), "hllc", 2, 2), (2, (32, 32, 1), "exact", 1, 3),
                                                       (3, (16, 16, 16), "llf", 8, 4), (3, (16, 16, 16), "hllc", 1, 3)])
def test_gravity_dense_sweep_emulated_at_the_floors(orc, grav_dev, floors, ndim, ext, solver, st, nblocks):
    """sweep_dense_kernel<..., GRAV> with the fused source term on a floor_state (densities below smallr, cold hypersonic cells,
    near-vacuum cells streamed out of) under the RAMSES floors and raised ones, with an acceleration strong enough that the
    predictor moves floored face densities: ctoprim's floors, the face resets after the gravity predictor and
    add_gravity_source_terms' d_old = max(uold, smallr) (hydro/godunov_fine.f90:267) all fire; the owned cells and the next dt
    equal the oracle's with the same f, bit for bit"""
    from helpers import FLOORS, Case, floor_counts, floor_state, level_slots
    smallr, smallc = FLOORS[floors]
    level = 4 if ndim == 3 else 5
    coarse = tuple(max(e >> level, 1) for e in ext)
    c = Case(ndim, level, riemann=solver, slope_type=st, slope_theta=1.3, coarse=coarse, boxlen=float(coarse[0]), order=1, seed=2,
             smallr=smallr, smallc=smallc)
    d0 = floor_state(ndim, c.mesh.extent(level), 31 + ndim, smallr, smallc)
    nrho, neint = floor_counts(d0, ndim, smallr, smallc)
    assert min(nrho, neint) >= max(2, 0.02 * d0[0].size), (nrho, neint)
    c.init_dense(d0)
    s = c.mesh.s
    f = force_field(ndim, s.ncell, 200.0, 17 + ndim)
    dt, unew = _oracle_level_step(c, f, 1)
    with Gravity(f):
        dt_next, sums = c.oracle_courant(unew)
    assert np.isfinite(unew).all() and np.isfinite(dt_next)
    uin, act, slot = level_slots(c.mesh, level, c.u, ndim + 2)
    fin, _, _ = level_slots(c.mesh, level, f.ravel(), ndim)
    uout = np.zeros_like(uin)
    part = np.zeros(4 * 64)
    nb = grav_dev.devnum_sweep_dense_grav_box(ndim, SOLVER_ID[solver], IP3(*c.mesh.extent(level)), IP3(0, 0, 0), nblocks, orc.dptr(uin),
                                              orc.dptr(uout), orc.dptr(fin), 1, None, dt, 2.0 ** -level, st, 1.3, 0.8, 1.4, smallr, smallc, 10,
                                              orc.dptr(part))
    U = unew.reshape(ndim + 2, s.ncell)
    for ind in range(1 << ndim):
        cells = s.ncoarse + ind * s.ngridmax + act - 1
        assert np.array_equal(uout[:, ind, slot], U[:, cells]), (ind, float(np.abs(uout[:, ind, slot] - U[:, cells]).max()))
    p4 = part[:4 * nb].reshape(4, nb)
    assert min(p4[0].min(), c.p.boxlen / c.p.smallc) == dt_next
