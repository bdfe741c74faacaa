"""Passive scalars on the GPU (NVAR = 6 and 7, NDIM = 3, AMR mode): the NPS = 1 and NPS = 2 instantiations of the oct-batch kernel,
the set_uold floor fix, upload_fine and the boundaries through the C-ABI, against the oracle bit for bit (`exact`: 1e-12, CUDA's
pow()).  Uniform levelmin = levelmax grids (every solver, slopes 0/1/2/3/7/8, walls and outflow), the nested tree with every
prolongation (host-driven amr_step and rgpu_amr_steps), the Level-0 drop-in on a 3-D adaptive run, floor states, and the
combinations rgpu_init refuses."""
import ctypes as C

import numpy as np
import pytest

from helpers import Case, max_rel_err, smooth_state

pytestmark = pytest.mark.gpu

EUNSUPPORTED = -3                 # RGPU_EUNSUPPORTED (include/ramses_gpu.h)


@pytest.fixture(scope="module")
def gpu():
    from ramses_b200 import lib
    lib.load()
    return lib


def _assert_close(got, ref, exact):
    assert np.isfinite(got).all()
    if exact:
        assert max_rel_err(got, ref) <= 1e-12
    else:
        assert np.array_equal(got, ref), float(np.abs(got - ref).max())


# (riemann, slope_type, nvar, bound): every solver with one and two scalars, slopes 0/1/2/3/7/8, walls in x / outflow in y or the
# other way round
UNIFORM_ROWS = [("llf", 0, 6, (1, 1, 2, 2, 0, 0)), ("llf", 3, 7, (2, 2, 1, 1, 0, 0)), ("hll", 1, 7, (1, 1, 2, 2, 0, 0)),
                ("hll", 7, 6, (2, 2, 1, 1, 0, 0)), ("hllc", 2, 6, (1, 1, 2, 2, 0, 0)), ("hllc", 8, 7, (2, 2, 1, 1, 0, 0)),
                ("acoustic", 3, 6, (1, 1, 2, 2, 0, 0)), ("acoustic", 1, 7, (2, 2, 1, 1, 0, 0)), ("exact", 2, 7, (1, 1, 2, 2, 0, 0)),
                ("exact", 8, 6, (2, 2, 1, 1, 0, 0))]


@pytest.mark.parametrize("riemann,slope_type,nvar,bound", UNIFORM_ROWS)
def test_scalars_uniform_grid_in_amr_mode(gpu, riemann, slope_type, nvar, bound):
    """a levelmin = levelmax 8^3 grid in AMR mode: three level steps in amr_step order (courant, set_unew, godunov_fine, set_uold
    with the floor fix, boundaries) == the oracle; the scalars moved"""
    from ramses_b200.hydro import HydroGPU
    n = 8
    u = np.zeros((nvar, n, n, n))
    u[:5] = smooth_state(3, n)
    x = (np.arange(n) + 0.5) / n
    u[5] = u[0] * (np.where(x > 0.5, 1.5, -0.5)[None, None, :] + 0.3 * np.sin(2 * np.pi * x)[None, :, None])
    if nvar > 6:
        u[6] = u[0] * (0.5 + 0.4 * np.cos(2 * np.pi * x))[:, None, None]
    c = Case(3, 3, riemann=riemann, slope_type=slope_type, nvar=nvar, bound=bound)
    c.init_dense(u)
    ref, dts_ref = c.oracle_steps(3)
    a = c.amr_commons()
    h = HydroGPU(a, amr_mode=True)
    for l in (1, 2, 3):
        h.bind_level(l)
    h.upload_state(0)
    h.make_boundary_hydro(3)
    dts = []
    for _ in range(3):
        a.dtnew[3] = a.boxlen / a.smallc
        dts.append(h.courant_fine(3))
        h.set_unew(3); h.godunov_fine_dev(3); h.set_uold(3); h.make_boundary_hydro(3)
    h.download_state(0)
    h.finalize()
    act = c.active_cells()
    ref = ref.reshape(nvar, -1)
    if riemann == "exact":
        assert np.allclose(dts, dts_ref, rtol=1e-12, atol=0)
    else:
        assert np.array_equal(np.array(dts), dts_ref)
    _assert_close(a.uold[:, act], ref[:, act], riemann == "exact")
    assert np.abs(ref[5:, act] - c.u.reshape(nvar, -1)[5:, act]).max() > 1e-4


def _nested_scalar_case(nvar, levelmin=4, levelmax=6):
    from ramses_b200.tree import build_nested_tree, cell_centers
    a = build_nested_tree(levelmin, levelmax, half_width=3, boxlen=1.0, nvar=nvar)
    a.gamma, a.courant_factor, a.slope_type, a.riemann = 1.4, 0.8, 1, "hllc"
    for l in range(levelmin, levelmax + 1):
        ig, cc = cell_centers(a, l)
        for ind in range(8):
            x, y, z = cc[ind][:, 0], cc[ind][:, 1], cc[ind][:, 2]
            r2 = (x - 0.5) ** 2 + (y - 0.5) ** 2 + (z - 0.5) ** 2
            u = np.zeros((nvar, len(x)))
            u[0] = 1.0 + 0.5 * np.exp(-r2 / 0.01)
            u[1] = 0.1 * u[0] * np.sin(2 * np.pi * y)
            u[3] = 0.05 * u[0] * np.cos(2 * np.pi * x)
            u[4] = (0.1 + 2.0 * np.exp(-r2 / 0.005)) / 0.4 + 0.5 * (u[1] ** 2 + u[3] ** 2) / u[0]
            u[5] = u[0] * (np.where(x < 0.5, 1.2, -0.3) + 0.1 * np.cos(2 * np.pi * x))
            if nvar > 6:
                u[6] = u[0] * np.exp(-r2 / 0.02)
            a.uold[:, a.ncoarse + ind * a.ngridmax + ig - 1] = u
    return a


def _nested_gpu(a, levelmin, levelmax, itype, ivar, resident=False, ncoarse=1):
    from ramses_b200.hydro import HydroGPU, amr_step
    h = HydroGPU(a, amr_mode=True, interpol_type=itype, interpol_var=ivar)
    for l in range(1, levelmax + 1):
        h.bind_level(l)
    h.upload_state(0)
    for l in range(levelmax - 1, 0, -1):
        h.upload_fine(l)
    h.download_state(0)
    u0 = a.uold.copy()
    nsub = [1] * (levelmin + 1) + [2] * 64
    if resident:
        dts = list(h.amr_steps(levelmin, nsub, ncoarse))
    else:
        dtnew = {l: 0.0 for l in range(0, levelmax + 2)}
        dtold = {l: 0.0 for l in range(0, levelmax + 2)}
        dts = []
        for _ in range(ncoarse):
            amr_step(h, levelmin, 1, levelmin, nsub, dtnew, dtold)
            dts.append(dtnew[levelmin])
    h.download_state(0)
    h.finalize()
    return u0, np.array(dts)


@pytest.mark.parametrize("nvar", [6, 7])
@pytest.mark.parametrize("itype,ivar", [(0, 0), (1, 0), (2, 1), (3, 2), (4, 2)])
def test_scalars_nested_tree_equal_oracle(gpu, itype, ivar, nvar):
    """the 3-level nested tree (prolongation of ghost octs incl. the coupled interpol_var 1 / 2 and interpol_type 4 path, coarse
    refluxing and upload_fine of all nvar variables, the patch-mode shell) driven by the host mirror of amr_step == the oracle's
    amr_step on the same arrays, bit for bit; the scalars moved"""
    from oracle.amr import AmrRun
    levelmin, levelmax = 4, 6
    a = _nested_scalar_case(nvar, levelmin, levelmax)
    u0, dts = _nested_gpu(a, levelmin, levelmax, itype, ivar)
    r = AmrRun(3, levelmin, levelmax, (0,) * 6, 1.0, nsubcycle=[1, 2, 2], ngridmax=a.ngridmax, riemann="hllc", slope_type=1,
               interpol_type=itype, interpol_var=ivar, tout=[1e9], nvar=nvar)
    r.uold[:] = u0.ravel()
    r.son[1:] = a.son; r.father[1:] = a.father; r.nbor[:, 1:] = a.nbor
    for l in range(1, levelmax + 1):
        r.active[l] = [int(g) for g in a.active[l]]
    r.push_all()
    r.static = True
    r.amr_step(levelmin, 1)
    ref = r.uold.reshape(nvar, -1)
    assert dts[0] == r.dtnew[levelmin]
    cells = np.concatenate([[a.ncoarse + ind * a.ngridmax + int(g) - 1 for g in a.active[l] for ind in range(8)] for l in range(1, levelmax + 1)])
    _assert_close(a.uold[:, cells], ref[:, cells], False)
    assert np.abs(a.uold[5:, cells] - u0[5:, cells]).max() > 1e-4


@pytest.mark.parametrize("nvar", [6, 7])
def test_scalars_amr_steps_device_resident_equal_host_driven(gpu, nvar):
    """rgpu_amr_steps with scalars (every time step on the device) == the host-driven amr_step sequence: the same dtnew(levelmin)
    and the same state over 2 coarse steps of the nested tree"""
    res = []
    for resident in (False, True):
        a = _nested_scalar_case(nvar)
        _, dts = _nested_gpu(a, 4, 6, 2, 1, resident=resident, ncoarse=2)
        res.append((dts, a.uold.copy()))
    assert (res[0][0] > 0).all()
    assert np.array_equal(res[0][0], res[1][0]), (res[0][0], res[1][0])
    assert np.array_equal(res[0][1], res[1][1])


@pytest.mark.parametrize("nvar", [6, 7])
def test_scalars_level0_dropin_equals_oracle(gpu, nvar):
    """the Level-0 drop-in (rgpu_godunov_fine behind the oracle's AMR driver, test_gpu_zz_golden.attach_gpu_godunov) on the 3-D
    scalar blast of the CPU drop-in test, regridding every coarse step: state, mesh and time equal the all-oracle run"""
    from test_gpu_zz_golden import attach_gpu_godunov
    from test_passive_scalars_host import scalar_blast_run
    runs = []
    for on_gpu in (False, True):
        r = scalar_blast_run(nvar)
        h = None
        if on_gpu:
            h, st = attach_gpu_godunov(r, riemann="hllc", slope_type=2, interpol_type=1)
        r.run(max_coarse=3)
        if h is not None:
            h.finalize()
            assert st["calls"] >= 3 * 3
        runs.append(r)
    a, b = runs
    assert a.t == b.t and a.nstep == b.nstep and a.t > 0
    assert np.array_equal(a.son, b.son) and np.array_equal(a.father, b.father) and np.array_equal(a.nbor, b.nbor)
    assert np.array_equal(a.uold, b.uold), float(np.abs(a.uold - b.uold).max())
    assert len(b.active[5]) > 0


@pytest.mark.parametrize("floors", ["default", "raised"])
@pytest.mark.parametrize("riemann,nscalar", [("hllc", 1), ("acoustic", 1), ("hll", 2), ("exact", 1)])
def test_scalars_at_the_floors(gpu, floors, riemann, nscalar):
    """a floor_state with one (and two) scalars on a 3x2x1 domain refined to level 3 in AMR mode: densities cross smallr in both
    directions, so both branches of amr_scalar_floor_kernel fire; 3 level steps equal the oracle"""
    from ramses_b200.hydro import HydroGPU
    from test_gpu_floors import _check, _floor_case, _oracle_steps
    level = 3
    c = _floor_case(3, level, (3, 2, 1), floors, riemann, 2, order=2, nscalar=nscalar)
    ref, dts_ref = _oracle_steps(c, 3)
    dt, _ = c.oracle_courant()
    one = c.oracle_godunov(dt, nthreads=8).reshape(c.nvar, -1)[0]
    old = c.u.reshape(c.nvar, -1)[0]
    idx = c.active_cells()
    assert ((old[idx] < c.p.smallr) & (one[idx] > old[idx])).sum() > 0
    assert ((one[idx] < c.p.smallr) & (old[idx] > one[idx])).sum() > 0
    a = c.amr_commons()
    h = HydroGPU(a, amr_mode=True)
    for l in range(1, level + 1):
        h.bind_level(l)
    h.upload_state(0)
    h.make_boundary_hydro(level)
    dts = []
    for _ in range(3):
        a.dtnew[level] = a.boxlen / a.smallc
        dts.append(h.courant_fine(level))
        h.set_unew(level); h.godunov_fine_dev(level); h.set_uold(level); h.make_boundary_hydro(level)
    h.download_state(0)
    h.finalize()
    _check(c, a.uold, np.array(dts), ref, dts_ref, exact=riemann == "exact")


@pytest.mark.parametrize("nvar", [6, 7])
@pytest.mark.parametrize("what", ["pressure_fix", "difmag"])
def test_scalars_rejected_combinations(gpu, what, nvar):
    """pressure_fix with scalars in AMR mode and difmag > 0 with scalars: rgpu_init answers RGPU_EUNSUPPORTED (launch_amr_godfine
    has no kernel for them, so a missing check would surface later as RGPU_ECUDA)"""
    from ramses_b200 import lib as _lib
    from ramses_b200.hydro import make_params
    L = _lib.load()
    a = Case(3, 3, nvar=nvar).amr_commons()
    if what == "pressure_fix":
        a.pressure_fix, a.beta_fix = True, 0.5
    else:
        a.difmag = 0.2
    p = make_params(a)
    assert L.rgpu_init(C.byref(p), 1, 1, 0) == EUNSUPPORTED
