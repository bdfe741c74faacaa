"""GPU parity on domains that are not one coarse cell refined to a cube: several coarse cells per axis (nx, ny, nz of AMR_PARAMS),
a different extent on every axis, thin periodic axes of 2 and 4 cells, ghost shells on one axis only, the boxes the multi-GPU
checks use as their single-GPU anchor, and a refined patch that is not a cube.  Every run goes through the C-ABI and is compared
with the oracle on the same arrays, bit for bit ('exact': 1e-12, CUDA pow vs libm pow).  A kernel that mixes up one axis's
extent with another's (tile counts, plane strides, cell decoding) gives the right answer on cubes and the wrong one here."""
import numpy as np
import pytest

from helpers import Case, MhdCase, box_state, max_rel_err, mhd_box_state

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu():
    from ramses_b200 import lib
    lib.load()
    return lib


def _box_case(ndim, level, coarse, riemann="hllc", slope_type=1, bound=(0,) * 6, order=1, seed=3, **kw):
    """Case on `coarse` domain cells with boxlen = coarse[0] (dx = 2^-level) holding a box_state: no symmetry hides a swapped axis"""
    c = Case(ndim, level, riemann=riemann, slope_type=slope_type, bound=bound, coarse=coarse, boxlen=float(coarse[0]), order=order,
             seed=seed, **kw)
    c.init_dense(box_state(ndim, c.mesh.extent(level), seed=seed))
    return c


def _level_steps(c, nstep, **attrs):
    from ramses_b200.hydro import HydroGPU
    a = c.amr_commons()
    for k, v in attrs.items():
        setattr(a, k, v)
    h = HydroGPU(a)
    h.bind_level(c.level)
    info = h.level_info(c.level)
    h.upload_state(c.level)
    dts, _ = h.level_steps(c.level, nstep)
    h.download_state(c.level)
    h.finalize()
    return a, np.asarray(dts), info


def _check(c, a, dts, ref, dts_ref, exact=False):
    idx = c.active_cells()
    nv = getattr(c, "nvs", c.nvar)
    ref = ref.reshape(nv, -1)
    assert np.abs(ref[:, idx] - c.u.reshape(nv, -1)[:, idx]).max() > 1e-4           # the state changed
    if exact:
        assert np.allclose(dts, dts_ref, rtol=1e-12, atol=0)
        assert max_rel_err(a.uold[:, idx], ref[:, idx]) <= 1e-12
    else:
        assert np.array_equal(dts, dts_ref), (dts, dts_ref)
        assert np.array_equal(a.uold[:, idx], ref[:, idx]), float(np.abs(a.uold[:, idx] - ref[:, idx]).max())


@pytest.mark.parametrize("coarse,level,riemann,slope_type,order", [
    ((3, 2, 1), 4, "hllc", 1, 0), ((1, 3, 2), 4, "llf", 2, 1), ((2, 1, 3), 4, "hll", 3, 2),
    ((3, 2, 1), 5, "acoustic", 7, 1), ((1, 3, 2), 5, "exact", 8, 2), ((2, 1, 3), 5, "hllc", 2, 0),
    ((3, 2, 1), 5, "exact", 1, 2), ((2, 1, 3), 4, "llf", 8, 1)])
def test_level_steps_on_non_cubic_boxes(gpu, coarse, level, riemann, slope_type, order):
    """rgpu_level_steps (3-D dense sweep, fused Courant scan) on 48x32x16 ... 64x32x96 periodic boxes: 8 steps, state and dt
    history equal the oracle's"""
    c = _box_case(3, level, coarse, riemann, slope_type, order=order)
    ref, dts_ref = c.oracle_steps(8, nthreads=8)
    a, dts, info = _level_steps(c, 8)
    ext = c.mesh.extent(level)
    assert info.dense == 1 and list(info.ncell_box)[:3] == list(ext)
    _check(c, a, dts, ref, dts_ref, exact=riemann == "exact")


@pytest.mark.parametrize("coarse", [(2, 1, 1), (2, 2, 1), (2, 2, 2)])
def test_multi_gpu_anchor_boxes_equal_oracle(gpu, coarse):
    """the single-GPU runs tests/mgpu_check.py compares every decomposed run with (coarse grid (2,1,1), (2,2,1), (2,2,2), level 5,
    mgpu_check.state_fn, 6 fused steps of hllc) equal the oracle: multi-GPU == single-GPU == oracle"""
    from mgpu_check import keys_and_state, state_fn
    from ramses_b200.hydro import HydroGPU
    from ramses_b200.tree import build_uniform_tree, fill_state
    level, steps = 5, 6
    g = build_uniform_tree(3, level, coarse=coarse, myid=1, ncpu=1, order="creation")
    g.riemann, g.slope_type, g.courant_factor = "hllc", 1, 0.8
    fill_state(g, level, state_fn(coarse))
    ext = [n << level for n in coarse]
    k0, u0 = keys_and_state(g, level)
    dense0 = np.zeros((5, ext[0] * ext[1] * ext[2]))
    dense0[:, k0] = u0
    h = HydroGPU(g)
    h.bind_level(level)
    h.upload_state(level)
    dts, _ = h.level_steps(level, steps)
    h.download_state(level)
    h.finalize()
    k1, u1 = keys_and_state(g, level)
    got = np.zeros_like(dense0)
    got[:, k1] = u1
    c = Case(3, level, riemann="hllc", slope_type=1, courant_factor=0.8, coarse=coarse, boxlen=1.0, order=0)
    c.init_dense(dense0.reshape(5, ext[2], ext[1], ext[0]))
    ref, dts_ref = c.oracle_steps(steps, nthreads=8)
    exp = c.dense(ref).reshape(5, -1)
    assert np.abs(exp - dense0).max() > 1e-4
    assert np.array_equal(np.asarray(dts), dts_ref)
    assert np.array_equal(got, exp)


@pytest.mark.parametrize("ndim,level,coarse,bound,riemann,slope_type", [
    (3, 4, (2, 1, 1), (1, 1, 0, 0, 0, 0), "hllc", 2),          # reflexive x walls, two domain cells in x
    (3, 4, (1, 1, 3), (0, 0, 0, 0, 2, 2), "llf", 1),           # outflow z faces, nz = 3
    (1, 5, (5, 1, 1), (0,) * 6, "hllc", 2),                    # 1-D, nx = 5: 160 cells
    (2, 4, (3, 2, 1), (0, 0, 1, 1, 0, 0), "hll", 3),           # 2-D 48 x 32, walls in y
    (3, 1, (8, 4, 1), (0,) * 6, "hllc", 1),                    # 16 x 8 x 2: 2-cell periodic z
    (3, 2, (4, 2, 1), (0,) * 6, "llf", 2),                     # 16 x 8 x 4: 4-cell periodic z
    (3, 1, (1, 4, 8), (0,) * 6, "hllc", 2),                    # 2 x 8 x 16: 2-cell periodic x
])
def test_boundaries_low_dimensions_and_thin_axes(gpu, ndim, level, coarse, bound, riemann, slope_type):
    """ghost shells on one axis of a non-cubic box, the 1-D and 2-D sweep_dense_kernel on several coarse cells, and periodic axes
    of 2 and 4 cells (halo and z ring wrap more than once): 8 fused steps equal the oracle"""
    c = _box_case(ndim, level, coarse, riemann, slope_type, bound=bound, order=2)
    ref, dts_ref = c.oracle_steps(8, nthreads=8)
    a, dts, info = _level_steps(c, 8)
    assert info.dense == 1
    _check(c, a, dts, ref, dts_ref)


@pytest.mark.parametrize("riemann", ["hllc", "exact"])
def test_level0_pipelined_equals_serial_and_oracle_on_box(gpu, monkeypatch, riemann):
    """rgpu_godunov_fine on host arrays of a 96x64x32 box in lattice order, z-slab pipeline with 3 slabs (does not divide the 16
    oct planes) and serial order: same bits as each other (every cell of the host arrays) and as the oracle"""
    from ramses_b200.hydro import HydroGPU
    monkeypatch.setenv("RGPU_E2E_SLABS", "3")
    c = _box_case(3, 5, (3, 2, 1), riemann, 1, order=1)
    dt, _ = c.oracle_courant()
    ref = c.oracle_godunov(dt, nthreads=8).reshape(c.nvar, -1)
    a = c.amr_commons()
    h = HydroGPU(a)
    h.bind_level(c.level)
    info = h.level_info(c.level)
    assert info.dense == 1 and info.pipeline_slabs == 3
    a.dtnew[c.level] = dt
    h.host_register(a.uold); h.host_register(a.unew)
    out = {}
    for mode in (1, 0):
        h.set_pipeline(mode)
        a.unew[:, :] = a.uold
        h.godunov_fine(c.level)
        out[mode] = a.unew.copy()
    h.host_unregister(a.uold); h.host_unregister(a.unew)
    h.finalize()
    idx = c.active_cells()
    assert np.abs(ref[:, idx] - c.u.reshape(c.nvar, -1)[:, idx]).max() > 1e-4
    assert np.array_equal(out[1], out[0])
    if riemann == "exact":
        assert max_rel_err(out[1][:, idx], ref[:, idx]) <= 1e-12
    else:
        assert np.array_equal(out[1][:, idx], ref[:, idx])


def test_fast_mode_on_box(gpu):
    """rgpu_params.fast = 1 on a 96x64x32 box: 12 steps within 1e-12 of the strict run and of the oracle"""
    c = _box_case(3, 5, (3, 2, 1), "hllc", 1, order=1)
    ref, dts_ref = c.oracle_steps(12, nthreads=8)
    ref = ref.reshape(c.nvar, -1)
    (as_, dts_s, _), (af, dts_f, _) = _level_steps(c, 12, fast=False), _level_steps(c, 12, fast=True)
    idx = c.active_cells()
    us, uf = as_.uold[:, idx], af.uold[:, idx]
    assert np.array_equal(us, ref[:, idx]) and np.array_equal(dts_s, dts_ref)
    assert not np.array_equal(us, uf)
    assert max_rel_err(uf, us) <= 1e-12 and max_rel_err(uf, ref[:, idx]) <= 1e-12
    assert np.allclose(dts_f, dts_ref, rtol=1e-12, atol=0)


@pytest.mark.parametrize("coarse,level,bound,riemann,riemann2d,slope_type", [
    ((3, 2, 1), 4, (0,) * 6, "roe", "llf", 1),
    ((3, 2, 1), 4, (0,) * 6, "hlld", "hlld", 2),
    ((1, 2, 1), 4, (2, 2, 0, 0, 0, 0), "hlld", "hlld", 1),     # zero-gradient x ends (xbound)
    ((8, 4, 1), 1, (0,) * 6, "hlld", "hlld", 2),               # 16 x 8 x 2: 2-cell periodic z
])
def test_mhd_six_pass_sweep_on_non_cubic_boxes(gpu, coarse, level, bound, riemann, riemann2d, slope_type):
    """the dense MHD sweep (W[..][ncz][ncy][ncx], cells decoded with ncx / ncy) on 48x32x16, 16x32x16 and 16x8x2 boxes: 4 fused
    steps equal the oracle, both copies of every face field included"""
    c = MhdCase(level, riemann=riemann, riemann2d=riemann2d, slope_type=slope_type, bound=bound, coarse=coarse,
                boxlen=float(coarse[0]), order=1)
    d0 = mhd_box_state(c.mesh.extent(level))
    d0[0] *= 1 + 0.2 * (np.random.default_rng(4).standard_normal(d0[0].shape) > 1.3)
    c.init_dense(d0)
    ref, dts_ref = c.oracle_steps(4, nthreads=8)
    a, dts, info = _level_steps(c, 4)
    assert info.dense == 1
    _check(c, a, dts, ref, dts_ref)


@pytest.mark.parametrize("dense", ["0", "1"])
@pytest.mark.parametrize("level", [1, 2, 4])
def test_amr_mode_uniform_box_level(gpu, monkeypatch, level, dense):
    """AMR mode (rgpu_set_amr) on a uniform 3x2x1 domain refined to `level`, swept by the oct-batch kernel (RGPU_AMR_DENSE=0) and by
    the dense AMR variant: 3 level steps in amr_step order equal the oracle.  At level 1 the oct-batch kernel finds the 27
    neighbouring father cells of every oct by decoding coarse cells with nx, ny, nz (the level-1 branch of get3cubefather); at
    level 2 through the level-1 octs of the neighbouring coarse cells.  level_info reports which kernel swept the level."""
    from ramses_b200.hydro import HydroGPU
    monkeypatch.setenv("RGPU_AMR_DENSE", dense)
    c = _box_case(3, level, (3, 2, 1), "hllc", 2, bound=(0,) * 6, order=2)
    ref, dts_ref = c.oracle_steps(3, nthreads=8)
    a = c.amr_commons()
    h = HydroGPU(a, amr_mode=True)
    for l in range(1, level + 1):
        h.bind_level(l)
    info = h.level_info(level)
    assert info.dense == int(dense)
    if info.dense:
        assert list(info.ncell_box) == list(c.mesh.extent(level)) and list(info.wrap) == [1, 1, 1]
    h.upload_state(0)
    h.make_boundary_hydro(level)
    dts = []
    for _ in range(3):
        a.dtnew[level] = a.boxlen / a.smallc
        dts.append(h.courant_fine(level))
        h.set_unew(level); h.godunov_fine_dev(level); h.set_uold(level); h.make_boundary_hydro(level)
    h.download_state(0)
    h.finalize()
    _check(c, a, np.array(dts), ref, dts_ref)


def test_nested_non_cubic_patch_matches_oracle(gpu, monkeypatch):
    """a nested tree whose two refined levels are 12x6x8-oct boxes, driven by the host amr_step, == the oracle's amr_step on the
    same arrays, both in patch mode (dense kernel on the box + prolongated shell, surface octs refluxed by the oct-batch kernel)
    and with patch mode switched off (RGPU_AMR_PATCH=0: oct-batch kernel); level_info reports which kernel swept each level"""
    from oracle.amr import AmrRun
    from ramses_b200.hydro import HydroGPU, amr_step
    from ramses_b200.tree import build_nested_tree, cell_centers
    levelmin, levelmax = 4, 6

    def ic(x, y, z):          # off-centre blast inside the refined box, waves of different lengths per axis
        r2 = ((x - 0.55) / 1.5) ** 2 + ((y - 0.48) / 0.8) ** 2 + (z - 0.52) ** 2
        u = np.zeros((5, len(x)))
        u[0] = 1.0 + 0.5 * np.exp(-r2 / 0.01) + 0.1 * np.sin(2 * np.pi * z)
        u[1] = 0.1 * u[0] * np.sin(2 * np.pi * y)
        u[2] = -0.05 * u[0] * np.cos(4 * np.pi * x)
        u[4] = (0.1 + 2.0 * np.exp(-r2 / 0.005)) / 0.4 + 0.5 * (u[1] ** 2 + u[2] ** 2) / u[0]
        return u

    def run_gpu():
        a = build_nested_tree(levelmin, levelmax, half_width=(6, 3, 4))
        assert [len(a.active[l]) for l in (5, 6)] == [12 * 6 * 8] * 2
        a.gamma, a.courant_factor, a.slope_type, a.riemann = 1.4, 0.8, 1, "hllc"
        for l in range(levelmin, levelmax + 1):
            ig, cc = cell_centers(a, l)
            for ind in range(8):
                a.uold[:, a.ncoarse + ind * a.ngridmax + ig - 1] = ic(cc[ind][:, 0], cc[ind][:, 1], cc[ind][:, 2])
        h = HydroGPU(a, amr_mode=True)
        for l in range(1, levelmax + 1):
            h.bind_level(l)
        h.upload_state(0)
        for l in range(levelmax - 1, 0, -1):
            h.upload_fine(l)
        nsub = [1] * (levelmin + 1) + [2] * 64
        nsub[levelmin - 1] = 1
        dtnew = {l: 0.0 for l in range(0, levelmax + 2)}
        dtold = {l: 0.0 for l in range(0, levelmax + 2)}
        h.download_state(0)
        u0 = a.uold.copy()
        amr_step(h, levelmin, 1, levelmin, nsub, dtnew, dtold)
        h.download_state(0)
        dense = [h.level_info(l).dense for l in (4, 5, 6)]
        h.finalize()
        return a, u0, dtnew, dense

    a, u0, dtnew, dense = run_gpu()
    monkeypatch.setenv("RGPU_AMR_PATCH", "0")
    b, u0b, dtnew_b, dense_b = run_gpu()
    assert np.array_equal(u0, u0b)
    assert dense == [1, 1, 1] and dense_b == [1, 0, 0]          # base box dense in both runs, the patches only in the first
    r = AmrRun(3, levelmin, levelmax, (0,) * 6, 1.0, nsubcycle=[1, 2, 2], ngridmax=a.ngridmax, riemann="hllc", slope_type=1,
               tout=[1e9])
    assert r.ncell == a.ncell
    r.son[1:] = a.son; r.father[1:] = a.father; r.nbor[:, 1:] = a.nbor
    for l in range(1, levelmax + 1):
        r.active[l] = [int(g) for g in a.active[l]]
    r.push_all()
    r.uold[:] = u0.ravel()
    r.static = True
    r.amr_step(levelmin, 1)
    ref = r.uold.reshape(5, -1)
    cells = np.concatenate([[a.ncoarse + ind * a.ngridmax + int(g) - 1 for g in a.active[l] for ind in range(8)]
                            for l in range(1, levelmax + 1)])
    assert np.abs(ref[:, cells] - u0[:, cells]).max() > 1e-4
    for got, dt in ((a.uold, dtnew), (b.uold, dtnew_b)):
        assert dt[levelmin] == r.dtnew[levelmin]
        assert np.array_equal(got[:, cells], ref[:, cells]), float(np.abs(got[:, cells] - ref[:, cells]).max())
