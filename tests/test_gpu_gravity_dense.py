"""poisson through the dense sweep on the GPU: levelmin=levelmax levels (rgpu_level_steps, the split Level-1 sequence, the Level-0
call on host arrays, FAST mode) and the dense base box and refined patch of AMR mode, every run compared with the oracle fed the
same acceleration f (orc_set_gravity), bit for bit ('exact': 1e-12, CUDA pow vs libm pow)."""
import ctypes as C

import numpy as np
import pytest

from helpers import Case, box_state, max_rel_err

pytestmark = pytest.mark.gpu

EINVAL, EUNSUPPORTED = -1, -3         # RGPU_EINVAL, RGPU_EUNSUPPORTED (include/ramses_gpu.h)


@pytest.fixture(scope="module")
def gpu():
    from ramses_b200 import lib
    lib.load()
    return lib


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
        self.L.orc_set_gravity.argtypes = [C.POINTER(C.c_double)]

    def __enter__(self):
        from oracle import orc
        self.L.orc_set_gravity(orc.dptr(self.f))

    def __exit__(self, *exc):
        self.L.orc_set_gravity(None)


def _box_case(ndim, level, coarse, riemann="hllc", slope_type=1, bound=(0,) * 6, order=1, seed=3):
    c = Case(ndim, level, riemann=riemann, slope_type=slope_type, bound=bound, coarse=coarse, boxlen=float(coarse[0]), order=order,
             seed=seed)
    c.init_dense(box_state(ndim, c.mesh.extent(level), seed=seed))
    return c


def _check(c, got, dts, ref, dts_ref, exact=False):
    idx = c.active_cells()
    ref = ref.reshape(c.nvar, -1)
    assert np.abs(ref[:, idx] - c.u.reshape(c.nvar, -1)[:, idx]).max() > 1e-4
    if exact:
        assert np.allclose(dts, dts_ref, rtol=1e-12, atol=0)
        assert max_rel_err(got[:, idx], ref[:, idx]) <= 1e-12
    else:
        assert np.array_equal(dts, dts_ref), (dts, dts_ref)
        assert np.array_equal(got[:, idx], ref[:, idx]), float(np.abs(got[:, idx] - ref[:, idx]).max())


def _gpu_level_steps(c, f, nstep, **attrs):
    from ramses_b200.hydro import HydroGPU
    a = c.amr_commons()
    a.poisson = True
    for k, v in attrs.items():
        setattr(a, k, v)
    h = HydroGPU(a)
    h.bind_level(c.level)
    info = h.level_info(c.level)
    h.upload_state(c.level)
    h.upload_force(f)
    dts, _ = h.level_steps(c.level, nstep)
    h.download_state(c.level)
    h.finalize()
    return a, np.asarray(dts), info


@pytest.mark.parametrize("ndim,coarse,level,bound,riemann,slope_type", [
    (1, (5, 1, 1), 5, (0,) * 6, "hllc", 2),                     # 160 cells, periodic
    (1, (5, 1, 1), 5, (1, 1, 0, 0, 0, 0), "exact", 1),          # walls
    (2, (3, 2, 1), 4, (0, 0, 1, 1, 0, 0), "hll", 3),            # 48 x 32, walls in y
    (2, (3, 2, 1), 4, (2, 2, 0, 0, 0, 0), "llf", 8),            # outflow x
    (3, (3, 2, 1), 4, (0,) * 6, "hllc", 1),                     # 48 x 32 x 16
    (3, (1, 3, 2), 4, (0,) * 6, "acoustic", 7),                 # 16 x 48 x 32
    (3, (2, 1, 1), 4, (1, 1, 0, 0, 0, 0), "exact", 2),          # reflexive x walls
    (3, (1, 1, 3), 4, (0, 0, 0, 0, 2, 2), "llf", 3),            # outflow z faces
    (3, (8, 4, 1), 1, (0,) * 6, "hll", 8),                      # 16 x 8 x 2: 2-cell periodic z
])
def test_level_steps_with_gravity(gpu, ndim, coarse, level, bound, riemann, slope_type):
    """rgpu_level_steps with poisson (predictor in the sweep, source term and gravity-limited Courant scan fused): 6 steps with a
    fixed f equal orc_run_uniform with orc_set_gravity(f); the level runs on the dense kernel, in 3-D the round-1 form"""
    c = _box_case(ndim, level, coarse, riemann, slope_type, bound=bound, order=2)
    f = force_field(ndim, c.mesh.s.ncell, 20.0, 5 + ndim)
    with Gravity(f):
        ref, dts_ref = c.oracle_steps(6, nthreads=8)
    ref0, dts0 = c.oracle_steps(6, nthreads=8)
    assert not np.array_equal(dts_ref, dts0)                  # gravity changes the time steps
    a, dts, info = _gpu_level_steps(c, f, 6)
    assert info.dense == 1 and info.sweep_variant == 0
    _check(c, a.uold, dts, ref, dts_ref, exact=riemann == "exact")


def test_fast_flag_with_gravity_gives_the_strict_bits(gpu):
    """fast = 1 does not apply to poisson: the level binds the round-1 kernel and gives the strict result"""
    c = _box_case(3, 4, (3, 2, 1), "hllc", 1)
    f = force_field(3, c.mesh.s.ncell, 20.0, 8)
    with Gravity(f):
        ref, dts_ref = c.oracle_steps(6, nthreads=8)
    a, dts, info = _gpu_level_steps(c, f, 6, fast=True)
    assert info.sweep_variant == 0
    _check(c, a.uold, dts, ref, dts_ref)


@pytest.mark.parametrize("ndim,coarse,level,bound,riemann,slope_type", [
    (1, (5, 1, 1), 5, (1, 1, 0, 0, 0, 0), "hllc", 1),
    (2, (3, 2, 1), 4, (0,) * 6, "exact", 2),
    (3, (3, 2, 1), 4, (0, 0, 0, 0, 2, 2), "hllc", 2),
])
def test_split_sequence_with_new_force_every_step(gpu, ndim, coarse, level, bound, riemann, slope_type):
    """courant -> set_unew -> godunov_fine_dev -> set_uold -> make_boundary_hydro with a new f uploaded before every step (a
    self-gravity host loop): equals the oracle's split sequence fed the same sequence of f"""
    from oracle import orc
    from ramses_b200.hydro import HydroGPU
    c = _box_case(ndim, level, coarse, riemann, slope_type, bound=bound, order=1)
    fs = [force_field(ndim, c.mesh.s.ncell, 20.0, 30 + s) for s in range(3)]
    L = orc.lib()
    u = c.u.copy()
    unew = np.zeros_like(u)
    dts_ref = []
    for f in fs:
        with Gravity(f):
            dt = L.orc_courant_fine(C.byref(c.p), c.mesh.ptr, c.level, c.p.boxlen / c.p.smallc, orc.dptr(u), orc.dptr(np.zeros(3)))
            L.orc_set_unew(C.byref(c.p), c.mesh.ptr, c.level, orc.dptr(u), orc.dptr(unew))
            L.orc_godunov_fine(C.byref(c.p), c.mesh.ptr, c.level, dt, orc.dptr(u), orc.dptr(unew), 8)
            L.orc_set_uold(C.byref(c.p), c.mesh.ptr, c.level, orc.dptr(u), orc.dptr(unew))
            L.orc_make_boundary_hydro(C.byref(c.p), c.mesh.ptr, c.level, orc.dptr(u))
        dts_ref.append(dt)
    a = c.amr_commons()
    a.poisson = True
    h = HydroGPU(a)
    h.bind_level(c.level)
    h.upload_state(c.level)
    dts = []
    for f in fs:
        h.upload_force(f)
        a.dtnew[c.level] = a.boxlen / a.smallc
        dts.append(h.courant_fine(c.level))
        h.set_unew(c.level); h.godunov_fine_dev(c.level); h.set_uold(c.level); h.make_boundary_hydro(c.level)
    h.download_state(c.level)
    h.finalize()
    _check(c, a.uold, np.array(dts), u, np.array(dts_ref), exact=riemann == "exact")


@pytest.mark.parametrize("riemann", ["hllc", "exact"])
def test_level0_godunov_fine_with_gravity(gpu, monkeypatch, riemann):
    """rgpu_godunov_fine on host arrays with poisson returns uold + dF with the gravity predictor and without the source term
    (the host's set_uold adds it): equals orc_godunov_fine with the same f, in serial and slab-pipelined order"""
    from ramses_b200.hydro import HydroGPU
    monkeypatch.setenv("RGPU_E2E_SLABS", "3")
    c = _box_case(3, 5, (3, 2, 1), riemann, 1, order=1)
    f = force_field(3, c.mesh.s.ncell, 20.0, 41)
    with Gravity(f):
        dt, _ = c.oracle_courant()
        ref = c.oracle_godunov(dt, nthreads=8).reshape(c.nvar, -1)
    nograv = c.oracle_godunov(dt, nthreads=8).reshape(c.nvar, -1)
    a = c.amr_commons()
    a.poisson = True
    h = HydroGPU(a)
    h.bind_level(c.level)
    info = h.level_info(c.level)
    assert info.dense == 1 and info.pipeline_slabs == 3
    h.upload_force(f)
    a.dtnew[c.level] = dt
    out = {}
    for mode in (1, 0):
        h.set_pipeline(mode)
        a.unew[:, :] = a.uold
        h.godunov_fine(c.level)
        out[mode] = a.unew.copy()
    h.finalize()
    idx = c.active_cells()
    assert not np.array_equal(ref[:, idx], nograv[:, idx])
    assert np.array_equal(out[1], out[0])
    if riemann == "exact":
        assert max_rel_err(out[1][:, idx], ref[:, idx]) <= 1e-12
    else:
        assert np.array_equal(out[1][:, idx], ref[:, idx])


def test_rejected_combinations_and_missing_force(gpu):
    """poisson with pressure_fix outside AMR mode, with passive scalars, with difmag and in the MHD build: RGPU_EUNSUPPORTED; a
    gravity sweep or Courant scan before any rgpu_upload_force: RGPU_EINVAL"""
    from ramses_b200 import lib as _lib
    from ramses_b200.hydro import HydroGPU, _level_lists, make_params
    L = _lib.load()
    c = _box_case(3, 3, (1, 1, 1), "hllc", 1)
    a = c.amr_commons()
    a.poisson, a.pressure_fix, a.beta_fix = True, True, 0.5
    h = HydroGPU(a)
    keep = []
    assert L.rgpu_bind_level(c.level, *_level_lists(a, c.level, keep)) == EUNSUPPORTED
    h.finalize()
    for attrs in (dict(nvar=6), dict(difmag=0.1)):
        b = Case(3, 3, nvar=attrs.get("nvar")).amr_commons()
        b.poisson = True
        b.difmag = attrs.get("difmag", 0.0)
        p = make_params(b)
        assert L.rgpu_init(C.byref(p), 1, 1, 0) == EUNSUPPORTED
    p = make_params(a)
    p.pressure_fix, p.mhd, p.nvar = 0, 1, 8
    assert L.rgpu_init(C.byref(p), 1, 1, 0) == EUNSUPPORTED
    a.pressure_fix = False
    h = HydroGPU(a)
    h.bind_level(c.level)
    h.upload_state(c.level)
    a.dtnew[c.level] = a.boxlen / a.smallc
    dt = C.c_double(1.0)
    assert L.rgpu_courant_fine(c.level, C.byref(dt), None) == EINVAL
    assert L.rgpu_godunov_fine_dev(c.level, 1e-3) == EINVAL
    assert L.rgpu_level_steps(c.level, 1, None, None) == EINVAL
    h.upload_force(force_field(3, c.mesh.s.ncell, 1.0, 1))
    assert L.rgpu_level_steps(c.level, 1, None, None) == 0
    h.finalize()


def _nested_gravity_run(monkeypatch, env, resident):
    """config-4 style nested tree (levels 4-6, refined 12x6x8-oct boxes) with poisson, one coarse step driven by the host amr_step or
    by rgpu_amr_steps; returns the state, dtnew(levelmin), level_info.dense per level and the tree"""
    from ramses_b200.hydro import HydroGPU, amr_step
    from ramses_b200.tree import build_nested_tree, cell_centers
    for k in ("RGPU_AMR_DENSE", "RGPU_AMR_PATCH"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    levelmin, levelmax = 4, 6
    a = build_nested_tree(levelmin, levelmax, half_width=(6, 3, 4))
    a.gamma, a.courant_factor, a.slope_type, a.riemann = 1.4, 0.8, 1, "hllc"
    a.poisson = True
    for l in range(levelmin, levelmax + 1):
        ig, cc = cell_centers(a, l)
        for ind in range(8):
            x, y, z = cc[ind][:, 0], cc[ind][:, 1], cc[ind][:, 2]
            r2 = ((x - 0.55) / 1.5) ** 2 + ((y - 0.48) / 0.8) ** 2 + (z - 0.52) ** 2
            u = np.zeros((5, len(x)))
            u[0] = 1.0 + 0.5 * np.exp(-r2 / 0.01) + 0.1 * np.sin(2 * np.pi * z)
            u[1] = 0.1 * u[0] * np.sin(2 * np.pi * y)
            u[4] = (0.1 + 2.0 * np.exp(-r2 / 0.005)) / 0.4 + 0.5 * u[1] ** 2 / u[0]
            a.uold[:, a.ncoarse + ind * a.ngridmax + ig - 1] = u
    f = force_field(3, a.ncell, 20.0, 77)
    h = HydroGPU(a, amr_mode=True)
    for l in range(1, levelmax + 1):
        h.bind_level(l)
    h.upload_state(0)
    h.upload_force(f)
    for l in range(levelmax - 1, 0, -1):
        h.upload_fine(l)
    h.download_state(0)
    u0 = a.uold.copy()
    nsub = [1] * (levelmin + 1) + [2] * 64
    nsub[levelmin - 1] = 1
    dtnew = {l: 0.0 for l in range(0, levelmax + 2)}
    dtold = {l: 0.0 for l in range(0, levelmax + 2)}
    if resident:
        a.numbtot = {l: len(a.active[l]) for l in range(1, levelmax + 1)}
        dtnew[levelmin] = h.amr_steps(levelmin, nsub, 1)[0]
    else:
        amr_step(h, levelmin, 1, levelmin, nsub, dtnew, dtold)
    h.download_state(0)
    dense = [h.level_info(l).dense for l in (4, 5, 6)]
    h.finalize()
    return a, u0, f, dtnew[levelmin], dense


def test_amr_base_box_and_patch_with_gravity(gpu, monkeypatch):
    """AMR mode, poisson: the dense base box and the refined patches run the GRAV AMR variant (f gathered per call, the shell
    slots injected from their father cells, the refluxed surface faces with the predictor), host-driven and through
    rgpu_amr_steps: the same bits as the oracle's amr_step with orc_set_gravity, and as the oct-batch kernel (RGPU_AMR_DENSE=0,
    RGPU_AMR_PATCH=0)"""
    from oracle.amr import AmrRun
    runs = {
        "dense": _nested_gravity_run(monkeypatch, {}, False),
        "resident": _nested_gravity_run(monkeypatch, {}, True),
        "nopatch": _nested_gravity_run(monkeypatch, {"RGPU_AMR_PATCH": "0"}, False),
        "octbatch": _nested_gravity_run(monkeypatch, {"RGPU_AMR_DENSE": "0"}, False),
    }
    assert runs["dense"][4] == [1, 1, 1] and runs["resident"][4] == [1, 1, 1]
    assert runs["nopatch"][4] == [1, 0, 0] and runs["octbatch"][4] == [0, 0, 0]
    a, u0, f = runs["dense"][:3]
    r = AmrRun(3, 4, 6, (0,) * 6, 1.0, nsubcycle=[1, 2, 2], ngridmax=a.ngridmax, riemann="hllc", slope_type=1, tout=[1e9])
    r.son[1:] = a.son; r.father[1:] = a.father; r.nbor[:, 1:] = a.nbor
    for l in range(1, 7):
        r.active[l] = [int(g) for g in a.active[l]]
    r.push_all()
    r.uold[:] = u0.ravel()
    r.static = True
    with Gravity(f):
        r.amr_step(4, 1)
    ref = r.uold.reshape(5, -1)
    cells = np.concatenate([[a.ncoarse + ind * a.ngridmax + int(g) - 1 for g in a.active[l] for ind in range(8)] for l in range(1, 7)])
    assert np.abs(ref[:, cells] - u0[:, cells]).max() > 1e-4
    for name, (b, _, _, dt, _) in runs.items():
        assert dt == r.dtnew[4], name
        assert np.array_equal(b.uold[:, cells], ref[:, cells]), (name, float(np.abs(b.uold[:, cells] - ref[:, cells]).max()))


def test_amr_gravity_case_runs_its_base_level_dense(gpu, monkeypatch):
    """the 3-D gravity-only case of test_gpu_amr.py::test_amr_gravity_and_pressure_fix_bitwise (levelmin 3, periodic, through
    rgpu_amr_steps): its base level is now swept by the dense kernel's GRAV AMR variant, with the oracle's bits"""
    from ramses_b200.hydro import HydroGPU
    from test_gpu_amr import run_case
    seen = {}
    finalize = HydroGPU.finalize

    def record(self):                      # level_info before the library state is released
        seen.update({l: self.level_info(l).dense for l in self.a.active if len(self.a.active[l])})
        finalize(self)

    monkeypatch.setattr(HydroGPU, "finalize", record)
    regs = [dict(type="square", x_center=0.5, y_center=0.5, z_center=0.5, length_x=10, length_y=10, length_z=10, exp_region=10, d=1.0,
                 p=1e-5),
            dict(type="square", x_center=0.4, y_center=0.45, z_center=0.55, length_x=0.3, length_y=0.3, length_z=0.3, exp_region=2,
                 d=1.5, p=2.0)]
    got, ref, dtnew, r, nlev = run_case(3, 3, 4, (0,) * 6, regs, "hllc", 1, 1, 1, [2, 2], gravity=True, pressure_fix=False,
                                        device_resident=True)
    assert seen[3] == 1
    assert dtnew[3] == r.dtnew[3]
    assert np.array_equal(got, ref), (np.abs(got - ref).max(), nlev)
