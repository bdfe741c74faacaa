"""pressure_fix through the dense sweep on the GPU: the dense base box and the refined patches of AMR mode (nested tree, host-driven
and through rgpu_amr_steps, without and with poisson), levelmin=levelmax grids in AMR mode and a refined mesh at the raised
floors.  Every run is compared with the oracle under orc_set_pressure_fix in state, divu, enew and dtnew, bit for bit ('exact':
1e-12, CUDA pow vs libm pow)."""
import ctypes as C

import numpy as np
import pytest

from helpers import Case, box_state, max_rel_err

pytestmark = pytest.mark.gpu

DP = C.POINTER(C.c_double)


@pytest.fixture(scope="module")
def gpu():
    from ramses_b200 import lib
    lib.load()
    return lib


def force_field(ncell, amp, seed):
    """f[3][ncell]: a mean pull plus cell-to-cell noise on every cell of the tree (boundary octs included)"""
    rng = np.random.default_rng(seed)
    return np.ascontiguousarray(amp * (np.array([0.8, -0.5, 0.3])[:, None] + 0.4 * rng.standard_normal((3, ncell))))


class Sources:
    """orc_set_pressure_fix(divu, enew, beta_fix) and orc_set_gravity(f) of the oracle for the duration of a with-block"""

    def __init__(self, ncell, beta_fix, f=None):
        from oracle import orc
        self.L, self.f, self.beta_fix = orc.lib(), f, beta_fix
        self.L.orc_set_pressure_fix.argtypes = [DP, DP, C.c_double]
        self.L.orc_set_gravity.argtypes = [DP]
        self.divu, self.enew = np.zeros(ncell), np.zeros(ncell)

    def __enter__(self):
        from oracle import orc
        self.L.orc_set_pressure_fix(orc.dptr(self.divu), orc.dptr(self.enew), self.beta_fix)
        self.L.orc_set_gravity(orc.dptr(self.f) if self.f is not None else None)
        return self

    def __exit__(self, *exc):
        self.L.orc_set_pressure_fix(None, None, 0.0)
        self.L.orc_set_gravity(None)


def _nested_pfix_run(monkeypatch, env, resident, poisson, ncoarse=3):
    """config-4 style nested tree (levels 4-6, refined 12x6x8-oct boxes) with pressure_fix (and poisson), ncoarse coarse steps driven
    by the host amr_step or by one rgpu_amr_steps call (the first step is captured as a CUDA graph, the others replay it); returns
    the state, divu, enew, dtnew(levelmin) per coarse step, level_info.dense per level, the initial state, f and the tree"""
    from ramses_b200.hydro import HydroGPU, amr_step
    from ramses_b200.tree import build_nested_tree, cell_centers
    for k in ("RGPU_AMR_DENSE", "RGPU_AMR_PATCH"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    levelmin, levelmax = 4, 6
    a = build_nested_tree(levelmin, levelmax, half_width=(6, 3, 4))
    a.gamma, a.courant_factor, a.slope_type, a.riemann = 1.4, 0.8, 1, "hllc"
    a.poisson, a.pressure_fix, a.beta_fix = poisson, True, 0.5
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
    f = force_field(a.ncell, 20.0, 77) if poisson else None
    h = HydroGPU(a, amr_mode=True)
    for l in range(1, levelmax + 1):
        h.bind_level(l)
    h.upload_state(0)
    if poisson:
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
        dts = list(h.amr_steps(levelmin, nsub, ncoarse))
    else:
        dts = []
        for _ in range(ncoarse):
            amr_step(h, levelmin, 1, levelmin, nsub, dtnew, dtold)
            dts.append(dtnew[levelmin])
    h.download_state(0)
    divu, enew = h.download_pressure_fix()
    dense = [h.level_info(l).dense for l in (4, 5, 6)]
    h.finalize()
    return dict(a=a, u=a.uold.copy(), divu=divu, enew=enew, dts=dts, dense=dense, u0=u0, f=f)


@pytest.mark.parametrize("poisson", [False, True], ids=["pfix", "grav+pfix"])
def test_amr_base_box_and_patch_with_pressure_fix(gpu, monkeypatch, poisson):
    """AMR mode, pressure_fix (and poisson): the dense base box and the refined patches run the PFIX AMR variant (divu / enew
    gathered and scattered per call, the refluxed surface faces with tmp1 / tmp2), host-driven and through rgpu_amr_steps over
    three coarse steps: state, divu, enew and dtnew equal the oracle's amr_step with orc_set_pressure_fix, and equal the runs
    with the patches (RGPU_AMR_PATCH=0) or every level (RGPU_AMR_DENSE=0) on the oct-batch kernel"""
    from oracle.amr import AmrRun
    runs = {
        "dense": _nested_pfix_run(monkeypatch, {}, False, poisson),
        "resident": _nested_pfix_run(monkeypatch, {}, True, poisson),
        "nopatch": _nested_pfix_run(monkeypatch, {"RGPU_AMR_PATCH": "0"}, False, poisson),
        "nopatch_resident": _nested_pfix_run(monkeypatch, {"RGPU_AMR_PATCH": "0"}, True, poisson),
        "octbatch": _nested_pfix_run(monkeypatch, {"RGPU_AMR_DENSE": "0"}, False, poisson),
        "octbatch_resident": _nested_pfix_run(monkeypatch, {"RGPU_AMR_DENSE": "0"}, True, poisson),
    }
    for name, run in runs.items():
        want = [1, 1, 1] if name.startswith(("dense", "resident")) else [1, 0, 0] if name.startswith("nopatch") else [0, 0, 0]
        assert run["dense"] == want, (name, run["dense"])
    a, u0, f = runs["dense"]["a"], runs["dense"]["u0"], runs["dense"]["f"]
    r = AmrRun(3, 4, 6, (0,) * 6, 1.0, nsubcycle=[1, 2, 2], ngridmax=a.ngridmax, riemann="hllc", slope_type=1, tout=[1e9])
    r.son[1:] = a.son; r.father[1:] = a.father; r.nbor[:, 1:] = a.nbor
    for l in range(1, 7):
        r.active[l] = [int(g) for g in a.active[l]]
    r.push_all()
    r.uold[:] = u0.ravel()
    r.static = True
    dts_ref = []
    with Sources(r.m.ncell, 0.5, f) as src:
        for _ in range(3):
            r.amr_step(4, 1)
            dts_ref.append(r.dtnew[4])
    ref = r.uold.reshape(5, -1)
    cells = np.concatenate([[a.ncoarse + ind * a.ngridmax + int(g) - 1 for g in a.active[l] for ind in range(8)] for l in range(1, 7)])
    assert np.abs(ref[:, cells] - u0[:, cells]).max() > 1e-4
    assert np.abs(src.divu[cells]).max() > 0
    for name, run in runs.items():
        assert run["dts"] == dts_ref, (name, run["dts"], dts_ref)
        assert np.array_equal(run["u"][:, cells], ref[:, cells]), (name, float(np.abs(run["u"][:, cells] - ref[:, cells]).max()))
        assert np.array_equal(run["divu"][cells], src.divu[cells]), name
        assert np.array_equal(run["enew"][cells], src.enew[cells]), name
    for name, run in runs.items():        # and the runs equal each other (every active cell of every level)
        assert np.array_equal(run["u"][:, cells], runs["dense"]["u"][:, cells]), name


@pytest.mark.parametrize("riemann,slope_type,bound", [
    ("llf", 1, (0,) * 6), ("exact", 2, (1, 1, 0, 0, 0, 0)), ("acoustic", 3, (0, 0, 0, 0, 2, 2)), ("hllc", 7, (0,) * 6),
    ("hll", 8, (0,) * 6)])
def test_uniform_grid_in_amr_mode_runs_dense_with_pressure_fix(gpu, riemann, slope_type, bound):
    """a levelmin=levelmax 24x16x8 grid in AMR mode with pressure_fix: the level reports the dense kernel (PFIX AMR variant); three
    level steps in amr_step order (courant, set_unew, godunov_fine, set_uold, make_boundary_hydro) equal the oracle's in state,
    divu, enew and the time steps"""
    from ramses_b200.hydro import HydroGPU
    level = 3
    c = Case(3, level, riemann=riemann, slope_type=slope_type, bound=bound, coarse=(3, 2, 1), boxlen=3.0, order=2, seed=4)
    c.init_dense(box_state(3, c.mesh.extent(level), seed=4))
    with Sources(c.mesh.s.ncell, 0.5) as src:
        ref, dts_ref = c.oracle_steps(3, nthreads=1)
    a = c.amr_commons()
    a.pressure_fix, a.beta_fix = True, 0.5
    h = HydroGPU(a, amr_mode=True)
    for l in range(1, level + 1):
        h.bind_level(l)
    info = h.level_info(level)
    assert info.dense == 1
    h.upload_state(0)
    h.make_boundary_hydro(level)
    dts = []
    for _ in range(3):
        a.dtnew[level] = a.boxlen / a.smallc
        dts.append(h.courant_fine(level))
        h.set_unew(level); h.godunov_fine_dev(level); h.set_uold(level); h.make_boundary_hydro(level)
    h.download_state(0)
    divu, enew = h.download_pressure_fix()
    h.finalize()
    idx = c.active_cells()
    ref = ref.reshape(c.nvar, -1)
    assert np.abs(ref[:, idx] - c.u.reshape(c.nvar, -1)[:, idx]).max() > 1e-4
    assert np.abs(src.divu[idx]).max() > 0
    got = np.concatenate([a.uold[:, idx], divu[None, idx], enew[None, idx]])
    want = np.concatenate([ref[:, idx], src.divu[None, idx], src.enew[None, idx]])
    if riemann == "exact":
        assert np.allclose(dts, dts_ref, rtol=1e-12, atol=0)
        assert max_rel_err(got, want) <= 1e-12
    else:
        assert np.array_equal(np.array(dts), dts_ref), (dts, dts_ref)
        assert np.array_equal(got, want), [float(np.abs(got[n] - want[n]).max()) for n in range(7)]


@pytest.mark.parametrize("gravity,resident", [(False, True), (True, False)])
def test_refined_mesh_pressure_fix_at_the_floors_sweeps_dense(gpu, monkeypatch, gravity, resident):
    """pressure_fix (and poisson) on a 3-D adaptively refined mesh whose every cell holds a floor_state cell under the raised
    floors, as test_gpu_floors.py::test_refined_mesh_pressure_fix_at_the_floors: the base level is swept by the PFIX AMR variant
    and one sub-cycled coarse step gives the oracle's state, divu, enew and dtnew bit for bit"""
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
    got, ref, dtnew, r, nlev = run_case(3, 3, 4, (0,) * 6, regs, "hllc", 1, 1, 1, [2, 2], gravity=gravity, pressure_fix=True,
                                        device_resident=resident, floors="raised")
    assert seen[3] == 1
    assert np.isfinite(ref).all()
    assert dtnew[3] == r.dtnew[3]
    assert np.array_equal(got, ref), float(np.abs(got - ref).max())
    dk, do, ek, eo = r.pfix_cmp
    assert np.array_equal(dk, do) and np.array_equal(ek, eo)
    assert np.abs(do).max() > 0
