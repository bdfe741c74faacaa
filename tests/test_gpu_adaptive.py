"""Adaptive runs on the GPU: the oracle's AMR driver regrids every coarse step while the library sweeps the levels.

Each test runs one problem twice -- all on the oracle (oracle/amr.py, oracle/amr_mhd.py) and with the driver's per-level
routines swapped for the device -- and compares state, mesh and time BITWISE after every coarse step: uold over the active
cells, son / father / nbor, the active and boundary lists, t, nstep.

Two hook layers (`attach`):

* Level-0 (`resident=False`): only `c_godunov_fine` goes to `rgpu_godunov_fine` (host arrays in and out), like
  test_gpu_zz_golden.attach_gpu_godunov.
* Level-1 (`resident=True`): the state lives on the device (INTEGRATION.md section 3).  set_unew, godunov_fine, set_uold,
  upload_fine, make_boundary_hydro and the Courant scan of newdt_fine run there; hydro_flag runs there too
  (`device_flag=True`) or on the host after a download.  The host reads uold only in refine_fine (make_grid_fine
  interpolates new octs from it), in a host hydro_flag and in dump: the state is downloaded right before those, and
  uploaded (then the tree re-bound) after every regrid.  Init (init_refine, init_refine_2) stays on the oracle.

Bind policies (when the level lists reach the library):

* "A", reference order: bind_level(i) right before refine_fine(i) -- where amr_step.f90 calls build_comm(i), i.e. BEFORE
  the level's own cells change their sons -- plus every level whose lists changed; bind_tree after the regrid.
* "B", signature: only levels whose (active, father, nbor, boundary) lists changed are re-bound, lazily.
* "C", everything: bind_tree and every level holding octs re-bound after every regrid.

tests/test_adaptive_hooks_host.py runs the same layer against a CPU stand-in of the device, so that a failure here is the
library's, not the harness's."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")

# the moving blob: a dense square (exp_region=2) of side 0.15 advected diagonally through a periodic box
BLOB = [dict(type="square", x_center=0.5, y_center=0.5, z_center=0.5, length_x=10, length_y=10, length_z=10, exp_region=10,
             d=1.0, u=1.0, v=0.5, p=1.0),
        dict(type="square", x_center=0.3, y_center=0.4, z_center=0.5, length_x=0.15, length_y=0.15, length_z=0.15, exp_region=2,
             d=3.0, u=1.0, v=0.5, p=1.0)]
SEDOV = [dict(type="square", x_center=0.5, y_center=0.5, z_center=0.5, length_x=10, length_y=10, length_z=10, exp_region=10, d=1.0,
              p=1e-5),
         dict(type="point", x_center=0.5, y_center=0.5, z_center=0.5, p=0.4)]


# ---- the hook layer ------------------------------------------------------------------------------------------------------------
def attach(r, h, resident, policy, device_flag=False, probe=False):
    """swap the driver's per-level routines of run `r` for the device `h` (HydroGPU, or the CPU stand-in of
    test_adaptive_hooks_host.py); returns the state dict: counters, `records` (one per coarse step) and `dense` (per coarse
    step, {level: level_info(level).dense} when `probe`)"""
    assert policy in ("A", "B", "C")
    a, m = h.a, r.m
    nb = m.nboundary
    st = dict(on=False, tree=True, host_newer=True, dev_newer=False, sig={}, bound=set(), binds=0, syncs=0, uploads=0,
              downloads=0, calls=0, records=[], dense=[])
    o = {n: getattr(r, n) for n in ("refine_fine", "make_boundary_hydro", "upload_fine", "c_set_unew", "c_godunov_fine",
                                    "c_set_uold", "newdt_fine", "hydro_flag", "dump", "init_refine_2", "make_grid_fine",
                                    "kill_grid", "amr_step")}

    def lists(l):
        return (np.array(r.active[l], dtype=np.int32), [np.array(r.bound[b][l], dtype=np.int32) for b in range(nb)])

    def bind(l, sig):
        h.bind_level(l)
        st["bound"].add(l)
        st["sig"][l] = sig
        st["binds"] += 1

    def rebind(levels, force):
        for l in levels:
            act, bnd = lists(l)
            a.active[l], a.boundary[l] = act, bnd
            if len(act) == 0 and not any(len(x) for x in bnd) and l not in st["bound"]:
                continue                      # never held an oct: nothing to bind, nothing will run on it
            sig = (act.tobytes(), a.father[act - 1].tobytes(), a.nbor[:, act - 1].tobytes(), tuple(x.tobytes() for x in bnd))
            if force or st["sig"].get(l) != sig:
                bind(l, sig)

    def sync():
        """after a regrid: upload the state (new octs were interpolated on the host), bind the tree, re-bind levels"""
        if st["host_newer"] and resident:
            h.upload_state(r.levelmin)
            st["uploads"] += 1
        st["host_newer"] = False
        if st["tree"]:
            a.nbor[:, :] = r.nbor[:, 1:]
            h.bind_tree()
            rebind(range(1, r.nlevelmax + 1), policy == "C")
            st["tree"] = False
            st["syncs"] += 1

    def pull():
        """the host is about to read uold: bring the device's newer copy back"""
        if resident and st["dev_newer"]:
            assert not st["host_newer"], "host and device both hold changes"
            h.download_state(r.levelmin)
            st["dev_newer"] = False
            st["downloads"] += 1

    def live(l):
        return l in st["bound"]

    # -- mesh changes (host) --------------------------------------------------------------------------------------------------
    def make_grid_fine(*args):
        st["tree"] = st["host_newer"] = True
        return o["make_grid_fine"](*args)

    def kill_grid(*args):
        st["tree"] = True
        return o["kill_grid"](*args)

    def refine_fine(l):
        if st["on"]:
            if policy == "A":
                sync()
                rebind([l], True)             # the lists as build_comm(l) leaves them, before refine_fine(l) changes son
            pull()
        return o["refine_fine"](l)

    def init_refine_2():
        o["init_refine_2"]()
        st["on"] = True                       # the device takes over right before the first amr_step

    # -- the per-level routines -----------------------------------------------------------------------------------------------
    def c_godunov_fine(l):
        if not st["on"]:
            return o["c_godunov_fine"](l)
        sync()
        if not live(l):
            return
        a.dtnew[l] = r.dtnew[l]
        if resident:
            h.godunov_fine_dev(l)
        else:
            h.godunov_fine(l)
        st["calls"] += 1

    def device_op(name, fn, writes_uold):
        def w(l):
            if not (st["on"] and resident):
                return o[name](l)
            sync()
            if live(l):
                fn(l)
                st["dev_newer"] = st["dev_newer"] or writes_uold
        return w

    def newdt_fine(l):
        if not (st["on"] and resident):
            return o["newdt_fine"](l)
        sync()
        r.dtold[l] = r.dtnew[l]
        a.dtnew[l] = r.p.boxlen / r.p.smallc
        r.dtnew[l] = h.courant_fine(l)

    def hydro_flag(l):
        if not (st["on"] and resident):
            return o["hydro_flag"](l)
        if not device_flag:
            pull()
            return o["hydro_flag"](l)
        if l == r.nlevelmax or r.numbtot(l) == 0:
            return
        sync()
        h.hydro_flag(l, r.flag1[1:], (r.err_grad_d, r.err_grad_u, r.err_grad_p), (r.floor_d, r.floor_u, r.floor_p))

    def dump():
        pull()
        return o["dump"]()

    def amr_step(l, icount):
        o["amr_step"](l, icount)
        if l == r.levelmin:
            st["records"].append(record(r, peek() if resident else r.uold))
            if probe:
                st["dense"].append({k: h.level_info(k).dense for k in sorted(st["bound"])})

    def peek():
        """the device's uold, without touching the host copy"""
        if hasattr(h, "peek"):
            return h.peek()
        import ctypes as C
        buf = np.empty_like(a.uold)
        h.L.rgpu_download_state(r.levelmin, buf.ctypes.data_as(C.POINTER(C.c_double)))
        return buf

    r.make_grid_fine, r.kill_grid, r.refine_fine, r.init_refine_2 = make_grid_fine, kill_grid, refine_fine, init_refine_2
    r.c_godunov_fine, r.newdt_fine, r.hydro_flag, r.dump, r.amr_step = c_godunov_fine, newdt_fine, hydro_flag, dump, amr_step
    r.c_set_unew = device_op("c_set_unew", h.set_unew, False)
    r.c_set_uold = device_op("c_set_uold", h.set_uold, True)
    r.upload_fine = device_op("upload_fine", h.upload_fine, True)
    r.make_boundary_hydro = device_op("make_boundary_hydro", h.make_boundary_hydro, True)
    return st


def record_oracle(r):
    """per-coarse-step records of an all-oracle run"""
    recs = []
    orig = r.amr_step

    def amr_step(l, icount):
        orig(l, icount)
        if l == r.levelmin:
            recs.append(record(r, r.uold))
    r.amr_step = amr_step
    return recs


def record(r, uold):
    U = np.asarray(uold).reshape(-1, r.ncell)
    out = dict(t=r.t, nstep=r.nstep, lev={})
    for l in range(1, r.nlevelmax + 1):
        act = np.array(r.active[l], dtype=np.int64)
        cells = (r.ncoarse + np.arange(r.T)[:, None] * r.ngridmax + act[None, :]).ravel()
        out["lev"][l] = dict(active=act, bound=[np.array(r.bound[b][l]) for b in range(r.m.nboundary)], father=r.father[act].copy(),
                             nbor=r.nbor[:, act].copy(), son=r.son[cells].copy(), cells=cells, u=U[:, cells - 1].copy())
    return out


def first_divergence(ref, got):
    """None if the two record lists are bitwise equal, else where they first differ (coarse step, level, field, cell)"""
    if len(ref) != len(got):
        return f"{len(ref)} coarse steps in the oracle run, {len(got)} in the device run"
    for k, (x, y) in enumerate(zip(ref, got)):
        if x["t"] != y["t"] or x["nstep"] != y["nstep"]:
            return f"coarse step {k + 1}: t/nstep {x['t']!r}/{x['nstep']} != {y['t']!r}/{y['nstep']}"
        for l in x["lev"]:
            a, b = x["lev"][l], y["lev"][l]
            for key in ("active", "father", "nbor", "son"):
                if not np.array_equal(a[key], b[key]):
                    return f"coarse step {k + 1}, level {l}: {key} differs"
            if any(not np.array_equal(p, q) for p, q in zip(a["bound"], b["bound"])):
                return f"coarse step {k + 1}, level {l}: boundary lists differ"
            bad = np.argwhere(~((a["u"] == b["u"]) | (np.isnan(a["u"]) & np.isnan(b["u"]))))
            if len(bad):
                iv, j = bad[0]
                return (f"coarse step {k + 1}, level {l}: {len(bad)} values differ, first cell {a['cells'][j]} (son {a['son'][j]}) "
                        f"var {iv}: {a['u'][iv, j]!r} != {b['u'][iv, j]!r}")
    return None


def base_switches(recs, l):
    """(cells of level l that became refined, cells that became leaves) between consecutive coarse steps, summed"""
    up = down = 0
    for x, y in zip(recs, recs[1:]):
        assert np.array_equal(x["lev"][l]["active"], y["lev"][l]["active"])
        s0, s1 = x["lev"][l]["son"] > 0, y["lev"][l]["son"] > 0
        up += int(np.sum(~s0 & s1))
        down += int(np.sum(s0 & ~s1))
    return up, down


def make_gpu(r, mhd=False, riemann="hllc", riemann2d="llf", slope_type=1, interpol_type=1, interpol_var=0):
    """a HydroGPU in AMR mode on the tree arrays of run r (views, not copies)"""
    from ramses_b200.hydro import AmrCommons, HydroGPU
    m = r.m
    a = AmrCommons(r.ndim, 8 if mhd else r.nvar, m.ncoarse, m.ngridmax, m.nx, m.ny, m.nz, (m.icoarse_min, m.icoarse_max),
                   (m.jcoarse_min, m.jcoarse_max), (m.kcoarse_min, m.kcoarse_max), nlevelmax=r.nlevelmax, boxlen=r.p.boxlen, mhd=mhd)
    a.son, a.father = r.son[1:], r.father[1:]
    a.uold, a.unew = r.uold.reshape(-1, m.ncell), r.unew.reshape(-1, m.ncell)
    a.nbor[:, :] = r.nbor[:, 1:]
    a.boundary_type = [m.boundary_type[b] for b in range(m.nboundary)]
    pp = r.pm if mhd else r.p
    a.gamma, a.courant_factor = pp.gamma, pp.courant_factor
    a.slope_type, a.riemann, a.nvector = slope_type, riemann, r.nvector
    if mhd:
        a.slope_mag_type, a.riemann2d = -1, riemann2d
    return HydroGPU(a, amr_mode=True, interpol_type=interpol_type, interpol_var=interpol_var)


def run_pair(make_run, ncoarse, resident, policy, device_flag=True, probe=False, gpu_kw=None):
    """the problem all-oracle, then through the device; returns (oracle run, records, device run, hook state)"""
    ref = make_run()
    recs = record_oracle(ref)
    ref.run(max_coarse=ncoarse)
    r = make_run()
    h = make_gpu(r, **(gpu_kw or {}))
    try:
        st = attach(r, h, resident, policy, device_flag=device_flag, probe=probe)
        r.run(max_coarse=ncoarse)
    finally:
        h.finalize()
    assert len(recs) == ncoarse or ref.done      # (a run to its end stops at tout)
    return ref, recs, r, st


def _same(ref, recs, r, st):
    where = first_divergence(recs, st["records"])
    assert where is None, where
    assert np.array_equal(ref.son, r.son) and np.array_equal(ref.father, r.father) and np.array_equal(ref.nbor, r.nbor)
    assert ref.t == r.t and ref.nstep == r.nstep and ref.nstep_coarse == r.nstep_coarse


# ---- 3-D hydro: the moving blob, levels 4..6 -----------------------------------------------------------------------------------
def blob_run(riemann="hllc", slope_type=1, nsubcycle=(1, 2), interpol_type=1, interpol_var=0, bound_type=(0,) * 6, nvar=None,
             seed=None, bound_regions=None):
    from oracle.amr import FastAmrRun
    r = FastAmrRun(3, 4, 6, bound_type, 1.0, nsubcycle=list(nsubcycle), ngridmax=40000, riemann=riemann, slope_type=slope_type,
                   err_grad_d=0.05, interpol_type=interpol_type, interpol_var=interpol_var, regions=BLOB, tout=[1e9], nvar=nvar,
                   bound_regions=bound_regions)
    if seed is not None:
        seed(r)
    return r


def seed_scalars(r):
    """passive scalars set by init_flow_fine on every level: Z1 = 1 in the blob, Z2 smooth (like a condinit with scalars)"""
    from test_passive_scalars_host import _cell_positions
    base = r.init_flow_fine

    def init_flow_fine(l):
        base(l)
        if r.numbtot(l) == 0:
            return
        U = r.uold.reshape(r.nvar, r.ncell)
        ig, x = _cell_positions(r, l)
        for ind in range(r.T):
            c = r.ncoarse + ind * r.ngridmax + ig - 1
            X, Y, Z = x[ind]
            U[5, c] = U[0, c] * ((np.abs(X - 0.3) < 0.1) & (np.abs(Y - 0.4) < 0.1))
            if r.nvar > 6:
                U[6, c] = U[0, c] * (0.5 + 0.3 * np.sin(2 * np.pi * X) * np.cos(2 * np.pi * Z))
    r.init_flow_fine = init_flow_fine


BLOB_ROWS = [("hllc", 1), ("llf", 2), ("hll", 8), ("acoustic", 3)]
LAYERS = [(False, "A"), (False, "B"), (True, "A"), (True, "B"), (True, "C")]
_blob_oracle = {}


def _blob_reference(riemann, slope_type):
    """the all-oracle blob run of one row, once per module; and the count of base cells that switched"""
    key = (riemann, slope_type)
    if key not in _blob_oracle:
        ref = blob_run(riemann, slope_type)
        recs = record_oracle(ref)
        ref.run(max_coarse=40)
        _blob_oracle[key] = (ref, recs, base_switches(recs, 4))
    return _blob_oracle[key]


@pytest.mark.parametrize("resident,policy", LAYERS, ids=[f"{'level1' if x else 'level0'}-{p}" for x, p in LAYERS])
@pytest.mark.parametrize("riemann,slope_type", BLOB_ROWS)
def test_blob_3d_adaptive_bitwise(orc, riemann, slope_type, resident, policy):
    """40 coarse steps, levels 4..6: the base (level 4, a full box) runs the dense kernel while its cells refine and derefine"""
    ref, recs, (up, down) = _blob_reference(riemann, slope_type)
    assert up > 0 and down > 0, (up, down)          # base cells refined AND derefined during the run
    r = blob_run(riemann, slope_type)
    h = make_gpu(r, riemann=riemann, slope_type=slope_type)
    try:
        st = attach(r, h, resident, policy, device_flag=True, probe=True)
        r.run(max_coarse=40)
    finally:
        h.finalize()
    assert all(d.get(4) == 1 for d in st["dense"]), st["dense"][:3]
    _same(ref, recs, r, st)


def test_blob_3d_adaptive_oct_batch_control(orc, monkeypatch):
    """the same run with the dense base disabled: the oct-batch kernel sweeps level 4"""
    monkeypatch.setenv("RGPU_AMR_DENSE", "0")
    ref, recs, _ = _blob_reference("hllc", 1)
    r = blob_run("hllc", 1)
    h = make_gpu(r, riemann="hllc", slope_type=1)
    try:
        st = attach(r, h, True, "A", device_flag=True, probe=True)
        r.run(max_coarse=40)
    finally:
        h.finalize()
    assert all(d.get(4) == 0 for d in st["dense"])
    _same(ref, recs, r, st)


VARIANTS = {
    "interpol-2-1": dict(interpol_type=2, interpol_var=1),
    "interpol-4-2": dict(interpol_type=4, interpol_var=2),
    "nsubcycle-2-2": dict(nsubcycle=(2, 2)),
    # walls on x, outflow on y, periodic z; the y regions span the x boundary columns, so that the four box edges are covered
    # (like the corners of tests/hydro/implosion): with face regions only, octs along an edge have no oct across it
    "walls-x-outflow-y": dict(bound_type=(1, 1, 2, 2, 0, 0), bound_regions=[(1, (0, 0), (1, 1), (0, 0)), (2, (2, 2), (1, 1), (0, 0)),
                                                                             (13, (0, 2), (0, 0), (0, 0)), (14, (0, 2), (2, 2), (0, 0))]),
    "scalars-1": dict(nvar=6, seed=seed_scalars),
    "scalars-2": dict(nvar=7, seed=seed_scalars),
}


@pytest.mark.parametrize("name", list(VARIANTS))
def test_blob_3d_adaptive_level1_variants(orc, name):
    """Level-1 (A) on the blob away from its default: prolongation, sub-cycling (a regrid inside the recursion while level 4's
    unew holds the first sub-step's refluxes on the device only), physical boundaries, passive scalars (oct-batch path and the
    host hydro_flag: rgpu_hydro_flag is nvar = ndim+2 only)"""
    kw = VARIANTS[name]
    scalars = "nvar" in kw
    gkw = dict(riemann="hllc", slope_type=1, interpol_type=kw.get("interpol_type", 1), interpol_var=kw.get("interpol_var", 0))
    ref, recs, r, st = run_pair(lambda: blob_run(**kw), 20, True, "A", device_flag=not scalars, probe=True, gpu_kw=gkw)
    _same(ref, recs, r, st)
    assert all(d.get(4) == (0 if scalars else 1) for d in st["dense"])
    if scalars:    # the scalars moved with the flow
        assert not np.array_equal(recs[0]["lev"][4]["u"][5:], recs[-1]["lev"][4]["u"][5:])


# ---- 3-D hydro: the Sedov blast, levels 3..5 (level 4 fills the box and changes kernel mid-run) --------------------------------
@pytest.mark.parametrize("policy", ["A", "B"])
def test_sedov_3d_level_changes_kernel_mid_run(orc, policy):
    from oracle.amr import FastAmrRun

    def make():
        return FastAmrRun(3, 3, 5, (0,) * 6, 1.0, nsubcycle=[1, 2], ngridmax=8000, riemann="hllc", slope_type=1, err_grad_p=0.1,
                          interpol_type=1, regions=SEDOV, tout=[1e9])
    ref, recs, r, st = run_pair(make, 8, True, policy, probe=True, gpu_kw=dict(riemann="hllc", slope_type=1))
    _same(ref, recs, r, st)
    d4 = [d.get(4, 0) for d in st["dense"]]
    assert d4[0] == 0 and d4[-1] == 1, d4
    assert [len(x["lev"][4]["active"]) == 512 for x in recs] == [x == 1 for x in d4]


# ---- golden problems through the Level-1 layer -----------------------------------------------------------------------------------
def test_sod_tube_golden_level1(orc):
    import json
    from oracle.amr import AmrRun, check_sums
    from test_oracle_golden import SOD

    def make():
        return AmrRun(1, 3, 10, (1, 1, 0, 0, 0, 0), 1.0, nsubcycle=[1, 1, 1, 2], nexpand=1, ngridmax=2000, riemann="hllc",
                      slope_type=2, gamma=1.4, courant_factor=0.8, err_grad_d=0.05, err_grad_u=0.05, err_grad_p=0.05,
                      interpol_type=2, interpol_var=0, regions=SOD, tout=[0.245])
    ref, recs, r, st = run_pair(make, 100000, True, "A", gpu_kw=dict(riemann="hllc", slope_type=2, interpol_type=2))
    _same(ref, recs, r, st)
    snap = r.snapshot
    gold = json.load(open(os.path.join(GOLD, "sod_tube_ref.json")))
    sums = check_sums(snap["rows"], 1)
    sums["time"] = snap["t"]
    for key in ("ncells", "level", "x", "density", "pressure", "velocity_x", "time"):
        err = abs(sums[key] - gold[key]) / max(min(abs(sums[key]), abs(gold[key])), 1e-300)
        assert err <= 3.0e-13, (key, sums[key], gold[key], err)
    assert snap["nstep_coarse"] == 43 and snap["nstep"] == 688 and st["downloads"] > 0


def test_implosion_first_steps_level1(orc):
    from conftest import IMPL, IMPL_BOUND
    from oracle.amr import FastAmrRun

    def make():
        return FastAmrRun(2, 5, 8, (1, 1, 1, 1, 0, 0), 1.0, nsubcycle=[2] * 10, nexpand=[4], ngridmax=12000, riemann="hllc",
                          slope_type=2, gamma=1.4, courant_factor=0.8, err_grad_d=0.05, err_grad_u=0.05, err_grad_p=0.05,
                          interpol_type=2, interpol_var=0, regions=IMPL, tout=[1e9], bound_regions=IMPL_BOUND)
    ref, recs, r, st = run_pair(make, 20, True, "A", gpu_kw=dict(riemann="hllc", slope_type=2, interpol_type=2))
    _same(ref, recs, r, st)
    assert len(r.active[8]) > 0


def test_imhd_tube_first_steps_level1(orc):
    from oracle.amr_mhd import MhdAmrRun
    from test_oracle_golden import IMHD

    def make():
        return MhdAmrRun(5, 15, (2, 2, 0, 0, 0, 0), 3.5, nsubcycle=[1, 1, 1, 1], riemann="hlld", slope_type=0, gamma=1.6666667,
                         courant_factor=0.8, err_grad_d=0.01, err_grad_u=0.05, err_grad_p=0.05, interpol_type=2, regions=IMHD,
                         tout=[1e9], ngridmax=10000)
    ref, recs, r, st = run_pair(make, 25, True, "A", device_flag=False,
                                gpu_kw=dict(mhd=True, riemann="hlld", slope_type=0, interpol_type=2))
    _same(ref, recs, r, st)
    assert sum(1 for l in range(1, 16) if r.active[l]) >= 10


def test_orszag_tang_first_steps_level1(orc):
    from oracle.amr_mhd import MhdAmrRun2D

    def make():
        return MhdAmrRun2D(4, 6, 1.0, nsubcycle=[1, 2], riemann="hlld", riemann2d="hlld", slope_type=2, gamma=1.6666667,
                           courant_factor=0.8, err_grad_p=0.1, interpol_type=2, tout=[1e9], nexpand=1, ngridmax=20000)
    ref, recs, r, st = run_pair(make, 4, True, "A", device_flag=False,
                                gpu_kw=dict(mhd=True, riemann="hlld", riemann2d="hlld", slope_type=2, interpol_type=2))
    _same(ref, recs, r, st)
    assert r.divb_max() < 5e-14 and len(r.active[5]) > 0


# ---- 3-D MHD on a changing mesh -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("resident", [False, True], ids=["level0-A", "level1-A"])
def test_mhd_3d_adaptive(orc, resident):
    """the z-invariant Orszag-Tang state in 3-D, levels 3..5: the mesh regrids every coarse step"""
    from oracle.amr_mhd import MhdAmrRun3D

    def make():
        return MhdAmrRun3D(3, 5, 1.0, nsubcycle=[1, 2], riemann="hlld", riemann2d="hlld", slope_type=2, gamma=1.6666667,
                           courant_factor=0.8, err_grad_p=0.1, interpol_type=2, tout=[1e9], nexpand=1, ngridmax=12000)
    ref, recs, r, st = run_pair(make, 4, resident, "A", device_flag=False,
                                gpu_kw=dict(mhd=True, riemann="hlld", riemann2d="hlld", slope_type=2, interpol_type=2))
    _same(ref, recs, r, st)
    changed = sum(not np.array_equal(x["lev"][4]["son"], y["lev"][4]["son"]) or len(x["lev"][5]["active"]) != len(y["lev"][5]["active"])
                  for x, y in zip(recs, recs[1:]))
    assert changed > 0 and r.divb_max() < 5e-14
