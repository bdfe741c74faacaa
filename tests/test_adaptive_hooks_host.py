"""The hook layer of tests/test_gpu_adaptive.py checked without a GPU.

`FakeDevice` has the HydroGPU methods the layer calls and runs them with the oracle's own routines on PRIVATE copies of
uold / unew; upload_state / download_state copy between those and the driver's arrays.  Whenever the fake device changes its
state it overwrites the host copy with NaN, so a host read of uold that is not preceded by a download poisons the run.  It
also checks, on every call, that the tree and the level's lists it was last bound with are the driver's current ones.

With it the blob (3-D, levels 4..6) and the sod-tube (1-D) run under every bind policy and come out bitwise equal to the
all-oracle run: the downloads and uploads of the Level-1 layer are complete, and the layer never reads the host state while
the device holds a newer copy.  A GPU failure of test_gpu_adaptive.py is then the library's, not the harness's."""
from types import SimpleNamespace

import numpy as np
import pytest

from test_gpu_adaptive import attach, blob_run, first_divergence, record_oracle


class FakeDevice:
    ROUTINES = ("c_set_unew", "c_godunov_fine", "c_set_uold", "upload_fine", "make_boundary_hydro", "hydro_flag", "newdt_fine")

    def __init__(self, r):
        self.r = r
        self.a = SimpleNamespace(active={}, boundary={}, dtnew={}, father=r.father[1:], nbor=np.zeros_like(r.nbor[:, 1:]))
        self.uold, self.unew = np.full_like(r.uold, np.nan), np.full_like(r.unew, np.nan)
        self.fn = {n: getattr(type(r), n).__get__(r) for n in self.ROUTINES}    # the oracle's, not the hooks'
        self.tree, self.lists = None, {}
        self.calls = 0

    # -- bookkeeping ---------------------------------------------------------------------------------------------------------
    def bind_tree(self):
        assert np.array_equal(self.a.nbor, self.r.nbor[:, 1:])
        self.tree = (self.r.son.copy(), self.r.father.copy(), self.r.nbor.copy())

    def bind_level(self, l):
        self.lists[l] = (np.array(self.a.active[l]), [np.array(x) for x in self.a.boundary[l]])

    def _check(self, l):
        r = self.r
        assert self.tree is not None and all(np.array_equal(x, y) for x, y in zip(self.tree, (r.son, r.father, r.nbor))), \
            "device tree is stale"
        act, bnd = self.lists[l]
        assert np.array_equal(act, np.array(r.active[l])), f"level {l} bound with stale active list"
        assert all(np.array_equal(x, np.array(r.bound[b][l])) for b, x in enumerate(bnd)), f"level {l} bound with stale boundary lists"

    def _run(self, name, l, poison):
        """one oracle routine on the device's arrays"""
        self._check(l)
        r = self.r
        hu, hn = r.uold, r.unew
        r.uold, r.unew = self.uold, self.unew
        try:
            self.fn[name](l)
        finally:
            r.uold, r.unew = hu, hn
        if poison:
            hu[:] = np.nan       # the host copy is stale from here on
        self.calls += 1

    # -- the HydroGPU calls of the Level-1 layer ------------------------------------------------------------------------------
    def upload_state(self, l):
        self.uold[:] = self.r.uold

    def download_state(self, l):
        self.r.uold[:] = self.uold

    def peek(self):
        return self.uold.copy()

    def set_unew(self, l):
        self._run("c_set_unew", l, False)

    def godunov_fine_dev(self, l):
        assert self.a.dtnew[l] == self.r.dtnew[l]
        self._run("c_godunov_fine", l, False)

    def set_uold(self, l):
        self._run("c_set_uold", l, True)

    def upload_fine(self, l):
        self._run("upload_fine", l, True)

    def make_boundary_hydro(self, l):
        self._run("make_boundary_hydro", l, True)

    def hydro_flag(self, l, flag1, err_grad, floor):
        r = self.r
        assert flag1.ctypes.data == r.flag1[1:].ctypes.data
        assert tuple(err_grad) == (r.err_grad_d, r.err_grad_u, r.err_grad_p) and tuple(floor) == (r.floor_d, r.floor_u, r.floor_p)
        self._run("hydro_flag", l, False)

    def courant_fine(self, l):
        """dtnew(l) = min(dtnew(l), CFL dt): the oracle's newdt_fine starts from boxlen/smallc, which the layer passes"""
        r = self.r
        assert self.a.dtnew[l] == r.p.boxlen / r.p.smallc
        keep = r.dtold[l], r.dtnew[l]
        self._run("newdt_fine", l, False)
        self.a.dtnew[l] = r.dtnew[l]
        r.dtold[l], r.dtnew[l] = keep
        return self.a.dtnew[l]


def _sod():
    from oracle.amr import AmrRun
    from test_oracle_golden import SOD
    return AmrRun(1, 3, 10, (1, 1, 0, 0, 0, 0), 1.0, nsubcycle=[1, 1, 1, 2], nexpand=1, ngridmax=2000, riemann="hllc",
                  slope_type=2, gamma=1.4, courant_factor=0.8, err_grad_d=0.05, err_grad_u=0.05, err_grad_p=0.05,
                  interpol_type=2, interpol_var=0, regions=SOD, tout=[1e9])


PROBLEMS = {"blob": (lambda: blob_run("hllc", 1, nsubcycle=(2, 2)), 10), "sod": (_sod, 5)}
_ref = {}


def _reference(name):
    if name not in _ref:
        make, n = PROBLEMS[name]
        r = make()
        recs = record_oracle(r)
        r.run(max_coarse=n)
        _ref[name] = (r, recs)
    return _ref[name]


@pytest.mark.parametrize("device_flag", [True, False], ids=["device-flag", "host-flag"])
@pytest.mark.parametrize("policy", ["A", "B", "C"])
@pytest.mark.parametrize("problem", list(PROBLEMS))
def test_level1_hooks_on_a_cpu_device_equal_the_oracle(orc, problem, policy, device_flag):
    ref, recs = _reference(problem)
    make, n = PROBLEMS[problem]
    r = make()
    dev = FakeDevice(r)
    st = attach(r, dev, True, policy, device_flag=device_flag)
    r.run(max_coarse=n)
    where = first_divergence(recs, st["records"])
    assert where is None, where
    assert ref.t == r.t and ref.nstep == r.nstep and np.array_equal(ref.son, r.son)
    # the state did live on the device: the host copy was stale (NaN) in between, downloads and uploads happened
    assert st["downloads"] > 0 and st["uploads"] > 0 and dev.calls > 0
    switched = sum(not np.array_equal(x["lev"][l]["son"], y["lev"][l]["son"]) for x, y in zip(recs, recs[1:]) for l in x["lev"])
    assert switched > 0                      # the mesh changed while the device held the state


def test_level0_hooks_equal_the_oracle(orc):
    """the Level-0 layer on the fake device: godunov_fine on the host arrays"""
    ref, recs = _reference("blob")
    r = PROBLEMS["blob"][0]()
    dev = FakeDevice(r)
    dev.godunov_fine = lambda l: (dev._check(l), dev.fn["c_godunov_fine"](l))
    st = attach(r, dev, False, "A")
    r.run(max_coarse=10)
    assert first_divergence(recs, st["records"]) is None
    assert st["calls"] > 0 and st["downloads"] == 0
