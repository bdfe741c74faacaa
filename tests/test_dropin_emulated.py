"""The drop-in flow WITHOUT a GPU: the oracle's AMR driver (the host code RAMSES keeps: flagging, refinement, time-step control,
set_unew / set_uold, upload_fine, boundaries) with its `godunov_fine` replaced by the DEVICE code -- the oct-batch kernels of
ramses_b200/csrc compiled for the host and executed by the emulated launch of tests/host_numerics (one OS thread per CUDA thread),
followed by the coarse-reflux kernels with the schedules rgpu_api.cu builds at bind time (amr_schedules.h).  Full adaptive runs
with regridding every coarse step:

* tests/hydro/sod-tube to its end: the golden sums of the reference come out (3e-13) from the device code;
* the first coarse steps of imhd-tube (1-D AMR MHD), implosion (2-D AMR hydro, four walls) and orszag-tang (2-D AMR MHD): state,
  mesh and time bit-identical to the all-oracle run.

The same flow with the real GPU behind `rgpu_godunov_fine` is tests/test_gpu_zz_golden.py (all four golden files, full length)."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from test_device_numerics_host import dev, MHD_R1D, MHD_R2D   # noqa: F401  (the harness fixture)

GOLD = os.path.join(os.path.dirname(__file__), "golden")
HYD = {"llf": 0, "exact": 1, "acoustic": 2, "hllc": 3, "hll": 4}


def _tree(r):
    m = r.m
    son = np.ascontiguousarray(r.son[1:], dtype=np.int32)
    father = np.ascontiguousarray(r.father[1:], dtype=np.int32)
    nbor = np.ascontiguousarray(r.nbor[:, 1:], dtype=np.int32)
    return (r.ncoarse, r.ngridmax, m.nx, m.ny, m.nz), (son, father, nbor)


def attach_emulated_hydro(r, orc, dev, riemann, slope_type, interpol_type):
    calls = [0]

    def c_godunov_fine(l):
        act = np.ascontiguousarray(r.active[l], dtype=np.int32)
        if len(act) == 0:
            return
        dims, (son, father, nbor) = _tree(r)
        dx = 0.5 ** l * r.p.boxlen / (r.m.icoarse_max - r.m.icoarse_min + 1)
        dev.devnum_amr_godunov(r.ndim, HYD[riemann], *dims, orc.iptr(son), orc.iptr(father), orc.iptr(nbor), orc.iptr(act), len(act), l,
                               orc.dptr(r.uold), orc.dptr(r.unew), r.dtnew[l], dx, interpol_type, slope_type, r.p.slope_theta, r.p.gamma, r.p.smallr,
                               r.p.smallc, 10, r.nvector)
        calls[0] += 1
    r.c_godunov_fine = c_godunov_fine
    return calls


def attach_emulated_mhd(r, orc, dev, ndim, riemann, riemann2d, slope_type, interpol_type):
    calls = [0]

    def c_godunov_fine(l):
        act = np.ascontiguousarray(r.active[l], dtype=np.int32)
        if len(act) == 0:
            return
        dims, (son, father, nbor) = _tree(r)
        dx = 0.5 ** l * r.p.boxlen / (r.m.icoarse_max - r.m.icoarse_min + 1)
        dev.devnum_mhd_amr_godunov(ndim, *dims, orc.iptr(son), orc.iptr(father), orc.iptr(nbor), orc.iptr(act), len(act), l,
                                   orc.dptr(r.uold), orc.dptr(r.unew), r.dtnew[l], dx, interpol_type, -1, MHD_R1D[riemann], MHD_R2D[riemann2d],
                                   slope_type, slope_type, r.pm.gamma, r.pm.smallr, r.pm.smallc, r.nvector)
        calls[0] += 1
    r.c_godunov_fine = c_godunov_fine
    return calls


@pytest.fixture(scope="module", autouse=True)
def _argtypes(dev):
    ip, dp = C.POINTER(C.c_int), C.POINTER(C.c_double)
    dev.devnum_amr_godunov.argtypes = [C.c_int] * 7 + [ip, ip, ip, ip, C.c_int, C.c_int, dp, dp, C.c_double, C.c_double, C.c_int, C.c_int,
                                       C.c_double, C.c_double, C.c_double, C.c_double, C.c_int, C.c_int]


def _same_run(a, b):
    assert a.t == b.t and a.nstep == b.nstep
    assert np.array_equal(a.son, b.son) and np.array_equal(a.nbor, b.nbor) and np.array_equal(a.father, b.father)
    assert np.array_equal(a.uold, b.uold)


def test_sod_tube_golden_from_the_device_code_on_the_cpu(orc, dev):
    from oracle.amr import AmrRun, check_sums
    from test_oracle_golden import SOD
    r = AmrRun(1, 3, 10, (1, 1, 0, 0, 0, 0), 1.0, nsubcycle=[1, 1, 1, 2], nexpand=1, ngridmax=2000, riemann="hllc",
               slope_type=2, gamma=1.4, courant_factor=0.8, err_grad_d=0.05, err_grad_u=0.05, err_grad_p=0.05,
               interpol_type=2, interpol_var=0, regions=SOD, tout=[0.245])
    calls = attach_emulated_hydro(r, orc, dev, "hllc", 2, 2)
    snap = r.run()
    ref = json.load(open(os.path.join(GOLD, "sod_tube_ref.json")))
    sums = check_sums(snap["rows"], 1)
    sums["time"] = snap["t"]
    for key in ("ncells", "level", "x", "density", "pressure", "velocity_x", "time"):
        err = abs(sums[key] - ref[key]) / min(abs(sums[key]), abs(ref[key]))
        assert err <= 3.0e-13, (key, sums[key], ref[key], err)
    assert snap["nstep_coarse"] == 43 and snap["nstep"] == 688 and calls[0] > 688


def test_imhd_tube_first_steps_device_code_equals_oracle(orc, dev):
    from oracle.amr_mhd import MhdAmrRun
    from test_oracle_golden import IMHD
    runs = []
    for emulated in (False, True):
        r = MhdAmrRun(5, 15, (2, 2, 0, 0, 0, 0), 3.5, nsubcycle=[1, 1, 1, 1], riemann="hlld", slope_type=0, gamma=1.6666667,
                      courant_factor=0.8, err_grad_d=0.01, err_grad_u=0.05, err_grad_p=0.05, interpol_type=2, regions=IMHD,
                      tout=[1e9], ngridmax=10000)
        calls = attach_emulated_mhd(r, orc, dev, 1, "hlld", "llf", 0, 2) if emulated else None
        r.run(max_coarse=25)
        runs.append(r)
    _same_run(*runs)
    assert calls[0] > 500 and sum(1 for l in range(1, 16) if runs[1].active[l]) >= 10


def test_implosion_first_steps_device_code_equals_oracle(orc, dev):
    from conftest import IMPL, IMPL_BOUND
    from oracle.amr import FastAmrRun
    runs = []
    for emulated in (False, True):
        r = FastAmrRun(2, 4, 6, (1, 1, 1, 1, 0, 0), 1.0, nsubcycle=[2] * 10, nexpand=[4], ngridmax=20000, riemann="hllc",
                       slope_type=2, gamma=1.4, courant_factor=0.8, err_grad_d=0.05, err_grad_u=0.05, err_grad_p=0.05,
                       interpol_type=2, interpol_var=0, regions=IMPL, tout=[1e9], bound_regions=IMPL_BOUND)
        calls = attach_emulated_hydro(r, orc, dev, "hllc", 2, 2) if emulated else None
        r.run(max_coarse=3)
        runs.append(r)
    _same_run(*runs)
    assert calls[0] >= 3 * 7 and len(runs[1].active[6]) > 0


def test_orszag_tang_first_steps_device_code_equals_oracle(orc, dev):
    from oracle.amr_mhd import MhdAmrRun2D
    runs = []
    for emulated in (False, True):
        r = MhdAmrRun2D(4, 6, 1.0, nsubcycle=[1, 2], riemann="hlld", riemann2d="hlld", slope_type=2, gamma=1.6666667, courant_factor=0.8,
                        err_grad_p=0.1, interpol_type=2, tout=[1e9], nexpand=1, ngridmax=20000)
        calls = attach_emulated_mhd(r, orc, dev, 2, "hlld", "hlld", 2, 2) if emulated else None
        r.run(max_coarse=4)
        runs.append(r)
    _same_run(*runs)
    assert runs[1].divb_max() < 5e-14 and len(runs[1].active[5]) > 0
