"""The DEVICE numerics (ramses_b200/csrc/hydro_device.cuh, real64.cuh, mhd_device.cuh -- the formulas the kernels execute)
compiled for the host by tests/host_numerics (g++, a stub <cuda_runtime.h>, RGPU_HOST_NUMERICS turning the three reciprocal /
sqrt / division primitives into the IEEE operations they are bit-identical to) and compared with the oracle BIT FOR BIT on the
CPU.  This is a test harness for machines without a GPU (a slip in a device formula shows up here before any GPU time is
spent); the parity tests proper remain the `-m gpu` tests through the C-ABI.  Nothing here is a product path."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from helpers import FLOORS

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_numerics")
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "ramses_b200", "csrc")


@pytest.fixture(scope="module")
def dev():
    lib = os.path.join(HERE, "libdevnum_host.so")
    srcs = [os.path.join(HERE, "devnum.cpp"), os.path.join(HERE, "stub", "cuda_runtime.h")] + \
        [os.path.join(CSRC, f) for f in ("hydro_device.cuh", "real64.cuh", "mhd_device.cuh", "amr_kernels.cuh", "sweep_dense.cuh",
                                        "sweep_dense3.cuh", "sweep_dense4.cuh", "hydro_vec.cuh", "mhd_dense.cuh", "mhd_amr.cuh", "amr_schedules.h")]
    if not os.path.exists(lib) or os.path.getmtime(lib) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-fno-fast-math", "-std=c++17", "-fPIC", "-shared", "-pthread",
                               "-fvisibility=hidden", "-fvisibility-inlines-hidden", "-Wl,-Bsymbolic",
                               "-I" + os.path.join(HERE, "stub"), "-I" + CSRC, "-o", lib, os.path.join(HERE, "devnum.cpp")])
    L = C.CDLL(lib, mode=os.RTLD_LOCAL | os.RTLD_NOW)
    dp = C.POINTER(C.c_double)
    L.devnum_riemann.argtypes = [C.c_int, C.c_int, C.c_int, dp, dp, dp, C.c_double, C.c_double, C.c_double, C.c_int]
    L.devnum_cmpdt.argtypes = [C.c_int, C.c_int, dp, C.c_double, dp, C.c_double, C.c_double, C.c_double, C.c_double]
    L.devnum_mhd_riemann.argtypes = [C.c_int, C.c_int, dp, dp, dp, C.c_double, C.c_double, C.c_double]
    L.devnum_mhd_emf.argtypes = [C.c_int, C.c_int, dp, dp, dp, dp, dp, C.c_double, C.c_double, C.c_double]
    L.devnum_mhd_cmpdt.argtypes = [C.c_int, dp, C.c_double, dp, C.c_double, C.c_double, C.c_double, C.c_double]
    L.devnum_unsplit3d.argtypes = [C.c_int, C.c_int, C.c_double, dp, C.c_double, C.c_double, dp, C.c_double, C.c_double, C.c_double,
                                   C.c_int]
    ip = C.POINTER(C.c_int)
    L.devnum_amr_get3cubefather.argtypes = [C.c_int] * 6 + [ip, ip, ip, C.c_int, ip, C.c_int, ip]
    L.devnum_amr_getnborfather.argtypes = [C.c_int] * 6 + [ip, ip, ip, C.c_int, ip, C.c_int, ip]
    L.devnum_amr_interpol.argtypes = [C.c_int, C.c_int, C.c_int, dp, dp]
    L.devnum_amr_godfine.argtypes = [C.c_int] * 7 + [ip, ip, ip, ip, C.c_int, C.c_int, dp, dp, dp, C.c_double, C.c_double, C.c_int,
                                     C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int, C.c_double]
    L.devnum_amr_godfine_src.argtypes = [C.c_int] * 7 + [ip, ip, ip, ip, C.c_int, C.c_int, dp, dp, dp, C.c_double, C.c_double, C.c_int,
                                         C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int, dp, C.c_int, C.c_int]
    L.devnum_amr_src_pass.argtypes = [C.c_int] * 7 + [ip, ip, ip, ip, C.c_int, dp, dp, dp, dp, dp] + [C.c_double] * 5
    L.devnum_cmpdt_grav.argtypes = [C.c_int, C.c_int, dp, dp, C.c_double, dp, C.c_double, C.c_double, C.c_double, C.c_double]
    L.devnum_riemann_eflux.argtypes = [C.c_int, C.c_int, C.c_int, dp, dp, dp, C.c_double, C.c_double, C.c_double, C.c_int]
    L.devnum_mhd_amr_godunov.argtypes = [C.c_int] * 6 + [ip, ip, ip, ip, C.c_int, C.c_int, dp, dp, C.c_double, C.c_double] + [C.c_int] * 6 + \
        [C.c_double] * 3 + [C.c_int]
    L.devnum_mhd_amr_pass.argtypes = [C.c_int] * 7 + [ip, ip, ip, ip, C.c_int, dp] + [C.c_double] * 5 + [C.c_int, C.c_int, dp]
    i3 = C.c_int * 3
    L.devnum_sweep3_box.argtypes = [C.c_int, i3, i3, C.c_int, dp, dp] + [C.c_double] * 2 + [C.c_int] + [C.c_double] * 5 + \
        [C.c_int, dp, C.c_int, C.c_int]
    L.devnum_sweep_dense_box.argtypes = [C.c_int, C.c_int, i3, i3, C.c_int, dp, dp] + [C.c_double] * 2 + [C.c_int] + \
        [C.c_double] * 5 + [C.c_int, dp, C.c_int]
    L.devnum_sweep_dense_amr_box.argtypes = [C.c_int, i3, i3, C.c_int, dp, dp, C.POINTER(C.c_ubyte)] + [C.c_double] * 2 + \
        [C.c_int] + [C.c_double] * 4 + [C.c_int]
    L.devnum_mhd_sweep_box.argtypes = [i3, i3, C.c_int, C.c_int, C.c_int, dp, dp] + [C.c_double] * 5 + [C.c_int, C.c_int] + \
        [C.c_double] * 2
    return L


def _hydro_states(rng, n, ndim):
    """left/right primitive states in solver order (rho, u_n, P, u_t...): smooth pairs, strong shocks, near-vacuum, supersonic"""
    nv = ndim + 2
    ql, qr = np.zeros((n, nv)), np.zeros((n, nv))
    for q in (ql, qr):
        q[:, 0] = 10.0 ** rng.uniform(-3, 2, n)
        q[:, 2] = 10.0 ** rng.uniform(-5, 3, n)
        q[:, 1] = rng.standard_normal(n) * 10.0 ** rng.uniform(-2, 1.5, n)
        for k in range(3, nv):
            q[:, k] = rng.standard_normal(n)
    k = n // 4
    qr[:k] = ql[:k] * (1 + 1e-3 * rng.standard_normal((k, nv)))       # nearly equal states
    qr[k:2 * k, 0] = ql[k:2 * k, 0]
    ql[2 * k:2 * k + 50, 0] = 1e-12                                     # below smallr
    ql[2 * k + 50:2 * k + 100, 2] = 1e-30                               # below the pressure floor
    ql[2 * k + 100:2 * k + 200, 2] = qr[2 * k + 100:2 * k + 200, 2] = 1e-30 # both sides at the pressure floor
    ql[2 * k + 150:2 * k + 200, 0] = 1e-12                              # ... and at the density floor on one side
    # strong rarefactions out of thin, cold gas: the star state of exact / acoustic has rstar < smallr and cstar < smallc
    j, m = slice(2 * k + 200, 2 * k + 400), 200
    ql[j, 0], qr[j, 0] = 10.0 ** rng.uniform(-8, -3, m), 10.0 ** rng.uniform(-8, -3, m)
    ql[j, 2], qr[j, 2] = 10.0 ** rng.uniform(-16, -8, m), 10.0 ** rng.uniform(-16, -8, m)
    ql[j, 1], qr[j, 1] = -(10.0 ** rng.uniform(-1, 2, m)), 10.0 ** rng.uniform(-1, 2, m)
    return np.ascontiguousarray(ql), np.ascontiguousarray(qr)


@pytest.mark.parametrize("ndim", [1, 2, 3])
@pytest.mark.parametrize("solver", ["llf", "exact", "acoustic", "hllc", "hll"])
def test_hydro_riemann_device_formulas_equal_oracle(orc, dev, ndim, solver):
    """riemann_{llf,approx,acoustic,hllc,hll} of hydro_device.cuh == the oracle's restatement of hydro/godunov_utils.f90,
    bit for bit on 20 000 random face states -- including `exact`, whose only GPU-side deviation is CUDA's pow()."""
    n, nv = 20000, ndim + 2
    ql, qr = _hydro_states(np.random.default_rng(ndim * 10 + len(solver)), n, ndim)
    sid = {"llf": 0, "exact": 1, "acoustic": 2, "hllc": 3, "hll": 4}[solver]
    L = orc.lib()
    f = {"llf": L.orc_riemann_llf, "exact": L.orc_riemann_approx, "acoustic": L.orc_riemann_acoustic, "hllc": L.orc_riemann_hllc,
         "hll": L.orc_riemann_hll}[solver]
    f.argtypes = [C.POINTER(orc.Params), C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int]
    for smallr, smallc in FLOORS.values():
        fg = np.zeros((n, nv))
        dev.devnum_riemann(ndim, sid, n, orc.dptr(ql), orc.dptr(qr), orc.dptr(fg), 1.4, smallr, smallc, 10)
        p = orc.make_params(ndim=ndim, riemann=solver, nvector=n, niter_riemann=10, smallr=smallr, smallc=smallc)
        qlf, qrf = np.asfortranarray(ql), np.asfortranarray(qr)              # (nvector, nvar) column-major
        fgf = np.zeros((n, nv + 1), order="F")
        f(C.byref(p), qlf.ctypes.data_as(C.POINTER(C.c_double)), qrf.ctypes.data_as(C.POINTER(C.c_double)),
          fgf.ctypes.data_as(C.POINTER(C.c_double)), n)
        assert np.isfinite(fg).all()
        assert np.array_equal(fg, fgf[:, :nv])
        # the internal-energy flux fgdnv(nvar+1) that only pressure_fix consumes (tmp2 of cmpflxm, umuscl.f90:848)
        fe = np.zeros(n)
        dev.devnum_riemann_eflux(ndim, sid, n, orc.dptr(ql), orc.dptr(qr), orc.dptr(fe), 1.4, smallr, smallc, 10)
        assert np.isfinite(fe).all() and np.abs(fe).max() > 0
        assert np.array_equal(fe, fgf[:, nv])


def _with_floor_cells(u, rng, ndim, k=400):
    """u (n, ndim+2) conservative cells plus k cells on the floors of cmpdt (hydro/godunov_utils.f90:25,64) under both settings of
    helpers.FLOORS: densities 1e-13-1e-4 (below smallr), and cold cells whose (gamma-1) e is below rho * smallp -- E = ekin (1 -
    delta) with delta in {0, 1e-14, 1e-3}, or a specific internal energy of 1e-24-1e-5"""
    nv = ndim + 2
    f = np.zeros((2 * k, nv))
    f[:, 0] = 10.0 ** rng.uniform(-4, 0, 2 * k)
    f[:k, 0] = 10.0 ** rng.uniform(-13, -4, k)
    vel = rng.standard_normal((2 * k, ndim)) * 10.0 ** rng.uniform(-2, 1, (2 * k, 1))
    f[:, 1:1 + ndim] = f[:, :1] * vel
    ekin = 0.5 * f[:, 0] * (vel ** 2).sum(axis=1)
    f[:, nv - 1] = ekin + f[:, 0] * 10.0 ** rng.uniform(-5, 0, 2 * k)
    f[k:, nv - 1] = np.where(rng.random(k) < 0.5, ekin[k:] * (1 - rng.choice([0.0, 1e-14, 1e-3], k)),
                             ekin[k:] + f[k:, 0] * 10.0 ** rng.uniform(-24, -5, k))
    return np.ascontiguousarray(np.concatenate([u, f]))


def _assert_cmpdt_floors_fire(u, ndim, smallr, smallc, gamma=1.4):
    r = np.maximum(u[:, 0], smallr)
    e = u[:, ndim + 1] - 0.5 * r * sum((u[:, 1 + d] / r) ** 2 for d in range(ndim))
    assert (u[:, 0] < smallr).sum() >= 100
    assert ((gamma - 1) * e < r * smallc ** 2 / gamma).sum() >= 100


@pytest.mark.parametrize("ndim", [1, 2, 3])
def test_hydro_cmpdt_with_gravity_device_formula_equals_oracle(orc, dev, ndim):
    """cmpdt with the gravity strength ratio (hydro/godunov_utils.f90:99-111): weak, comparable and dominant accelerations."""
    n, nv = 5000, ndim + 2
    rng = np.random.default_rng(55 + ndim)
    u = np.zeros((n, nv))
    u[:, 0] = 10.0 ** rng.uniform(-3, 2, n)
    vel = rng.standard_normal((n, ndim)) * 3
    u[:, 1:1 + ndim] = u[:, :1] * vel
    u[:, nv - 1] = 10.0 ** rng.uniform(-4, 2, n) + 0.5 * u[:, 0] * (vel ** 2).sum(axis=1)
    u = _with_floor_cells(u, rng, ndim)
    n = len(u)
    g = rng.standard_normal((n, ndim)) * 10.0 ** rng.uniform(-3, 5, (n, 1))
    g[:50] = 0.0
    dx = 1.0 / 128
    gsum = np.zeros(n)
    for d in range(ndim):                      # uu(k,1) = uu(k,1) + abs(gg(k,idim)) in this order
        gsum = gsum + np.abs(g[:, d])
    L = orc.lib()
    L.orc_cmpdt.argtypes = [C.POINTER(orc.Params), C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_double, C.POINTER(C.c_double), C.c_int]
    for smallr, smallc in FLOORS.values():
        dt = np.zeros(n)
        dev.devnum_cmpdt_grav(ndim, n, orc.dptr(np.ascontiguousarray(u)), orc.dptr(gsum), dx, orc.dptr(dt), 1.4, smallr, smallc, 0.8)
        p = orc.make_params(ndim=ndim, nvector=1, courant_factor=0.8, smallr=smallr, smallc=smallc)
        ref = np.zeros(n)
        for i in range(n):
            uu = u[i].copy()
            gg = np.zeros(3)
            gg[:ndim] = g[i]
            o = C.c_double(0)
            L.orc_cmpdt(C.byref(p), orc.dptr(uu), orc.dptr(gg), dx, C.byref(o), 1)
            ref[i] = o.value
        assert np.isfinite(ref).all()
        assert np.array_equal(dt, ref)
        assert (dt[50:] < 0.999 * dt[:50].max()).any()
        _assert_cmpdt_floors_fire(u, ndim, smallr, smallc)


@pytest.mark.parametrize("ndim", [1, 2, 3])
def test_hydro_cmpdt_device_formula_equals_oracle(orc, dev, ndim):
    n, nv = 5000, ndim + 2
    rng = np.random.default_rng(5 + ndim)
    u = np.zeros((n, nv))
    u[:, 0] = 10.0 ** rng.uniform(-3, 2, n)
    vel = rng.standard_normal((n, ndim)) * 3
    u[:, 1:1 + ndim] = u[:, :1] * vel
    u[:, nv - 1] = 10.0 ** rng.uniform(-4, 2, n) + 0.5 * u[:, 0] * (vel ** 2).sum(axis=1)
    u = _with_floor_cells(u, rng, ndim)
    n = len(u)
    dx = 1.0 / 128
    L = orc.lib()
    L.orc_cmpdt.argtypes = [C.POINTER(orc.Params), C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_double, C.POINTER(C.c_double), C.c_int]
    for smallr, smallc in FLOORS.values():
        dt = np.zeros(n)
        dev.devnum_cmpdt(ndim, n, orc.dptr(np.ascontiguousarray(u)), dx, orc.dptr(dt), 1.4, smallr, smallc, 0.8)
        p = orc.make_params(ndim=ndim, nvector=1, courant_factor=0.8, smallr=smallr, smallc=smallc)
        ref = np.zeros(n)
        for i in range(n):
            uu = u[i].copy()
            d = C.c_double(0.0)
            L.orc_cmpdt(C.byref(p), orc.dptr(uu), None, dx, C.byref(d), 1)
            ref[i] = d.value
        assert np.isfinite(ref).all()
        assert np.array_equal(dt, ref)
        _assert_cmpdt_floors_fire(u, ndim, smallr, smallc)


def _mhd_states(rng, n):
    """(rho, P, v_n, B_n, v_t1, B_t1, v_t2, B_t2) left/right with a common B_n"""
    ql, qr = np.zeros((n, 8)), np.zeros((n, 8))
    for q in (ql, qr):
        q[:, 0] = 10.0 ** rng.uniform(-2, 1, n)
        q[:, 1] = 10.0 ** rng.uniform(-3, 2, n)
        q[:, 2], q[:, 4], q[:, 6] = (rng.standard_normal(n) * 2 for _ in range(3))
        q[:, 5], q[:, 7] = rng.standard_normal(n), rng.standard_normal(n)
    bn = rng.standard_normal(n)
    bn[: n // 10] = 0.0
    ql[:, 3], qr[:, 3] = bn, bn
    k = n // 5
    qr[:k] = ql[:k] * (1 + 1e-3 * rng.standard_normal((k, 8)))
    qr[:k, 3] = ql[:k, 3]
    return np.ascontiguousarray(ql), np.ascontiguousarray(qr)


MHD_CLASSES = ("vacuum", "pfloor", "free", "aligned_fast", "aligned_slow", "mdom", "tiny_bt")


def _mhd_degenerate_states(rng, k, gamma=5 / 3.):
    """k left/right pairs per degenerate class, in the solver order of _mhd_states (equal B_n on both sides):
    vacuum -- densities 1e-12-1e-3, one side or both, below smallr under both helpers.FLOORS settings;
    pfloor -- pressure 0 or 1e-40 on one side or both (hydro_acoustic's pressure floor);
    free -- B = 0 on both sides; half of them strong rarefactions out of thin, cold gas (rstar / cstar of hydro_acoustic floored);
    aligned_fast / aligned_slow -- B = (B_n, 0, 0) with vA^2 / c_s^2 in 2-20 / 0.05-0.5 (never 1), a third of the pairs with
      equal sides (the HLLD star state degenerates: |estar| < 1e-4 B_n^2), a third nearly equal;
    mdom -- near-vacuum magnetically dominated, plasma beta 1e-20-1e-6;
    tiny_bt -- tangential fields 1e-16-1e-6 next to an O(1) normal field.
    Returns ql, qr and {class: row slice}."""
    rows, cls = [], {}
    for name in MHD_CLASSES:
        l, r = _mhd_states(rng, k)
        if name == "vacuum":
            l[:, 0] = 10.0 ** rng.uniform(-12, -3, k)
            both = rng.random(k) < 0.5
            r[both, 0] = 10.0 ** rng.uniform(-12, -3, int(both.sum()))
        elif name == "pfloor":
            l[:, 1] = rng.choice([0.0, 1e-40], k)
            both = rng.random(k) < 0.5
            r[both, 1] = rng.choice([0.0, 1e-40], int(both.sum()))
        elif name == "free":
            l[:, [3, 5, 7]] = 0.0
            r[:, [3, 5, 7]] = 0.0
            h = k // 2
            l[:h, 0], r[:h, 0] = 10.0 ** rng.uniform(-12, -3, h), 10.0 ** rng.uniform(-12, -3, h)
            l[:h, 1], r[:h, 1] = 10.0 ** rng.uniform(-30, -12, h), 10.0 ** rng.uniform(-30, -12, h)
            l[:h, 2], r[:h, 2] = -(10.0 ** rng.uniform(-1, 2, h)), 10.0 ** rng.uniform(-1, 2, h)
        elif name in ("aligned_fast", "aligned_slow"):
            for q in (l, r):
                q[:, [5, 7]] = 0.0
            bn = rng.uniform(0.2, 2.0, k) * rng.choice([-1.0, 1.0], k)
            l[:, 3] = r[:, 3] = bn
            ratio = rng.uniform(2.0, 20.0, k) if name == "aligned_fast" else rng.uniform(0.05, 0.5, k)
            for q in (l, r):
                q[:, 1] = bn ** 2 / (gamma * ratio)
            t = k // 3
            r[:t] = l[:t]
            r[t:2 * t] = l[t:2 * t] * (1 + 1e-6 * rng.standard_normal((t, 8)))
            r[t:2 * t, [3, 5, 7]] = l[t:2 * t, [3, 5, 7]]
            for q in (l, r):
                q[:, 1] = q[:, 3] ** 2 / (gamma * ratio)
            zt = rng.random(k) < 0.5                          # half of them move along the field only
            l[zt, 4] = l[zt, 6] = r[zt, 4] = r[zt, 6] = 0.0
        elif name == "mdom":
            for q in (l, r):
                q[:, 0] = 10.0 ** rng.uniform(-11, -6, k)
                q[:, 1] = 0.5 * (q[:, 3] ** 2 + q[:, 5] ** 2 + q[:, 7] ** 2) * 10.0 ** rng.uniform(-20, -6, k)
        else:
            for q in (l, r):
                q[:, [5, 7]] = rng.standard_normal((k, 2)) * 10.0 ** rng.uniform(-16, -6, (k, 1))
            bn = rng.uniform(0.2, 2.0, k)
            l[:, 3] = r[:, 3] = bn
        cls[name] = slice(len(rows) * k, (len(rows) + 1) * k)
        rows.append((l, r))
    ql = np.concatenate([a for a, _ in rows])
    qr = np.concatenate([b for _, b in rows])
    return np.ascontiguousarray(ql), np.ascontiguousarray(qr), cls


def _assert_mhd_classes_present(ql, qr, cls, smallr, smallc, gamma=5 / 3.):
    """every degenerate class of _mhd_degenerate_states is in the inputs, and its defining property holds"""
    smallp = smallr * smallc ** 2 / gamma
    q = {n: (ql[s], qr[s]) for n, s in cls.items()}
    assert (q["vacuum"][0][:, 0] < smallr).sum() >= 10
    assert (q["pfloor"][0][:, 1] < smallp).all()
    assert all((a[:, [3, 5, 7]] == 0).all() for a in q["free"])
    for name, fast in (("aligned_fast", True), ("aligned_slow", False)):
        l, r = q[name]
        assert (l[:, [5, 7]] == 0).all() and (r[:, [5, 7]] == 0).all() and (l[:, 3] != 0).all()
        va2, cs2 = l[:, 3] ** 2 / l[:, 0], gamma * l[:, 1] / l[:, 0]
        assert ((va2 > 1.5 * cs2) if fast else (va2 < 0.6 * cs2)).all()
        assert (l == r).all(axis=1).sum() > 0
    l, _ = q["mdom"]
    assert (2 * l[:, 1] / (l[:, 3] ** 2 + l[:, 5] ** 2 + l[:, 7] ** 2)).min() < 1e-18
    assert (np.abs(q["tiny_bt"][0][:, 5]) < 1e-12).sum() > 0


@pytest.mark.parametrize("solver", ["llf", "roe", "hll", "hlld", "upwind", "hydro"])
def test_mhd_riemann_device_formulas_equal_oracle(orc, dev, solver):
    """lax_friedrich / athena_roe (restructured on the device: left eigenvectors column by column, shared reciprocals) / hll /
    hlld / upwind / hydro_acoustic of mhd_device.cuh == the oracle's restatement of mhd/godunov_utils.f90, bit for bit on every
    row and no row NaN, under both helpers.FLOORS settings: random pairs plus the degenerate
    classes of _mhd_degenerate_states (near-vacuum, floored pressure, zero field, field along the normal with vA above and below
    c_s, beta down to 1e-20, tiny tangential fields).  Roe falls back to the LLF flux on some rows (unphysical intermediate
    state); the count of those rows is asserted and reported."""
    n, k = 20000, 600
    rng = np.random.default_rng(40 + len(solver))
    ql0, qr0 = _mhd_states(rng, n)
    qld, qrd, cls = _mhd_degenerate_states(rng, k)
    ql, qr = np.concatenate([ql0, qld]), np.concatenate([qr0, qrd])
    cls = {c: slice(s.start + n, s.stop + n) for c, s in cls.items()}
    n = len(ql)
    L = orc.lib()
    L.orc_mhd_riemann.argtypes = [C.POINTER(orc.MhdParams)] + [C.POINTER(C.c_double)] * 3
    for smallr, smallc in FLOORS.values():
        _assert_mhd_classes_present(ql, qr, cls, smallr, smallc)
        fg = np.zeros((n, 9))
        dev.devnum_mhd_riemann(orc.MHD_RIEMANN[solver], n, orc.dptr(ql), orc.dptr(qr), orc.dptr(fg), 5 / 3., smallr, smallc)
        pm = orc.make_mhd_params(riemann=solver, gamma=5 / 3., smallr=smallr, smallc=smallc)
        ref = np.zeros((n, 9))
        for i in range(n):
            L.orc_mhd_riemann(C.byref(pm), orc.dptr(ql[i]), orc.dptr(qr[i]), orc.dptr(ref[i]))
        nan = ~np.isfinite(ref[:, :8]).all(axis=1)
        print(f"{solver} smallr={smallr:g}: {int(nan.sum())} non-finite rows of {n}")
        assert not nan.any()
        assert np.array_equal(fg[:, :8], ref[:, :8], equal_nan=True), \
            [c for c, s in cls.items() if not np.array_equal(fg[s, :8], ref[s, :8], equal_nan=True)]
        if solver == "roe":
            fl = np.zeros((n, 9))
            dev.devnum_mhd_riemann(orc.MHD_RIEMANN["llf"], n, orc.dptr(ql), orc.dptr(qr), orc.dptr(fl), 5 / 3., smallr, smallc)
            nllf = int((fl[:, :8] == fg[:, :8]).all(axis=1).sum())
            print(f"roe rows equal to the LLF flux (unphysical intermediate state): {nllf}")
            assert nllf > 0


def _emf_corners(rng, n):
    """RT, RB, LT, LB corner states (rho, u, v, w, P, A, B, C) of the E_z edge"""
    RT, RB, LT, LB = (np.zeros((n, 8)) for _ in range(4))
    for q in (RT, RB, LT, LB):
        q[:, 0] = 10.0 ** rng.uniform(-1, 1, n)
        q[:, 4] = 10.0 ** rng.uniform(-2, 1, n)
        q[:, 1:4] = rng.standard_normal((n, 3))
        q[:, 5:8] = rng.standard_normal((n, 3))
    return RT, RB, LT, LB


def _emf_degenerate_corners(rng, k, gamma=5 / 3.):
    """k edges per class: vacuum (corner densities 1e-12-1e-3), free (all fields zero), tiny (fields 1e-16-1e-6: the Alfven
    speeds of 2-D HLLD fall below smallc), aligned (B along x or y only, vA^2 / c_s^2 in 2-20 or 0.05-0.5), mdom (beta down to
    1e-20); returns the four corner arrays and {class: row slice}"""
    parts, cls = [], {}
    for j, name in enumerate(("vacuum", "free", "tiny", "aligned", "mdom")):
        c = _emf_corners(rng, k)
        for q in c:
            if name == "vacuum":
                q[:, 0] = 10.0 ** rng.uniform(-12, -3, k)
            elif name == "free":
                q[:, 5:8] = 0.0
            elif name == "tiny":
                q[:, 5:8] *= 10.0 ** rng.uniform(-16, -6, (k, 1))
            elif name == "mdom":
                q[:, 0] = 10.0 ** rng.uniform(-11, -6, k)
                q[:, 4] = 0.5 * (q[:, 5:8] ** 2).sum(axis=1) * 10.0 ** rng.uniform(-20, -6, k)
        if name == "aligned":
            ax = np.where(rng.random(k) < 0.5, 5, 6)
            b = rng.uniform(0.2, 2.0, k)
            ratio = np.where(rng.random(k) < 0.5, rng.uniform(2.0, 20.0, k), rng.uniform(0.05, 0.5, k))
            for q in c:
                q[:, 5:8] = 0.0
                q[np.arange(k), ax] = b
                q[:, 4] = b ** 2 / (gamma * ratio)
        cls[name] = slice(j * k, (j + 1) * k)
        parts.append(c)
    return tuple(np.concatenate([p[i] for p in parts]) for i in range(4)), cls


@pytest.mark.parametrize("solver2d", ["llf", "roe", "upwind", "hll", "hlla", "hlld"])
def test_mhd_corner_emf_device_formulas_equal_oracle(orc, dev, solver2d):
    """emf_edge<R2D> (cmp_mag_flx, mhd/umuscl.f90:1453) for the E_z call: the four corner states in the reference's dummy-argument
    order; the oracle is called with the cell-order corner states of the same edge.  Random edges plus near-vacuum, field-free,
    tiny-field (the smallc floor of the 2-D HLLD Alfven speeds), axis-aligned and magnetically dominated edges, under both
    helpers.FLOORS settings: every row bit for bit and finite on both sides"""
    n, k = 10000, 400
    rng = np.random.default_rng(77 + len(solver2d))
    RT, RB, LT, LB = _emf_corners(rng, n)
    (dRT, dRB, dLT, dLB), cls = _emf_degenerate_corners(rng, k)
    RT, RB, LT, LB = (np.concatenate([a, b]) for a, b in ((RT, dRT), (RB, dRB), (LT, dLT), (LB, dLB)))
    cls = {c: slice(s.start + n, s.stop + n) for c, s in cls.items()}
    n = len(RT)
    for q in (RT, RB, LT, LB):
        assert (q[cls["free"], 5:8] == 0).all() and (np.abs(q[cls["tiny"], 5:8]) < 1e-5).all()
        assert (q[cls["vacuum"], 0] < 1e-10).sum() > 0
        a = q[cls["aligned"]]
        assert ((a[:, 5:8] != 0).sum(axis=1) == 1).all() and (a[:, 7] == 0).all()
        va2, cs2 = (a[:, 5:8] ** 2).sum(axis=1) / a[:, 0], 5 / 3. * a[:, 4] / a[:, 0]
        assert ((va2 > 1.5 * cs2) | (va2 < 0.6 * cs2)).all() and (va2 > 1.5 * cs2).any() and (va2 < 0.6 * cs2).any()
        md = q[cls["mdom"]]
        assert (2 * md[:, 4] / (md[:, 5:8] ** 2).sum(axis=1)).min() < 1e-18
    # face fields are shared: A (x-face) by the left/right pair, B (y-face) by the top/bottom pair (umuscl.f90:1506-1541)
    lp1, lp2, lor, bp1, bp2, bor = 2, 3, 4, 6, 7, 8
    LL, RL, LR, RR = (np.zeros((n, 8)) for _ in range(4))
    for dst, src in ((LL, RT), (RL, LT), (LR, RB), (RR, LB)):
        dst[:, 0], dst[:, 1] = src[:, 0], src[:, 4]
        dst[:, 2], dst[:, 3], dst[:, 4], dst[:, 7] = src[:, lp1 - 1], src[:, lp2 - 1], src[:, lor - 1], src[:, bor - 1]
    LL[:, 5] = RL[:, 5] = 0.5 * (RT[:, bp1 - 1] + LT[:, bp1 - 1])
    LR[:, 5] = RR[:, 5] = 0.5 * (RB[:, bp1 - 1] + LB[:, bp1 - 1])
    LL[:, 6] = LR[:, 6] = 0.5 * (RT[:, bp2 - 1] + RB[:, bp2 - 1])
    RL[:, 6] = RR[:, 6] = 0.5 * (LT[:, bp2 - 1] + LB[:, bp2 - 1])
    L = orc.lib()
    L.orc_mhd_emf.restype = C.c_double
    L.orc_mhd_emf.argtypes = [C.POINTER(orc.MhdParams)] + [C.POINTER(C.c_double)] * 4 + [C.c_int]
    for smallr, smallc in FLOORS.values():
        emf = np.zeros(n)
        dev.devnum_mhd_emf(orc.MHD_RIEMANN2D[solver2d], n, *(orc.dptr(np.ascontiguousarray(a)) for a in (LL, RL, LR, RR)),
                           orc.dptr(emf), 5 / 3., smallr, smallc)
        pm = orc.make_mhd_params(riemann2d=solver2d, gamma=5 / 3., smallr=smallr, smallc=smallc)
        ref = np.array([L.orc_mhd_emf(C.byref(pm), orc.dptr(RT[i]), orc.dptr(RB[i]), orc.dptr(LT[i]), orc.dptr(LB[i]), 2)
                        for i in range(n)])
        nan = ~np.isfinite(ref)
        print(f"{solver2d} smallr={smallr:g}: {int(nan.sum())} non-finite rows of {n}")
        assert not nan.any()
        assert np.array_equal(emf, ref, equal_nan=True), \
            [c for c, s in cls.items() if not np.array_equal(emf[s], ref[s], equal_nan=True)]


def _mhd_cmpdt_cells(rng, n, k=300, gamma=5 / 3.):
    """n ordinary cells [11] plus k cells per class: densities 1e-13-1e-4 (below smallr), cold magnetised E = ekin + emag (1 -
    delta), field-free, field along x, y or z with vA^2 / c_s^2 in 2-20 or 0.05-0.5, magnetically dominated near-vacuum"""
    u = np.zeros((n + 5 * k, 11))
    u[:, 0] = 10.0 ** rng.uniform(-2, 1, len(u))
    vel = rng.standard_normal((len(u), 3)) * 2
    u[:, 5:8] = rng.standard_normal((len(u), 3))
    u[:, 8:11] = u[:, 5:8] + 0.1 * rng.standard_normal((len(u), 3))
    P = 10.0 ** rng.uniform(-3, 1, len(u))
    s = [slice(n + j * k, n + (j + 1) * k) for j in range(5)]
    u[s[0], 0] = 10.0 ** rng.uniform(-13, -4, k)
    u[s[2], 5:11] = 0.0
    ax = rng.integers(0, 3, k)
    b = rng.uniform(0.2, 2.0, k)
    u[s[3], 5:11] = 0.0
    rows = np.arange(s[3].start, s[3].stop)
    u[rows, 5 + ax] = u[rows, 8 + ax] = b
    ratio = np.where(rng.random(k) < 0.5, rng.uniform(2.0, 20.0, k), rng.uniform(0.05, 0.5, k))
    P[s[3]] = b ** 2 / (gamma * ratio)
    u[s[4], 0] = 10.0 ** rng.uniform(-11, -6, k)
    bc = 0.5 * (u[:, 5:8] + u[:, 8:11])
    emag = 0.5 * (bc ** 2).sum(axis=1)
    P[s[4]] = (emag * 10.0 ** rng.uniform(-20, -6, len(u)))[s[4]]
    u[:, 1:4] = u[:, :1] * vel
    ekin = 0.5 * u[:, 0] * (vel ** 2).sum(axis=1)
    u[:, 4] = P / (gamma - 1) + ekin + emag
    u[s[1], 4] = (ekin + emag * (1 - rng.choice([0.0, 1e-14, 1e-3], len(u))))[s[1]]
    return np.ascontiguousarray(u), s


def test_mhd_cmpdt_device_formula_equals_oracle(orc, dev):
    """cmpdt of the MHD build (mhd/godunov_utils.f90:5-111) on ordinary cells plus cells below smallr, cold magnetised cells whose
    pressure floor fires, field-free, axis-aligned and magnetically dominated cells, under both helpers.FLOORS settings: every
    time step bit for bit, the oracle finite"""
    rng = np.random.default_rng(9)
    u, s = _mhd_cmpdt_cells(rng, 5000)
    n = len(u)
    dx = 1.0 / 64
    L = orc.lib()
    L.orc_mhd_cmpdt_cell.restype = C.c_double
    L.orc_mhd_cmpdt_cell.argtypes = [C.POINTER(orc.MhdParams), C.POINTER(C.c_double), C.c_double]
    for smallr, smallc in FLOORS.values():
        dt = np.zeros(n)
        dev.devnum_mhd_cmpdt(n, orc.dptr(u), dx, orc.dptr(dt), 5 / 3., smallr, smallc, 0.8)
        pm = orc.make_mhd_params(gamma=5 / 3., courant_factor=0.8, smallr=smallr, smallc=smallc)
        ref = np.array([L.orc_mhd_cmpdt_cell(C.byref(pm), orc.dptr(u[i].copy()), dx) for i in range(n)])
        assert np.isfinite(ref).all()
        assert np.array_equal(dt, ref)
        nrho, npr, nfree, nfast = _cmpdt_cell_counts(u, smallr, smallc)
        assert min(nrho, npr, nfree, nfast) >= 50, (nrho, npr, nfree, nfast)


def _cmpdt_cell_counts(u, smallr, smallc, gamma=5 / 3.):
    """mhd_floor_counts of the cells u [n][11], with the field-aligned count taken over the three axes"""
    from helpers import mhd_floor_counts
    nrho, npr, nfree, _ = mhd_floor_counts(u.T.reshape(11, 1, 1, -1), smallr, smallc)
    nfast = 0
    for ax in range(3):
        p3 = np.array([ax, (ax + 1) % 3, (ax + 2) % 3])        # the field axis becomes x
        w = u[:, np.concatenate([[0], 1 + p3, [4], 5 + p3, 8 + p3])]
        nfast += mhd_floor_counts(w.T.reshape(11, 1, 1, -1), smallr, smallc)[3]
    return nrho, npr, nfree, nfast


@pytest.mark.parametrize("solver", ["hllc", "llf", "exact", "acoustic", "hll"])
@pytest.mark.parametrize("slope_type", [0, 1, 2, 7, 8])
def test_unsplit_from_device_pieces_equals_oracle_unsplit(orc, dev, solver, slope_type):
    """ctoprim -> slope_lcr -> trace_sources -> trace_faces -> riemann -> flux*dt/dx assembled from the per-cell DEVICE functions
    on 6^3 patches == unsplit of the oracle (hydro/umuscl.f90:22), bit for bit, for the 36 faces of every patch"""
    L = orc.lib()
    L.orc_work_new.restype = C.c_void_p
    L.orc_work_new.argtypes = [C.POINTER(orc.Params)]
    L.orc_work_free.argtypes = [C.c_void_p]
    dp = C.POINTER(C.c_double)
    L.orc_unsplit.argtypes = [C.POINTER(orc.Params), C.c_void_p, dp, dp, dp, dp, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int]
    p = orc.make_params(ndim=3, riemann=solver, slope_type=slope_type, slope_theta=1.3, nvector=1, niter_riemann=10)
    w = L.orc_work_new(C.byref(p))
    rng = np.random.default_rng(100 + slope_type)
    sid = {"llf": 0, "exact": 1, "acoustic": 2, "hllc": 3, "hll": 4}[solver]
    dx = 1.0 / 64
    for trial in range(12):
        rho = 1 + 0.5 * rng.random((6, 6, 6))
        if trial % 3 == 0:
            rho[3:] *= 8.0                                             # a jump through the patch
        vel = (0.5 if trial % 2 else 3.0) * rng.standard_normal((3, 6, 6, 6))
        pres = 10.0 ** rng.uniform(-2, 1, (6, 6, 6))
        uin = np.zeros((5, 216))
        uin[0] = rho.reshape(-1)
        for k in range(3):
            uin[1 + k] = (rho * vel[k]).reshape(-1)
        uin[4] = (pres / 0.4 + 0.5 * rho * (vel ** 2).sum(axis=0)).reshape(-1)
        uin = np.ascontiguousarray(uin)
        dt = 0.3 * dx / 5.0
        f_dev = np.zeros(3 * 5 * 27)
        dev.devnum_unsplit3d(sid, slope_type, 1.3, orc.dptr(uin), dx, dt, orc.dptr(f_dev), 1.4, 1e-10, 1e-10, 10)
        f_orc = np.zeros(3 * 5 * 27)
        tmp = np.zeros(3 * 2 * 27)
        L.orc_unsplit(C.byref(p), w, orc.dptr(uin), None, orc.dptr(f_orc), orc.dptr(tmp), dx, dx, dx, dt, 1)
        fd, fo = f_dev.reshape(3, 5, 3, 3, 3), f_orc.reshape(3, 5, 3, 3, 3)      # [idim][ivar][k3][j3][i3]
        assert np.array_equal(fd[0][:, 0:2, 0:2, 0:3], fo[0][:, 0:2, 0:2, 0:3])
        assert np.array_equal(fd[1][:, 0:2, 0:3, 0:2], fo[1][:, 0:2, 0:3, 0:2])
        assert np.array_equal(fd[2][:, 0:3, 0:2, 0:2], fo[2][:, 0:3, 0:2, 0:2])
        assert np.abs(fo).max() > 1e-4
    L.orc_work_free(w)


@pytest.mark.parametrize("ndim", [1, 2, 3])
def test_amr_tree_walks_of_the_kernels_equal_oracle(orc, dev, ndim):
    """amr_get3cubefather / amr_getnborfather (the device restatement of amr/nbors_utils.f90:5-194,404-525 used by the AMR kernels)
    against the oracle's on an adaptively refined mesh (1-D / 2-D with physical boundaries incl. corner octs, 3-D periodic): every
    oct and every cell of every level"""
    from oracle.amr import FastAmrRun
    if ndim == 1:
        reg = [dict(type="square", x_center=0.25, length_x=0.5, d=1.0, p=1.0), dict(type="square", x_center=0.75, length_x=0.5, d=0.125, p=0.1)]
        r = FastAmrRun(1, 3, 8, (1, 1, 0, 0, 0, 0), 1.0, nsubcycle=[1, 2], ngridmax=500, err_grad_d=0.05, err_grad_p=0.05,
                       interpol_type=2, regions=reg, tout=[0.05])
    elif ndim == 2:
        from conftest import IMPL, IMPL_BOUND
        r = FastAmrRun(2, 4, 7, (1, 1, 1, 1, 0, 0), 1.0, nsubcycle=[2] * 10, nexpand=[2], ngridmax=20000, err_grad_d=0.05,
                       err_grad_u=0.05, err_grad_p=0.05, interpol_type=2, regions=IMPL, tout=[0.0, 0.05], bound_regions=IMPL_BOUND)
    else:
        reg = [dict(type="square", x_center=0.5, y_center=0.5, z_center=0.5, length_x=10, length_y=10, length_z=10, exp_region=10, d=1.0, p=1e-5),
               dict(type="point", x_center=0.5, y_center=0.5, z_center=0.5, p=0.4)]
        r = FastAmrRun(3, 3, 5, (0,) * 6, 1.0, nsubcycle=[1, 2], ngridmax=4000, riemann="hllc", slope_type=1,
                       err_grad_p=0.1, interpol_type=1, regions=reg, tout=[1e9])
    r.run(max_coarse=3)
    m = r.m
    T, n3, nn = 1 << ndim, 3 ** ndim, 2 * ndim + 1
    son = np.ascontiguousarray(r.son[1:], dtype=np.int32)
    father = np.ascontiguousarray(r.father[1:], dtype=np.int32)
    nbor = np.ascontiguousarray(r.nbor[:, 1:], dtype=np.int32)
    geo = (ndim, r.ncoarse, r.ngridmax, m.nx, m.ny, m.nz)
    L = orc.lib()
    L.orc_getnborfather.argtypes = [C.POINTER(orc.MeshS), C.c_int, C.c_int, C.POINTER(C.c_int)]
    checked = 0
    for l in range(1, r.nlevelmax + 1):
        octs = list(r.active[l]) + [g for b in range(m.nboundary) for g in r.bound[b][l]]
        act = np.asarray(r.active[l], dtype=np.int32)
        if len(act):
            got = np.zeros((len(act), n3), dtype=np.int32)
            dev.devnum_amr_get3cubefather(*geo, orc.iptr(son), orc.iptr(father), orc.iptr(nbor), len(act), orc.iptr(act), l, orc.iptr(got))
            ref = np.zeros((len(act), n3), dtype=np.int32)
            buf = (C.c_int * 27)()
            for i, g in enumerate(act):
                L.orc_get3cubefather(r.mp, int(r.father[g]), l, buf, None)
                ref[i] = buf[:n3]
            assert np.array_equal(got, ref)
            checked += len(act)
        if l < r.nlevelmax and len(octs):
            cells = np.array([r.ncoarse + ind * r.ngridmax + g for g in octs for ind in range(T)], dtype=np.int32)
            got = np.zeros((len(cells), nn), dtype=np.int32)
            dev.devnum_amr_getnborfather(*geo, orc.iptr(son), orc.iptr(father), orc.iptr(nbor), len(cells), orc.iptr(cells), l + 1, orc.iptr(got))
            ref = np.zeros((len(cells), nn), dtype=np.int32)
            buf = (C.c_int * 7)()
            for i, c in enumerate(cells):
                L.orc_getnborfather(r.mp, int(c), l + 1, buf)
                ref[i] = buf[:nn]
            assert np.array_equal(got, ref)
    assert checked > 50 and len(r.active[r.levelmin + 1]) > 0


@pytest.mark.parametrize("ndim", [1, 2, 3])
def test_amr_hydro_flag_kernel_equals_oracle(orc, dev, ndim):
    """amr_hydro_flag_kernel (hydro_flag + hydro_refine, hydro/hydro_flag.f90, godunov_utils.f90:125-263) executed thread by thread
    on the CPU == the oracle's hydro_flag on an adaptively refined mesh with a developed flow: every active cell of every level,
    all three criteria (density, velocity, pressure)."""
    from oracle.amr import FastAmrRun
    if ndim == 1:
        reg = [dict(type="square", x_center=0.25, length_x=0.5, d=1.0, p=1.0), dict(type="square", x_center=0.75, length_x=0.5, d=0.125, p=0.1)]
        r = FastAmrRun(1, 3, 8, (1, 1, 0, 0, 0, 0), 1.0, nsubcycle=[1, 2], ngridmax=500, err_grad_d=0.05, err_grad_u=0.1, err_grad_p=0.05,
                       interpol_type=2, regions=reg, tout=[0.05])
    elif ndim == 2:
        from conftest import IMPL, IMPL_BOUND
        r = FastAmrRun(2, 4, 7, (1, 1, 1, 1, 0, 0), 1.0, nsubcycle=[2] * 10, nexpand=[2], ngridmax=20000, err_grad_d=0.05,
                       err_grad_u=0.05, err_grad_p=0.05, interpol_type=2, regions=IMPL, tout=[0.0, 0.05], bound_regions=IMPL_BOUND)
    else:
        reg = [dict(type="square", x_center=0.5, y_center=0.5, z_center=0.5, length_x=10, length_y=10, length_z=10, exp_region=10, d=1.0, p=1e-5),
               dict(type="point", x_center=0.5, y_center=0.5, z_center=0.5, p=0.4)]
        r = FastAmrRun(3, 3, 5, (0,) * 6, 1.0, nsubcycle=[1, 2], ngridmax=4000, riemann="hllc", slope_type=1,
                       err_grad_d=0.2, err_grad_u=0.3, err_grad_p=0.1, interpol_type=1, regions=reg, tout=[1e9])
    r.run(max_coarse=3)
    m = r.m
    T = 1 << ndim
    son = np.ascontiguousarray(r.son[1:], dtype=np.int32)
    father = np.ascontiguousarray(r.father[1:], dtype=np.int32)
    nbor = np.ascontiguousarray(r.nbor[:, 1:], dtype=np.int32)
    geo = (ndim, r.ncoarse, r.ngridmax, m.nx, m.ny, m.nz)
    dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int)
    dev.devnum_amr_hydro_flag.argtypes = [C.c_int] * 6 + [ip, ip, ip, ip, C.c_int, C.c_int, dp, C.c_double, C.c_double, dp, dp, ip]
    err = np.array([r.err_grad_d, r.err_grad_u, r.err_grad_p])
    flo = np.array([r.floor_d, r.floor_u, r.floor_p])
    nflag = 0
    for l in range(r.levelmin, r.nlevelmax):
        act = np.asarray(r.active[l], dtype=np.int32)
        if not len(act):
            continue
        got = np.zeros((len(act), T), dtype=np.int32)
        dev.devnum_amr_hydro_flag(*geo, orc.iptr(son), orc.iptr(father), orc.iptr(nbor), orc.iptr(act), len(act), l, orc.dptr(r.uold),
                                  r.p.gamma, r.p.smallr, orc.dptr(err), orc.dptr(flo), orc.iptr(got))
        r.flag1[:] = 0
        r.hydro_flag(l)
        ref = np.array([[r.flag1[r.cell(ind, int(g))] for ind in range(T)] for g in act], dtype=np.int32)
        assert np.array_equal(got, ref), l
        nflag += int(ref.sum())
    assert nflag > 10


@pytest.mark.parametrize("ndim", [1, 2, 3])
@pytest.mark.parametrize("itype", [0, 1, 2, 3])
def test_amr_prolongation_of_the_kernels_equals_oracle(orc, dev, ndim, itype):
    """amr_interpol_var (interpol_hydro on the device, one variable at a time) == orc_interpol_hydro, bit for bit"""
    L = orc.lib()
    L.orc_set_interpol.argtypes = [C.c_int, C.c_int]
    L.orc_interpol_hydro.argtypes = [C.POINTER(orc.Params), C.POINTER(C.c_double), C.POINTER(C.c_double)]
    n, na, T = 4000, 2 * ndim + 1, 1 << ndim
    rng = np.random.default_rng(ndim * 7 + itype)
    a = rng.standard_normal((n, na)) * 10.0 ** rng.uniform(-3, 3, (n, 1))
    a[: n // 4] = np.abs(a[: n // 4])
    a[n // 4: n // 2, 1:] = a[n // 4: n // 2, :1] * (1 + 1e-3 * rng.standard_normal((n // 4, na - 1)))
    a = np.ascontiguousarray(a)
    got = np.zeros((n, T))
    dev.devnum_amr_interpol(ndim, itype, n, orc.dptr(a), orc.dptr(got))
    p = orc.make_params(ndim=ndim, nvar=1)
    ref = np.zeros((n, T))
    try:
        L.orc_set_interpol(itype, 0)
        for i in range(n):
            L.orc_interpol_hydro(C.byref(p), orc.dptr(a[i]), orc.dptr(ref[i]))
    finally:
        L.orc_set_interpol(1, 0)
    assert np.array_equal(got, ref)


@pytest.mark.parametrize("ndim", [1, 2, 3])
@pytest.mark.parametrize("itype,ivar", [(1, 1), (2, 1), (3, 1), (0, 2), (1, 2), (2, 2), (3, 2), (4, 2), (2, 0)])
def test_amr_coupled_prolongation_equals_oracle(orc, dev, ndim, itype, ivar):
    """amr_interpol_hydro (the whole state: interpol_var 1 = internal energy, 2 = velocities + internal energy with the momentum
    correction, interpol_type 4 = central slopes for the velocities; hydro/interpol_hydro.f90:318-440) == orc_interpol_hydro"""
    L = orc.lib()
    dp = C.POINTER(C.c_double)
    L.orc_set_interpol.argtypes = [C.c_int, C.c_int]
    L.orc_interpol_hydro.argtypes = [C.POINTER(orc.Params), dp, dp]
    dev.devnum_amr_interpol_full.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, dp, dp, C.c_double]
    n, na, T, nv = 3000, 2 * ndim + 1, 1 << ndim, ndim + 2
    rng = np.random.default_rng(100 * ndim + 10 * itype + ivar)
    u1 = np.zeros((n, na, nv))
    rho = 10.0 ** rng.uniform(-2, 2, (n, 1)) * (1 + 0.3 * rng.standard_normal((n, na)))
    rho = np.abs(rho) + 1e-3
    rho[:50, 2] = 1e-13                                    # below smallr: the floor of the velocity / kinetic-energy divisions
    v = rng.standard_normal((n, na, ndim)) * 10.0 ** rng.uniform(-2, 1, (n, 1, 1))
    eint = 10.0 ** rng.uniform(-3, 2, (n, na))
    u1[:, :, 0] = rho
    u1[:, :, 1:1 + ndim] = rho[:, :, None] * v
    u1[:, :, ndim + 1] = eint + 0.5 * rho * (v ** 2).sum(axis=2)
    u1 = np.ascontiguousarray(u1)
    got = np.zeros((n, T, nv))
    dev.devnum_amr_interpol_full(ndim, itype, ivar, n, orc.dptr(u1), orc.dptr(got), 1e-10)
    p = orc.make_params(ndim=ndim)
    ref = np.zeros((n, T, nv))
    try:
        L.orc_set_interpol(itype, ivar)
        for i in range(n):
            L.orc_interpol_hydro(C.byref(p), orc.dptr(u1[i]), orc.dptr(ref[i]))
    finally:
        L.orc_set_interpol(1, 0)
    assert np.isfinite(got).all()
    assert np.array_equal(got, ref)


@pytest.mark.parametrize("ndim,solver,difmag", [(1, "hllc", 0.0), (2, "hllc", 0.0), (2, "llf", 0.0), (3, "hllc", 0.0), (3, "exact", 0.0),
                                                 (2, "hllc", 0.1), (3, "hllc", 0.1)])
def test_amr_oct_batch_kernel_emulated_on_the_cpu_equals_oracle(orc, dev, ndim, solver, difmag):
    """amr_godfine_kernel itself -- 64 cooperating threads per oct, the 6^ndim patch and the face states in shared memory, five
    block barriers -- executed by the emulated launch of tests/host_numerics (one OS thread per CUDA thread, `static` for
    __shared__, a pthread barrier for __syncthreads) on an adaptively refined mesh: the update of the level's own cells equals
    godfine1 of the oracle (gather with prolongated ghost octs, unsplit, flux reset at refined faces, conservative update) bit
    for bit on every level.  The kernels that use warp shuffles / cp.async (the dense sweep) are outside this harness."""
    _amr_oct_batch_compare(orc, dev, ndim, solver, difmag)


@pytest.mark.parametrize("floors", ["default", "raised"])
@pytest.mark.parametrize("ndim,solver,difmag", [(1, "hllc", 0.0), (2, "llf", 0.0), (2, "hllc", 0.1), (3, "hllc", 0.0), (3, "exact", 0.1)])
def test_amr_oct_batch_kernel_emulated_at_the_floors(orc, dev, floors, ndim, solver, difmag):
    """amr_godfine_kernel on the adaptively refined meshes of the test above with every cell holding a floor_state cell under the
    RAMSES floors and raised ones: ctoprim's density and internal-energy floors and the face-density resets of the predictor
    fire; the update of every level equals godfine1 of the oracle, bit for bit"""
    _amr_oct_batch_compare(orc, dev, ndim, solver, difmag, floors)


def _put_floor_state(r, ndim, floors, seed):
    """a floor_state on every cell of the AMR run r (helpers.fill_floor_state) with the run's floors set to match; returns a time
    step of Courant number ~0.3 on the finest level"""
    from helpers import fill_floor_state
    r.p.smallr, r.p.smallc = fill_floor_state(r.uold, ndim, ndim + 2, r.ncell, floors, seed)
    d = r.uold.reshape(ndim + 2, r.ncell)
    rho = np.maximum(d[0], r.p.smallr)
    v2 = sum((d[1 + k] / rho) ** 2 for k in range(ndim))
    eint = np.maximum(d[ndim + 1] / rho - 0.5 * v2, r.p.smallc ** 2 / 1.4 / 0.4)
    vmax = float((np.sqrt(v2) + np.sqrt(1.4 * 0.4 * eint)).max())
    return 0.3 * 0.5 ** r.nlevelmax * r.p.boxlen / vmax


def _amr_oct_batch_compare(orc, dev, ndim, solver, difmag, floors=None):
    """the body of test_amr_oct_batch_kernel_emulated_on_the_cpu_equals_oracle; floors: a floor_state on every cell instead of the
    developed flow, under helpers.FLOORS[floors]"""
    from oracle.amr import FastAmrRun
    if ndim == 1:
        reg = [dict(type="square", x_center=0.25, length_x=0.5, d=1.0, p=1.0), dict(type="square", x_center=0.75, length_x=0.5, d=0.125, p=0.1)]
        r = FastAmrRun(1, 3, 8, (1, 1, 0, 0, 0, 0), 1.0, nsubcycle=[1, 2], ngridmax=500, riemann=solver, slope_type=2,
                       err_grad_d=0.05, err_grad_p=0.05, interpol_type=2, regions=reg, tout=[1e9])
        itype, st = 2, 2
    elif ndim == 2:
        from conftest import IMPL, IMPL_BOUND
        r = FastAmrRun(2, 4, 6, (1, 1, 1, 1, 0, 0), 1.0, nsubcycle=[2] * 10, nexpand=[2], ngridmax=20000, riemann=solver, slope_type=2,
                       err_grad_d=0.05, err_grad_u=0.05, err_grad_p=0.05, interpol_type=2, regions=IMPL, tout=[0.0, 1e9],
                       bound_regions=IMPL_BOUND)
        itype, st = 2, 2
    else:
        reg = [dict(type="square", x_center=0.5, y_center=0.5, z_center=0.5, length_x=10, length_y=10, length_z=10, exp_region=10, d=1.0, p=1e-5),
               dict(type="point", x_center=0.5, y_center=0.5, z_center=0.5, p=0.4)]
        r = FastAmrRun(3, 3, 5, (0,) * 6, 1.0, nsubcycle=[1, 2], ngridmax=4000, riemann=solver, slope_type=1, err_grad_p=0.1,
                       interpol_type=1, regions=reg, tout=[1e9])
        itype, st = 1, 1
    r.run(max_coarse=3)
    dt_floor = _put_floor_state(r, ndim, floors, 40 + ndim) if floors else None
    r.p.difmag = difmag                                  # artificial diffusion (cmpdivu / consup) for the comparison step only
    m = r.m
    T, nvar = 1 << ndim, ndim + 2
    son = np.ascontiguousarray(r.son[1:], dtype=np.int32)
    father = np.ascontiguousarray(r.father[1:], dtype=np.int32)
    nbor = np.ascontiguousarray(r.nbor[:, 1:], dtype=np.int32)
    sid = {"llf": 0, "exact": 1, "acoustic": 2, "hllc": 3, "hll": 4}[solver]
    L = orc.lib()
    nlev, moved = 0, 0.0
    for l in range(r.levelmin, r.nlevelmax + 1):
        act = np.ascontiguousarray(r.active[l], dtype=np.int32)
        if len(act) == 0:
            continue
        dt = 0.4 * r.dtnew[r.levelmin] / 2 ** (l - r.levelmin) if r.dtnew[r.levelmin] > 0 else 1e-4
        if floors:
            dt = dt_floor * 2 ** (r.nlevelmax - l)
        dx = 0.5 ** l * r.p.boxlen / (m.icoarse_max - m.icoarse_min + 1)
        # oracle: set_unew + godunov_fine of this level only
        unew_o = np.zeros_like(r.uold)
        L.orc_set_unew(C.byref(r.p), r.mp, l, orc.dptr(r.uold), orc.dptr(unew_o))
        L.orc_godunov_fine(C.byref(r.p), r.mp, l, dt, orc.dptr(r.uold), orc.dptr(unew_o), 1)
        # emulated kernel: unew = uold on the level's cells, then the kernel adds the flux differences
        unew_k = np.zeros_like(r.uold)
        L.orc_set_unew(C.byref(r.p), r.mp, l, orc.dptr(r.uold), orc.dptr(unew_k))
        rflux = np.zeros(len(act) * 2 * ndim * (T // 2) * nvar)
        dev.devnum_amr_godfine(ndim, sid, r.ncoarse, r.ngridmax, m.nx, m.ny, m.nz, orc.iptr(son), orc.iptr(father), orc.iptr(nbor),
                               orc.iptr(act), len(act), l, orc.dptr(r.uold), orc.dptr(unew_k), orc.dptr(rflux), dt, dx, itype, st,
                               r.p.slope_theta, 1.4, r.p.smallr, r.p.smallc, 10, difmag)
        assert np.isfinite(unew_o).all()
        Uo, Uk = unew_o.reshape(nvar, r.ncell), unew_k.reshape(nvar, r.ncell)
        for ind in range(T):
            c = r.ncoarse + ind * r.ngridmax + act.astype(np.int64) - 1
            assert np.array_equal(Uk[:, c], Uo[:, c]), (l, ind)
            moved = max(moved, float(np.abs(Uo[:, c] - r.uold.reshape(nvar, r.ncell)[:, c]).max()))
        nlev += 1
    assert nlev >= 3 and moved > 1e-6


@pytest.mark.parametrize("ndim,solver,grav,pfix", [(1, "hllc", True, True), (2, "hllc", True, True), (2, "exact", False, True),
                                                    (3, "hllc", True, True), (3, "llf", True, False), (3, "acoustic", False, True),
                                                    (3, "hll", True, True)])
def test_amr_source_terms_emulated_on_the_cpu_equal_oracle(orc, dev, ndim, solver, grav, pfix):
    """poisson and pressure_fix on an adaptively refined mesh, one level step per level: the SRC instantiation of the oct-batch
    kernel (gloc gather incl. the father's f in buffer cells, gravity predictor in ctoprim, tmp1/tmp2 -> divu/enew) run by the
    emulated launch, and the list passes of set_unew / set_uold (divu/enew reset, add_gravity_source_terms,
    add_pdv_source_terms, the energy switch) equal the oracle's set_unew -> godunov_fine -> set_uold bit for bit on the level's
    own cells (state, divu and enew)."""
    _amr_source_terms_compare(orc, dev, ndim, solver, grav, pfix)


@pytest.mark.parametrize("floors", ["default", "raised"])
@pytest.mark.parametrize("ndim,solver,grav,pfix", [(1, "hllc", True, True), (2, "exact", False, True), (2, "llf", True, False),
                                                    (3, "hllc", True, True), (3, "acoustic", False, True)])
def test_amr_source_terms_emulated_at_the_floors(orc, dev, floors, ndim, solver, grav, pfix):
    """poisson and pressure_fix on the refined meshes of the test above with every cell holding a floor_state cell: the gravity
    predictor and add_gravity_source_terms on floored densities (d_old = max(uold, smallr), godunov_fine.f90:267), enew / divu
    and add_pdv_source_terms at cold hypersonic cells, and the energy switch, which fires there on every level -- equal the
    oracle's set_unew -> godunov_fine -> set_uold bit for bit"""
    _amr_source_terms_compare(orc, dev, ndim, solver, grav, pfix, floors)


def _amr_source_terms_compare(orc, dev, ndim, solver, grav, pfix, floors=None, run=None, beta_fix=0.5):
    """the body of test_amr_source_terms_emulated_on_the_cpu_equal_oracle; floors: a floor_state on every cell, under
    helpers.FLOORS[floors]; run: a developed AMR run (interpolation type 2 below 3-D, 1 in 3-D) used instead of the meshes above,
    with its slope_type, gamma, slope_theta, niter_riemann and boxlen.  Returns (cells where the energy switch fired, cells
    compared)."""
    from oracle.amr import FastAmrRun
    if run is not None:
        r, itype, st = run, (2 if ndim < 3 else 1), run.p.slope_type
    elif ndim == 1:
        reg = [dict(type="square", x_center=0.25, length_x=0.5, d=1.0, p=1.0), dict(type="square", x_center=0.75, length_x=0.5, d=0.125, p=0.1)]
        r = FastAmrRun(1, 3, 8, (1, 1, 0, 0, 0, 0), 1.0, nsubcycle=[1, 2], ngridmax=500, riemann=solver, slope_type=2,
                       err_grad_d=0.05, err_grad_p=0.05, interpol_type=2, regions=reg, tout=[1e9])
        itype, st = 2, 2
    elif ndim == 2:
        from conftest import IMPL, IMPL_BOUND
        r = FastAmrRun(2, 4, 6, (1, 1, 1, 1, 0, 0), 1.0, nsubcycle=[2] * 10, nexpand=[2], ngridmax=20000, riemann=solver, slope_type=2,
                       err_grad_d=0.05, err_grad_u=0.05, err_grad_p=0.05, interpol_type=2, regions=IMPL, tout=[0.0, 1e9],
                       bound_regions=IMPL_BOUND)
        itype, st = 2, 2
    else:
        reg = [dict(type="square", x_center=0.5, y_center=0.5, z_center=0.5, length_x=10, length_y=10, length_z=10, exp_region=10, d=1.0, p=1e-5),
               dict(type="point", x_center=0.5, y_center=0.5, z_center=0.5, p=0.4)]
        r = FastAmrRun(3, 3, 5, (0,) * 6, 1.0, nsubcycle=[1, 2], ngridmax=4000, riemann=solver, slope_type=1, err_grad_p=0.1,
                       interpol_type=1, regions=reg, tout=[1e9])
        itype, st = 1, 1
    if run is None:
        r.run(max_coarse=3)
    dt_floor = _put_floor_state(r, ndim, floors, 50 + ndim) if floors else None
    m = r.m
    T, nvar, nc = 1 << ndim, ndim + 2, r.ncell
    son = np.ascontiguousarray(r.son[1:], dtype=np.int32)
    father = np.ascontiguousarray(r.father[1:], dtype=np.int32)
    nbor = np.ascontiguousarray(r.nbor[:, 1:], dtype=np.int32)
    sid = {"llf": 0, "exact": 1, "acoustic": 2, "hllc": 3, "hll": 4}[solver]
    L = orc.lib()
    L.orc_set_pressure_fix.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_double]
    L.orc_set_gravity.argtypes = [C.POINTER(C.c_double)]
    rng = np.random.default_rng(7 * ndim + sid)
    # an arbitrary acceleration field (f is an input of the path): a uniform pull plus cell-to-cell structure, strong enough to matter
    force = np.ascontiguousarray((np.array([0.7, -0.4, 0.3])[:ndim, None] + 0.3 * rng.standard_normal((ndim, nc))) * 5.0)
    nlev, switched, gmoved, dmax, nrefl, ncmp = 0, 0, 0.0, 0.0, 0, 0
    try:
        for l in range(r.levelmin, r.nlevelmax + 1):
            act = np.ascontiguousarray(r.active[l], dtype=np.int32)
            if len(act) == 0:
                continue
            dt = 0.4 * r.dtnew[r.levelmin] / 2 ** (l - r.levelmin) if r.dtnew[r.levelmin] > 0 else 1e-4
            if floors:
                dt = dt_floor * 2 ** (r.nlevelmax - l)
            dx = 0.5 ** l * r.p.boxlen / (m.icoarse_max - m.icoarse_min + 1)
            cells = np.concatenate([r.ncoarse + ind * r.ngridmax + act.astype(np.int64) - 1 for ind in range(T)])
            # ---- oracle: set_unew -> godunov_fine -> set_uold of this level with the options on
            uold_o, unew_o = r.uold.copy(), np.zeros_like(r.uold)
            divu_o, enew_o = np.full(nc, 7.0), np.full(nc, -3.0)          # garbage that set_unew must overwrite on the level
            L.orc_set_pressure_fix(orc.dptr(divu_o) if pfix else None, orc.dptr(enew_o) if pfix else None, beta_fix)
            L.orc_set_gravity(orc.dptr(force) if grav else None)
            L.orc_set_unew(C.byref(r.p), r.mp, l, orc.dptr(uold_o), orc.dptr(unew_o))
            L.orc_godunov_fine(C.byref(r.p), r.mp, l, dt, orc.dptr(uold_o), orc.dptr(unew_o), 1)
            divu_mid, enew_mid, unew_mid = divu_o.copy(), enew_o.copy(), unew_o.copy()
            L.orc_set_uold(C.byref(r.p), r.mp, l, orc.dptr(uold_o), orc.dptr(unew_o))
            L.orc_set_pressure_fix(None, None, 0.0)
            L.orc_set_gravity(None)
            # ---- device code on the host: unew holds nvar (+2) columns
            ncol = nvar + (2 if pfix else 0)
            uold_k = r.uold.copy()
            unew_k = np.zeros(ncol * nc)
            unew_k[: nvar * nc].reshape(nvar, nc)[:, cells] = r.uold.reshape(nvar, nc)[:, cells]                 # set_unew copy
            divu_k = unew_k[nvar * nc: (nvar + 1) * nc] if pfix else np.zeros(nc)
            enew_k = unew_k[(nvar + 1) * nc:] if pfix else np.zeros(nc)
            if pfix:
                divu_k[:] = 7.0; enew_k[:] = -3.0
            args = (ndim, r.ncoarse, r.ngridmax, m.nx, m.ny, m.nz, orc.iptr(son), orc.iptr(father), orc.iptr(nbor), orc.iptr(act), len(act))
            tail = (orc.dptr(force), r.p.gamma, r.p.smallr, beta_fix, dx, dt)
            if pfix:
                dev.devnum_amr_src_pass(0, *args, orc.dptr(uold_k), orc.dptr(unew_k), orc.dptr(divu_k), orc.dptr(enew_k), *tail)
            rflux = np.zeros(len(act) * 2 * ndim * (T // 2) * ncol)
            dev.devnum_amr_godfine_src(ndim, sid, r.ncoarse, r.ngridmax, m.nx, m.ny, m.nz, orc.iptr(son), orc.iptr(father), orc.iptr(nbor),
                                       orc.iptr(act), len(act), l, orc.dptr(uold_k), orc.dptr(unew_k), orc.dptr(rflux), dt, dx, itype, st,
                                       r.p.slope_theta, r.p.gamma, r.p.smallr, r.p.smallc, r.p.niter_riemann,
                                       orc.dptr(force) if grav else None, 1 if pfix else 0, r.nvector)
            # after the sweep and the coarse reflux pass, before the sources: the WHOLE arrays -- the level's own cells and the coarser
            # cells that received refluxes (state, and with pressure_fix divu / enew, which reflux like two more variables)
            assert np.array_equal(unew_k[: nvar * nc], unew_mid), l
            nrefl += int((unew_mid.reshape(nvar, nc)[:, np.setdiff1d(np.arange(nc), cells)] != 0).any(axis=0).sum())
            if pfix:
                assert np.array_equal(divu_k, divu_mid), l
                assert np.array_equal(enew_k, enew_mid), l
                dmax = max(dmax, float(np.abs(divu_mid[cells]).max()))
            if grav:
                dev.devnum_amr_src_pass(1, *args, orc.dptr(uold_k), orc.dptr(unew_k), orc.dptr(divu_k), orc.dptr(enew_k), *tail)
            if pfix:
                dev.devnum_amr_src_pass(2, *args, orc.dptr(uold_k), orc.dptr(unew_k), orc.dptr(divu_k), orc.dptr(enew_k), *tail)
            before = uold_k.reshape(nvar, nc)[:, cells].copy()
            uold_k.reshape(nvar, nc)[:, cells] = unew_k[: nvar * nc].reshape(nvar, nc)[:, cells]                 # uold <- unew
            if pfix:
                pre = uold_k.reshape(nvar, nc)[nvar - 1, cells].copy()
                dev.devnum_amr_src_pass(3, *args, orc.dptr(uold_k), orc.dptr(unew_k), orc.dptr(divu_k), orc.dptr(enew_k), *tail)
                switched += int((uold_k.reshape(nvar, nc)[nvar - 1, cells] != pre).sum())
                assert np.array_equal(enew_k[cells], enew_o[cells]), l
            got, ref = uold_k.reshape(nvar, nc)[:, cells], uold_o.reshape(nvar, nc)[:, cells]
            assert np.array_equal(got, ref), (l, np.abs(got - ref).max())
            gmoved = max(gmoved, float(np.abs(ref - before).max()))
            ncmp += len(cells)
            nlev += 1
    finally:
        L.orc_set_pressure_fix(None, None, 0.0)
        L.orc_set_gravity(None)
    assert nlev >= 3 and gmoved > 1e-6 and (dmax > 0 or not pfix) and nrefl > 0
    if pfix and (ndim == 3 or floors) and beta_fix > 0:
        assert switched > 0          # the cold Sedov background (p = 1e-5) and the cold hypersonic cells trip the energy switch
    assert np.isfinite(uold_o).all()
    return switched, ncmp


MHD_R1D = {"llf": 0, "roe": 1, "hll": 2, "hlld": 3, "upwind": 4, "hydro": 5}
MHD_R2D = {"llf": 0, "roe": 1, "upwind": 2, "hll": 3, "hlla": 4, "hlld": 5}


def _mhd_amr_compare_levels(orc, dev, r, ndim, riemann, riemann2d, slope_type, interpol_type, godunov, upload, courant, boundary=None,
                            interpol_mag_type=-1):
    """every populated level of the run `r`: godunov_fine (own cells AND the refluxed coarse cells: the whole unew array),
    upload_fine, the leaf-cell Courant step and (1-D) make_boundary_hydro of the device code == the oracle's, bit for bit"""
    m = r.m
    T, nc = 1 << ndim, r.ncell
    son = np.ascontiguousarray(r.son[1:], dtype=np.int32)
    father = np.ascontiguousarray(r.father[1:], dtype=np.int32)
    nbor = np.ascontiguousarray(r.nbor[:, 1:], dtype=np.int32)
    L = orc.lib()
    tree = (ndim, r.ncoarse, r.ngridmax, m.nx, m.ny, m.nz, orc.iptr(son), orc.iptr(father), orc.iptr(nbor))
    nlev, nrefl, moved = 0, 0, 0.0
    for l in range(r.levelmin, r.nlevelmax + 1):
        act = np.ascontiguousarray(r.active[l], dtype=np.int32)
        if len(act) == 0:
            continue
        dt = 0.5 * r.dtnew[r.levelmin] / 2 ** (l - r.levelmin) if r.dtnew[r.levelmin] > 0 else 1e-4
        dx = 0.5 ** l * r.p.boxlen / (m.icoarse_max - m.icoarse_min + 1)
        # ---- godunov_fine
        unew_o, unew_k = np.zeros_like(r.uold), np.zeros_like(r.uold)
        if l > r.levelmin:          # the coarser level has been through set_unew: its cells carry the state, refluxes add to it
            L.orc_mhdn_set_unew(r.mp, l - 1, orc.dptr(r.uold), orc.dptr(unew_o))
            L.orc_mhdn_set_unew(r.mp, l - 1, orc.dptr(r.uold), orc.dptr(unew_k))
        L.orc_mhdn_set_unew(r.mp, l, orc.dptr(r.uold), orc.dptr(unew_o))
        L.orc_mhdn_set_unew(r.mp, l, orc.dptr(r.uold), orc.dptr(unew_k))
        before = unew_o.copy()
        godunov(C.byref(r.pm), r.mp, l, r.levelmin, r.nvector, dt, orc.dptr(r.uold), orc.dptr(unew_o))
        dev.devnum_mhd_amr_godunov(*tree[:9], orc.iptr(act), len(act), l, orc.dptr(r.uold), orc.dptr(unew_k), dt, dx, interpol_type, interpol_mag_type,
                                   MHD_R1D[riemann], MHD_R2D[riemann2d], slope_type, slope_type, r.pm.gamma, r.pm.smallr, r.pm.smallc, r.nvector)
        assert np.isfinite(unew_k).all()
        assert np.array_equal(unew_k, unew_o), (l, np.abs(unew_k - unew_o).max())
        moved = max(moved, float(np.abs(unew_o - before).max()))
        if l > r.levelmin:
            own = np.zeros(nc, dtype=bool)
            for ind in range(T):
                own[r.ncoarse + ind * r.ngridmax + act.astype(np.int64) - 1] = True
            d = (unew_o != before).reshape(11, nc)
            nrefl += int(d[:, ~own].any(axis=0).sum())
        # ---- upload_fine
        if l < r.nlevelmax:
            u_o, u_k = r.uold.copy(), r.uold.copy()
            upload(C.byref(r.pm), r.mp, l, orc.dptr(u_o))
            dev.devnum_mhd_amr_pass(0, *tree, orc.iptr(act), len(act), orc.dptr(u_k), r.pm.gamma, r.pm.smallr, r.pm.smallc, r.pm.courant_factor, dx, 0, 0, None)
            assert np.array_equal(u_k, u_o), l
        # ---- courant_fine
        dt_o = courant(C.byref(r.pm), r.mp, l, r.p.boxlen / r.p.smallc, orc.dptr(r.uold))
        dtc = np.zeros(len(act) * T)
        u_k = r.uold.copy()
        dev.devnum_mhd_amr_pass(2, *tree, orc.iptr(act), len(act), orc.dptr(u_k), r.pm.gamma, r.pm.smallr, r.pm.smallc, r.pm.courant_factor, dx, 0, 0, orc.dptr(dtc))
        if (dtc < 1e299).any():
            assert min(dtc.min(), r.pm.courant_factor * dx / r.pm.smallc, r.p.boxlen / r.p.smallc) == dt_o, l
        else:                       # a fully refined level has no leaf cell: courant_fine leaves dtnew alone
            assert dt_o == r.p.boxlen / r.p.smallc
        # ---- make_boundary_hydro (1-D)
        if boundary is not None:
            u_o, u_k = r.uold.copy(), r.uold.copy()
            # scramble the boundary octs first so that the pass has something to do
            for b in range(m.nboundary):
                for ig in r.bound[b][l]:
                    for ind in range(T):
                        u_o.reshape(11, nc)[:, r.cell(ind, ig) - 1] = 9.0
                        u_k.reshape(11, nc)[:, r.cell(ind, ig) - 1] = 9.0
            boundary(C.byref(r.pm), r.mp, l, orc.dptr(u_o))
            for b in range(m.nboundary):
                lst = np.ascontiguousarray(r.bound[b][l], dtype=np.int32)
                if len(lst) == 0:
                    continue
                bt = m.boundary_type[b]
                dev.devnum_mhd_amr_pass(1, *tree, orc.iptr(lst), len(lst), orc.dptr(u_k), r.pm.gamma, r.pm.smallr, r.pm.smallc, r.pm.courant_factor, dx,
                                        bt % 10, bt // 10, None)
            assert np.array_equal(u_k, u_o), l
        nlev += 1
    return nlev, nrefl, moved


@pytest.mark.parametrize("riemann,slope_type", [("hlld", 1), ("roe", 2), ("llf", 0), ("hll", 1)])
def test_mhd_amr_1d_kernels_emulated_on_the_cpu_equal_oracle(orc, dev, riemann, slope_type):
    """NDIM=1 ideal MHD on the refined mesh of the imhd-tube problem (tests/mhd/imhd-tube): mhd_amr1_godfine_kernel + the coarse
    reflux pass, upload_fine, cmpdt and the outflow boundaries (mhd_amr.cuh) against mhd1_godfine1 & co. of the oracle, which
    reproduces imhd-tube-ref.dat."""
    from oracle.amr_mhd import MhdAmrRun
    from test_oracle_golden import IMHD
    r = MhdAmrRun(5, 10, (2, 2, 0, 0, 0, 0), 3.5, nsubcycle=[1, 1, 1, 1], riemann=riemann, slope_type=slope_type, gamma=1.6666667,
                  courant_factor=0.8, err_grad_d=0.01, err_grad_u=0.05, err_grad_p=0.05, interpol_type=2, regions=IMHD,
                  tout=[1e9], ngridmax=10000)
    r.run(max_coarse=12)
    L = orc.lib()
    nlev, nrefl, moved = _mhd_amr_compare_levels(orc, dev, r, 1, riemann, "llf", slope_type, 2, L.orc_mhd1_godunov_fine, L.orc_mhd1_upload_fine,
                                                 L.orc_mhd1_courant_fine, boundary=L.orc_mhd1_make_boundary_hydro)
    assert nlev >= 4 and nrefl > 0 and moved > 1e-6


@pytest.mark.parametrize("r1,r2,slope_type", [("hlld", "hlld", 2), ("roe", "llf", 1), ("llf", "roe", 2), ("hll", "hll", 0), ("hydro", "hlla", 1),
                                               ("upwind", "upwind", 2)])
def test_mhd_amr_2d_kernels_emulated_on_the_cpu_equal_oracle(orc, dev, r1, r2, slope_type):
    """NDIM=2 ideal MHD on the adaptively refined Orszag-Tang vortex (tests/mhd/orszag-tang): mhd_amr2_godfine_kernel (64
    cooperating threads per oct: divergence-free prolongation of the ghost octs, trace2d, 12 face and 9 corner Riemann problems,
    constrained transport) + the Euler and corner-EMF coarse refluxes in the reference's accumulation order, upload_fine with
    face-centred restriction and cmpdt, against mhd2_godfine1 & co. of the oracle, which reproduces orszag-tang-ref.dat."""
    from oracle.amr_mhd import MhdAmrRun2D
    r = MhdAmrRun2D(4, 6, 1.0, nsubcycle=[1], riemann=r1, riemann2d=r2, slope_type=slope_type, gamma=1.6666667, courant_factor=0.8,
                    err_grad_p=0.1, interpol_type=2, tout=[1e9], nexpand=1, ngridmax=20000)
    r.run(max_coarse=16)
    L = orc.lib()
    nlev, nrefl, moved = _mhd_amr_compare_levels(orc, dev, r, 2, r1, r2, slope_type, 2, L.orc_mhd2_godunov_fine, L.orc_mhdn_upload_fine,
                                                 L.orc_mhdn_courant_fine)
    assert nlev >= 3 and nrefl > 0 and moved > 1e-6


def _mhd3_static_run(riemann, riemann2d, slope_type, lmin=3, lmax=5):
    """MhdAmrRun3D on a statically nested cube (levels lmin..lmax) with a genuinely three-dimensional, divergence-free state:
    the z-invariant Orszag-Tang fields + a B_z(x,y) component + z-dependent density and velocities, advanced by two sub-cycled
    coarse steps of the oracle so that every component of every face field and EMF is at work"""
    from oracle.amr_mhd import MhdAmrRun3D

    class Run(MhdAmrRun3D):
        def smooth_fine(self, l):
            pass

        def hydro_flag(self, l):
            if l == self.nlevelmax or self.numbtot(l) == 0:
                return
            hw = {lmin: 0.25, lmin + 1: 0.125}.get(l, 0.0)
            igs = np.asarray(self.active[l])
            dx = 0.5 ** l
            for ind in range(8):
                x = [self.xg[k, igs] + (((ind >> k) & 1) - 0.5) * dx for k in range(3)]
                inside = (np.abs(x[0] - 0.5) < hw) & (np.abs(x[1] - 0.4) < hw) & (np.abs(x[2] - 0.6) < hw)
                self.flag1[self.ncoarse + ind * self.ngridmax + igs[inside]] = 1

        def init_flow_fine(self, l):
            super().init_flow_fine(l)
            if self.numbtot(l) == 0:
                return
            U = self.uold.reshape(11, self.ncell)
            igs = np.asarray(self.active[l])
            dx = 0.5 ** l
            tp = 2 * np.pi
            for ind in range(8):
                x, y, z = [self.xg[k, igs] + (((ind >> k) & 1) - 0.5) * dx for k in range(3)]
                c = self.ncoarse + ind * self.ngridmax + igs - 1
                # B_z(x,y) as the exact average over the cell's (x,y) footprint: both z faces equal (d/dz = 0) and a coarse face
                # equals the mean of the four fine faces it covers, on every level: div B = 0 to round-off
                sx = (np.cos(tp * (x - 0.5 * dx)) - np.cos(tp * (x + 0.5 * dx))) / (tp * dx)
                cy = (np.sin(tp * (y + 0.5 * dx)) - np.sin(tp * (y - 0.5 * dx))) / (tp * dx)
                bz = 0.2 + 0.3 * sx * cy
                d0 = U[0, c].copy()
                vel = [U[1 + k, c] / d0 for k in range(3)]
                eint = U[4, c] - 0.5 * d0 * sum(v * v for v in vel) - 0.125 * sum((U[5 + k, c] + U[8 + k, c]) ** 2 for k in range(3))
                d = d0 * (1 + 0.3 * np.sin(tp * z) * np.cos(tp * x))
                vel[0] = vel[0] + 0.2 * np.sin(tp * z)
                vel[1] = vel[1] - 0.15 * np.cos(tp * z + 1.0)
                vel[2] = 0.3 * np.sin(tp * (x + y)) * np.cos(tp * z)
                U[7, c] = bz; U[10, c] = bz
                U[0, c] = d
                for k in range(3):
                    U[1 + k, c] = d * vel[k]
                U[4, c] = eint + 0.5 * d * sum(v * v for v in vel) + 0.125 * sum((U[5 + k, c] + U[8 + k, c]) ** 2 for k in range(3))
    r = Run(lmin, lmax, 1.0, nsubcycle=[1, 2], riemann=riemann, riemann2d=riemann2d, slope_type=slope_type, gamma=1.6666667, courant_factor=0.8,
            err_grad_p=0.1, interpol_type=2, tout=[1e9], nexpand=1, ngridmax=4000)
    r.flag_coarse(); r.init_refine(); r.init_refine_2()
    r.static = True
    for _ in range(2):
        r.amr_step(lmin, 1)
        r.nstep_coarse += 1
    return r


@pytest.mark.parametrize("r1,r2,slope_type", [("hlld", "hlld", 2), ("roe", "llf", 1), ("llf", "roe", 0), ("hll", "hlla", 2)])
def test_mhd_amr_3d_kernel_emulated_on_the_cpu_equals_oracle(orc, dev, r1, r2, slope_type):
    """NDIM=3 ideal MHD with AMR: mhd_amr3_godfine_kernel (128 cooperating threads per oct, the 6^3 patch and every intermediate of
    mag_unsplit in 155 KB of shared memory: 36 face and 54 edge Riemann problems, 3-D divergence-free prolongation of the ghost
    octs, constrained transport) + the Euler and twelve-edge EMF coarse refluxes, upload_fine and cmpdt, executed by the emulated
    launch on a nested three-level mesh with a fully three-dimensional field, against mhd3_godfine1 & co. of the oracle."""
    r = _mhd3_static_run(r1, r2, slope_type)
    assert [len(r.active[l]) for l in (3, 4, 5)] == [64, 64, 64]
    assert r.divb_max() < 1e-13
    L = orc.lib()
    nlev, nrefl, moved = _mhd_amr_compare_levels(orc, dev, r, 3, r1, r2, slope_type, 2, L.orc_mhd3_godunov_fine, L.orc_mhdn_upload_fine,
                                                 L.orc_mhdn_courant_fine)
    assert nlev == 3 and nrefl > 0 and moved > 1e-6


@pytest.mark.parametrize("ndim,itype,mtype", [(2, 1, -1), (2, 3, -1), (2, 0, 0), (2, 2, 3), (2, 1, 2), (3, 1, -1), (3, 3, -1), (3, 0, 0), (3, 2, 1),
                                              (1, 1, -1), (1, 3, -1), (1, 0, -1)])
def test_mhd_amr_prolongation_variants_emulated_on_the_cpu_equal_oracle(orc, dev, ndim, itype, mtype):
    """interpol_type 0..3 (cell-centred variables) and interpol_mag_type 0..3 (face fields; -1 = interpol_type) of the ghost-oct
    prolongation inside the MHD AMR kernels (mhd/interpol_hydro.f90:612-1400): the level update of refined meshes in 1-D / 2-D / 3-D
    stays bit-identical to the oracle for every limiter choice (the golden runs and the GPU tests use type 2)."""
    L = orc.lib()
    L.orc_mhd_set_interpol.argtypes = [C.c_int, C.c_int]
    if ndim == 1:
        from oracle.amr_mhd import MhdAmrRun
        from test_oracle_golden import IMHD
        r = MhdAmrRun(5, 9, (2, 2, 0, 0, 0, 0), 3.5, nsubcycle=[1, 1, 1, 1], riemann="hlld", slope_type=1, gamma=1.6666667,
                      courant_factor=0.8, err_grad_d=0.01, err_grad_u=0.05, err_grad_p=0.05, interpol_type=2, regions=IMHD,
                      tout=[1e9], ngridmax=10000)
        r.run(max_coarse=10)
        fns = (L.orc_mhd1_godunov_fine, L.orc_mhd1_upload_fine, L.orc_mhd1_courant_fine)
    elif ndim == 2:
        from oracle.amr_mhd import MhdAmrRun2D
        r = MhdAmrRun2D(4, 6, 1.0, nsubcycle=[1], riemann="hlld", riemann2d="hlld", slope_type=2, gamma=1.6666667, courant_factor=0.8,
                        err_grad_p=0.1, interpol_type=2, tout=[1e9], nexpand=1, ngridmax=20000)
        r.run(max_coarse=6)
        fns = (L.orc_mhd2_godunov_fine, L.orc_mhdn_upload_fine, L.orc_mhdn_courant_fine)
    else:
        r = _mhd3_static_run("hlld", "hlld", 2)
        fns = (L.orc_mhd3_godunov_fine, L.orc_mhdn_upload_fine, L.orc_mhdn_courant_fine)
    try:
        L.orc_mhd_set_interpol(itype, mtype)          # the oracle's godfine1 reads these globals (the 1-D path: interpol_type only)
        nlev, nrefl, moved = _mhd_amr_compare_levels(orc, dev, r, ndim, "hlld", "hlld" if ndim > 1 else "llf", 1 if ndim == 1 else 2, itype, *fns,
                                                     interpol_mag_type=mtype)
    finally:
        L.orc_mhd_set_interpol(2, -1)
    assert nlev >= 2 and moved > 1e-6


def _to_slots(dense, N):
    """dense [11][z][y][x] -> device layout [11][8][nslot] (cell_offset of sweep_dense.cuh, periodic cube, no ghost shell)"""
    h = N // 2
    z, y, x = np.meshgrid(np.arange(N), np.arange(N), np.arange(N), indexing="ij")
    ind = (x & 1) | ((y & 1) << 1) | ((z & 1) << 2)
    slot = (x >> 1) + h * ((y >> 1) + h * (z >> 1))
    u = np.zeros((11, 8, h ** 3))
    u[:, ind.ravel(), slot.ravel()] = dense.reshape(11, -1)
    return u, ind, slot


@pytest.mark.parametrize("r1d,r2d,st", [("roe", "llf", 0), ("hlld", "hlld", 1), ("llf", "llf", 2), ("hll", "hll", 1), ("hlld", "roe", 2),
                                        ("upwind", "upwind", 1), ("hydro", "hlla", 1)])
def test_mhd_six_pass_kernels_emulated_on_the_cpu_equal_oracle(orc, dev, r1d, r2d, st):
    """the six MHD kernels of mhd_dense.cuh (prim, efield, trace, flux, emf, update) executed thread by thread on the CPU in the
    order of launch_mhd_sweep, on a periodic 12^3 box in the device's slot layout: the new state equals set_unew + godunov_fine
    (fluxes, corner EMFs, constrained-transport update of both copies of every face) of the oracle, bit for bit"""
    from helpers import MhdCase, mhd_smooth_state
    dp = C.POINTER(C.c_double)
    dev.devnum_mhd_sweep.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, dp, dp, C.c_double, C.c_double, C.c_double, C.c_double,
                                     C.c_double, C.c_int, C.c_int, C.c_double, C.c_double]
    N, level = 16, 4
    c = MhdCase(level, riemann=r1d, riemann2d=r2d, slope_type=st)
    d0 = mhd_smooth_state(N)
    c.init_dense(d0)
    dt, _ = c.oracle_courant()
    dt *= 0.7
    ref = c.dense(c.oracle_godunov(dt, nthreads=2))
    uin, ind, slot = _to_slots(c.dense(), N)
    uout = np.zeros_like(uin)
    sl = 0 if st == 0 else 1
    dev.devnum_mhd_sweep(N, orc.MHD_RIEMANN[r1d], orc.MHD_RIEMANN2D[r2d], sl, orc.dptr(np.ascontiguousarray(uin)), orc.dptr(uout),
                         dt, 1.0 / N, c.p.gamma, c.p.smallr, c.p.smallc, st, st, c.p.slope_theta, c.p.courant_factor)
    got = uout[:, ind.ravel(), slot.ravel()].reshape(11, N, N, N)
    assert np.abs(ref - c.dense()).max() > 1e-4
    assert np.array_equal(got, ref)


def _hydro_to_slots(dense, ndim, N):
    """dense [nvar][z][y][x] (unused dimensions of extent 1) -> device layout [nvar][2^ndim][nslot]"""
    nvar = ndim + 2
    shp = [N if d < ndim else 1 for d in range(3)]            # x, y, z extents
    z, y, x = np.meshgrid(np.arange(shp[2]), np.arange(shp[1]), np.arange(shp[0]), indexing="ij")
    h = [max(s // 2, 1) for s in shp]
    ind = (x & 1)
    slot = (x >> 1)
    if ndim > 1:
        ind = ind | ((y & 1) << 1)
        slot = slot + h[0] * (y >> 1)
    if ndim > 2:
        ind = ind | ((z & 1) << 2)
        slot = slot + h[0] * h[1] * (z >> 1)
    nslot = h[0] * (h[1] if ndim > 1 else 1) * (h[2] if ndim > 2 else 1)
    u = np.zeros((nvar, 1 << ndim, nslot))
    u[:, ind.ravel(), slot.ravel()] = dense.reshape(nvar, -1)
    return u, ind, slot


@pytest.mark.parametrize("late", [0, 1])
@pytest.mark.parametrize("ndim,solver,st,N,nblocks", [(3, "hllc", 1, 16, 3), (3, "exact", 2, 16, 2), (3, "llf", 8, 16, 5), (2, "hllc", 2, 32, 3),
                                                      (2, "hll", 7, 32, 1), (1, "acoustic", 1, 64, 2), (3, "hllc", 3, 16, 4)])
def test_dense_sweep_kernel_emulated_on_the_cpu_equals_oracle(orc, dev, ndim, solver, st, N, nblocks, late):
    """sweep_dense_kernel -- THE hot kernel: persistent CTAs of 32 x BY threads, cp.async staging of the next plane, the ring of
    primitive planes in shared memory, warp shuffles for the x neighbours, shared-memory exchange for y, per-thread carry for z,
    fused set_unew + update + set_uold + Courant scan -- executed on the CPU by the emulated launch (one OS thread per CUDA
    thread, block barrier, per-warp shuffle exchange) for several persistent-grid sizes: the new state equals one level step of
    the oracle bit for bit, and the fused Courant partials reproduce the next time step.  late=1: the experimental two-barrier
    variant of the plane loop (template parameter LATE, not dispatched by the product yet) gives the same bits."""
    dp = C.POINTER(C.c_double)
    dev.devnum_sweep_dense.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, dp, dp, C.c_double, C.c_double, C.c_int, C.c_double,
                                       C.c_double, C.c_double, C.c_double, C.c_double, C.c_int, dp, C.c_int]
    from helpers import Case, smooth_state
    level = int(np.log2(N))
    c = Case(ndim, level, riemann=solver, slope_type=st, slope_theta=1.3)
    d0 = smooth_state(ndim, N)
    rough = np.random.default_rng(3).standard_normal(d0[0].shape)
    d0[0] *= 1 + 0.3 * (rough > 1.2)
    c.init_dense(d0)
    dt, _ = c.oracle_courant()
    unew = c.oracle_godunov(dt, nthreads=1)
    ref = c.dense(unew)
    dt_next, sums = c.oracle_courant(unew)
    uin, ind, slot = _hydro_to_slots(c.dense(), ndim, N)
    uout = np.zeros_like(uin)
    part = np.zeros(4 * 64)
    sid = {"llf": 0, "exact": 1, "acoustic": 2, "hllc": 3, "hll": 4}[solver]
    nb = dev.devnum_sweep_dense(ndim, sid, N, nblocks, orc.dptr(np.ascontiguousarray(uin)), orc.dptr(uout), dt, 1.0 / N, st, 1.3, 0.8,
                                1.4, 1e-10, 1e-10, 10, orc.dptr(part), late)
    got = uout[:, ind.ravel(), slot.ravel()].reshape(ref.shape)
    assert np.abs(ref - c.dense()).max() > 1e-4
    assert np.array_equal(got, ref)
    p4 = part[:4 * nb].reshape(4, nb)                      # fused courant_fine of the new state: min dt, mass, etot, eint per CTA
    assert p4[0].min() * 1.0 == dt_next or min(p4[0].min(), c.p.boxlen / c.p.smallc) == dt_next
    vol = (1.0 / N) ** ndim
    assert abs(p4[1].sum() * vol - sums[0]) <= 1e-13 * abs(sums[0]) and abs(p4[2].sum() * vol - sums[1]) <= 1e-13 * abs(sums[1])


@pytest.mark.parametrize("solver", ["hllc", "llf"])
def test_dense_sweep_amr_variant_emulated_on_the_cpu_equals_oracle(orc, dev, solver):
    """sweep_dense_kernel<..., AMRV=true>: the fully refined base level of an AMR run (part of its cells refined further) swept by
    the dense kernel -- flux masks of refined cells passed by shuffle (x), shared memory (y) and the plane carry (z), update
    accumulated into unew -- equals godfine1 of the oracle on that level, bit for bit"""
    from oracle.amr import FastAmrRun
    dp = C.POINTER(C.c_double)
    dev.devnum_sweep_dense_amr.argtypes = [C.c_int, C.c_int, C.c_int, dp, dp, C.POINTER(C.c_ubyte), C.c_double, C.c_double, C.c_int,
                                           C.c_double, C.c_double, C.c_double, C.c_double, C.c_int]
    reg = [dict(type="square", x_center=0.5, y_center=0.5, z_center=0.5, length_x=10, length_y=10, length_z=10, exp_region=10, d=1.0, p=1e-5),
           dict(type="point", x_center=0.5, y_center=0.5, z_center=0.5, p=0.4)]
    r = FastAmrRun(3, 4, 5, (0,) * 6, 1.0, nsubcycle=[1, 2], ngridmax=6000, riemann=solver, slope_type=1, err_grad_p=0.1,
                   interpol_type=1, regions=reg, tout=[1e9])
    r.run(max_coarse=3)
    l, N = 4, 16
    act = np.asarray(r.active[l], dtype=np.int64)
    assert len(act) == 8 ** 3 and len(r.active[5]) > 0
    L = orc.lib()
    dt = 0.5 * r.dtnew[l]
    unew_o = np.zeros_like(r.uold)
    L.orc_set_unew(C.byref(r.p), r.mp, l, orc.dptr(r.uold), orc.dptr(unew_o))
    # pretend the finer level has already refluxed into unew (the kernel must add to what is there)
    U0 = unew_o.reshape(5, r.ncell)
    rng = np.random.default_rng(2)
    for ind in range(8):
        c = r.ncoarse + ind * r.ngridmax + act - 1
        U0[:, c] += 1e-3 * rng.standard_normal((5, len(act))) * (r.son[c + 1] == 0)
    start = unew_o.copy()
    L.orc_godunov_fine(C.byref(r.p), r.mp, l, dt, orc.dptr(r.uold), orc.dptr(unew_o), 1)
    # device layout of the level: oct position -> slot
    pos = np.rint(r.xg[:, act] * 2 ** (l - 1) - 0.5).astype(np.int64)                # oct centre = (p+0.5)/2^(l-1)
    assert len(set(map(tuple, pos.T))) == len(act)
    h = N // 2
    slot = pos[0] + h * (pos[1] + h * pos[2])
    Uold, Ust, Uref = r.uold.reshape(5, r.ncell), start.reshape(5, r.ncell), unew_o.reshape(5, r.ncell)
    uin, uout, ref = np.zeros((5, 8, h ** 3)), np.zeros((5, 8, h ** 3)), np.zeros((5, 8, h ** 3))
    refined = np.zeros((8, h ** 3), dtype=np.uint8)
    for ind in range(8):
        c = r.ncoarse + ind * r.ngridmax + act - 1
        uin[:, ind, slot], uout[:, ind, slot], ref[:, ind, slot] = Uold[:, c], Ust[:, c], Uref[:, c]
        refined[ind, slot] = r.son[c + 1] > 0
    assert refined.sum() > 0
    sid = {"llf": 0, "exact": 1, "acoustic": 2, "hllc": 3, "hll": 4}[solver]
    uout = np.ascontiguousarray(uout)
    dev.devnum_sweep_dense_amr(sid, N, 4, orc.dptr(np.ascontiguousarray(uin)), orc.dptr(uout),
                               np.ascontiguousarray(refined).ctypes.data_as(C.POINTER(C.c_ubyte)), dt, 1.0 / N, 1, 1.5, 1.4, 1e-10, 1e-10, 10)
    assert np.abs(ref - uin).max() > 1e-5
    assert np.array_equal(uout, ref)


@pytest.mark.parametrize("solver", ["llf", "exact", "acoustic", "hllc", "hll"])
def test_vec_solvers_equal_scalar(orc, dev, solver):
    """hydro_vec.cuh: the branch-free scalar form and the 3-lane form of every solver == the branching scalar solver of
    hydro_device.cuh (which the test above ties to the oracle), bit for bit on 30 000 random face states."""
    dp = C.POINTER(C.c_double)
    dev.devnum_riemann_vec.argtypes = [C.c_int, C.c_int, dp, dp, dp, dp, C.c_double, C.c_double, C.c_double, C.c_int]
    n = 30000
    ql, qr = _hydro_states(np.random.default_rng(77 + len(solver)), n, 3)
    # supersonic pairs in both directions (the SL>0 / SR<0 branches of hllc, spout<0 of the samplers)
    ql[100:200, 1] = 50.0; qr[100:200, 1] = 50.0
    ql[200:300, 1] = -50.0; qr[200:300, 1] = -50.0
    sid = {"llf": 0, "exact": 1, "acoustic": 2, "hllc": 3, "hll": 4}[solver]
    for smallr, smallc in FLOORS.values():
        ref, f1, f3 = np.zeros((n, 5)), np.zeros((n, 5)), np.zeros((n, 5))
        dev.devnum_riemann(3, sid, n, orc.dptr(ql), orc.dptr(qr), orc.dptr(ref), 1.4, smallr, smallc, 10)
        dev.devnum_riemann_vec(sid, n, orc.dptr(ql), orc.dptr(qr), orc.dptr(f1), orc.dptr(f3), 1.4, smallr, smallc, 10)
        assert np.isfinite(ref).all()
        assert np.array_equal(f1, ref)
        assert np.array_equal(f3, ref)


@pytest.mark.parametrize("solver,st,N,nblocks,by,vec", [("hllc", 1, 16, 3, 12, 1), ("hllc", 2, 16, 2, 12, 0), ("hllc", 1, 16, 5, 12, 2),
                                                        ("exact", 1, 16, 2, 12, 1), ("llf", 8, 16, 4, 8, 1), ("hll", 7, 16, 3, 16, 1),
                                                        ("acoustic", 3, 16, 3, 12, 1), ("hllc", 1, 32, 7, 12, 1), ("exact", 2, 32, 5, 8, 1),
                                                        ("hllc", 1, 16, 3, 12, 12), ("hllc", 2, 32, 5, 12, 12), ("exact", 1, 32, 4, 16, 12),
                                                        ("hllc", 1, 16, 3, 12, 41), ("hllc", 2, 32, 5, 12, 41), ("exact", 1, 32, 4, 12, 40),
                                                        ("llf", 8, 32, 3, 12, 42), ("hllc", 3, 16, 2, 8, 41)])
def test_sweep3_kernel_emulated_on_the_cpu_equals_oracle(orc, dev, solver, st, N, nblocks, by, vec):
    """sweep3_kernel (sweep_dense3.cuh, the round-2 form of the hot kernel: 3-lane branch-free face solves, two barriers per
    plane, face states formed before the solve) executed on the CPU by the emulated launch: the new state equals one level
    step of the oracle bit for bit and the fused Courant partials give the oracle's next time step; tile heights 8/12/16,
    solver forms 0 (branching scalar), 1 (3-lane), 2 (branch-free scalar)."""
    dp = C.POINTER(C.c_double)
    dev.devnum_sweep3.argtypes = [C.c_int, C.c_int, C.c_int, dp, dp, C.c_double, C.c_double, C.c_int, C.c_double, C.c_double,
                                  C.c_double, C.c_double, C.c_double, C.c_int, dp, C.c_int, C.c_int]
    from helpers import Case, smooth_state
    level = int(np.log2(N))
    c = Case(3, level, riemann=solver, slope_type=st, slope_theta=1.3)
    d0 = smooth_state(3, N)
    rough = np.random.default_rng(3).standard_normal(d0[0].shape)
    d0[0] *= 1 + 0.3 * (rough > 1.2)
    c.init_dense(d0)
    dt, _ = c.oracle_courant()
    unew = c.oracle_godunov(dt, nthreads=1)
    ref = c.dense(unew)
    dt_next, sums = c.oracle_courant(unew)
    uin, ind, slot = _hydro_to_slots(c.dense(), 3, N)
    uout = np.zeros_like(uin)
    part = np.zeros(4 * 64)
    sid = {"llf": 0, "exact": 1, "acoustic": 2, "hllc": 3, "hll": 4}[solver]
    nb = dev.devnum_sweep3(sid, N, nblocks, orc.dptr(np.ascontiguousarray(uin)), orc.dptr(uout), dt, 1.0 / N, st, 1.3, 0.8,
                           1.4, 1e-10, 1e-10, 10, orc.dptr(part), by, vec)
    got = uout[:, ind.ravel(), slot.ravel()].reshape(ref.shape)
    assert np.abs(ref - c.dense()).max() > 1e-4
    assert np.array_equal(got, ref)
    p4 = part[:4 * nb].reshape(4, nb)
    assert p4[0].min() * 1.0 == dt_next or min(p4[0].min(), c.p.boxlen / c.p.smallc) == dt_next
    vol = (1.0 / N) ** 3
    assert abs(p4[1].sum() * vol - sums[0]) <= 1e-13 * abs(sums[0]) and abs(p4[2].sum() * vol - sums[1]) <= 1e-13 * abs(sums[1])


# ---- non-cubic boxes: per-axis extents, tile counts that do not divide them, thin periodic axes, a ghost shell on one axis ----
SOLVER_ID = {"llf": 0, "exact": 1, "acoustic": 2, "hllc": 3, "hll": 4}
IP3 = C.c_int * 3


def _box_case(ndim, level, coarse, bound, solver, st, order=1, seed=2):
    """oracle run set-up on a domain of `coarse` coarse cells (boxlen = coarse[0]: dx = 2^-level) with a box_state that has no
    symmetry to hide a swapped axis; returns the case, the owned extent in cells, dt and the oracle's new state"""
    from helpers import Case, box_state
    c = Case(ndim, level, riemann=solver, slope_type=st, slope_theta=1.3, bound=bound, coarse=coarse, boxlen=float(coarse[0]),
             order=order, seed=seed)
    ext = c.mesh.extent(level)
    c.init_dense(box_state(ndim, ext))
    dt, _ = c.oracle_courant()
    unew = c.oracle_godunov(dt, nthreads=1)
    return c, ext, dt, unew


def _check_box_result(c, uout, act, slot, unew, part, nb, ndim):
    """the owned cells of uout == the oracle's unew, bit for bit; the fused Courant partials give the oracle's next dt"""
    s = c.mesh.s
    T = 1 << ndim
    nv = getattr(c, "nvs", c.nvar)                         # MHD: 11 stored variables
    U, U0 = unew.reshape(nv, s.ncell), c.u.reshape(nv, s.ncell)
    moved = 0.0
    for ind in range(T):
        cells = s.ncoarse + ind * s.ngridmax + act - 1
        moved = max(moved, np.abs(U[:, cells] - U0[:, cells]).max())
        assert np.array_equal(uout[:, ind, slot], U[:, cells]), (ind, float(np.abs(uout[:, ind, slot] - U[:, cells]).max()))
    assert moved > 1e-4
    if part is not None:
        dt_next, sums = c.oracle_courant(unew)
        p4 = part[:4 * nb].reshape(4, nb)
        assert min(p4[0].min(), c.p.boxlen / c.p.smallc) == dt_next
        vol = (2.0 ** -c.level) ** ndim
        assert abs(p4[1].sum() * vol - sums[0]) <= 1e-13 * abs(sums[0])


@pytest.mark.parametrize("coarse,level,bound,solver,st,nblocks,by,vec", [
    ((3, 2, 1), 4, (0,) * 6, "hllc", 1, 7, 12, 1),              # 48 x 32 x 16
    ((1, 3, 2), 4, (0,) * 6, "exact", 2, 5, 8, 1),              # 16 x 48 x 32
    ((2, 1, 3), 4, (0,) * 6, "llf", 8, 5, 16, 1),               # 32 x 16 x 48
    ((3, 2, 1), 4, (0,) * 6, "hll", 3, 11, 12, 2),
    ((1, 3, 2), 4, (0,) * 6, "acoustic", 7, 7, 12, 41),         # one-barrier form (sweep_dense4.cuh)
    ((2, 1, 3), 4, (0,) * 6, "hllc", 2, 7, 12, 12),
    ((4, 2, 1), 2, (0,) * 6, "hllc", 1, 3, 12, 1),              # 16 x 8 x 4: 4-cell periodic z
    ((8, 4, 1), 1, (0,) * 6, "llf", 2, 3, 8, 1),                # 16 x 8 x 2: 2-cell periodic z
    ((1, 4, 8), 1, (0,) * 6, "hllc", 1, 3, 12, 1),              # 2 x 8 x 16: 2-cell periodic x
    ((3, 2, 1), 3, (1, 1, 0, 0, 0, 0), "hllc", 2, 5, 12, 1),    # 24 x 16 x 8, reflexive x walls: shell on x only
    ((2, 1, 3), 3, (0, 0, 0, 0, 2, 2), "exact", 1, 5, 8, 1),    # 16 x 8 x 24, outflow z faces: shell on z only
])
def test_sweep3_kernel_emulated_on_non_cubic_boxes(orc, dev, coarse, level, bound, solver, st, nblocks, by, vec):
    """sweep3_kernel / sweep4_kernel on boxes whose three extents differ (each axis the long one once, none a multiple of the
    30 x (by-2) tile), on thin periodic axes of 2 and 4 cells (the 2-cell halo and the 3-plane z warm-up wrap more than once) and
    on boxes with a ghost shell on one axis only: the owned cells equal one level step of the oracle bit for bit, and the fused
    Courant partials give the oracle's next time step.  nblocks never divides the work count."""
    dev.devnum_sweep3_box.argtypes = [C.c_int, IP3, IP3, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_double,
                                      C.c_double, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int,
                                      C.POINTER(C.c_double), C.c_int, C.c_int]
    from helpers import level_slots
    c, ext, dt, unew = _box_case(3, level, coarse, bound, solver, st)
    shell = [int(bound[2 * d] > 0) for d in range(3)]
    uin, act, slot = level_slots(c.mesh, level, c.u, 5)
    uout = np.zeros_like(uin)
    part = np.zeros(4 * 64)
    nb = dev.devnum_sweep3_box(SOLVER_ID[solver], IP3(*ext), IP3(*shell), nblocks, orc.dptr(uin), orc.dptr(uout), dt,
                               2.0 ** -level, st, 1.3, 0.8, 1.4, 1e-10, 1e-10, 10, orc.dptr(part), by, vec)
    ntx, nty = -(-ext[0] // 30), -(-ext[1] // (by - 2))
    assert nb == nblocks and (ntx * nty * ext[2]) % nblocks != 0
    _check_box_result(c, uout, act, slot, unew, part, nb, 3)


@pytest.mark.parametrize("ndim,coarse,level,bound,solver,st,nblocks", [
    (1, (5, 1, 1), 3, (0,) * 6, "hllc", 2, 1),                  # 40 cells
    (1, (5, 1, 1), 3, (1, 1, 0, 0, 0, 0), "exact", 1, 2),       # 40 cells between walls
    (2, (3, 2, 1), 4, (0,) * 6, "llf", 8, 5),                   # 48 x 32
    (2, (3, 2, 1), 4, (0, 0, 1, 1, 0, 0), "hll", 3, 3),         # 48 x 32, walls in y
    (2, (1, 4, 1), 2, (0,) * 6, "acoustic", 1, 2),              # 4 x 16
    (3, (3, 2, 1), 3, (0,) * 6, "hllc", 7, 4),                  # 24 x 16 x 8
    (3, (1, 2, 3), 3, (2, 2, 0, 0, 0, 0), "hllc", 1, 5),        # 8 x 16 x 24, outflow x
    (3, (8, 4, 1), 1, (0,) * 6, "hllc", 2, 3),                  # 16 x 8 x 2: 2-cell periodic z
    (3, (1, 4, 2), 2, (0,) * 6, "exact", 1, 2),                 # 4 x 16 x 8: 4-cell periodic x
])
def test_dense_sweep_kernel_emulated_on_non_cubic_boxes(orc, dev, ndim, coarse, level, bound, solver, st, nblocks):
    """sweep_dense_kernel (1-D, 2-D and 3-D forms) on boxes of several coarse cells with different extents per axis, periodic or
    with a ghost shell on one axis: the owned cells equal one level step of the oracle bit for bit."""
    dev.devnum_sweep_dense_box.argtypes = [C.c_int, C.c_int, IP3, IP3, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double),
                                           C.c_double, C.c_double, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double,
                                           C.c_int, C.POINTER(C.c_double), C.c_int]
    from helpers import level_slots
    c, ext, dt, unew = _box_case(ndim, level, coarse, bound, solver, st)
    shell = [int(bound[2 * d] > 0) for d in range(3)]
    uin, act, slot = level_slots(c.mesh, level, c.u, ndim + 2)
    uout = np.zeros_like(uin)
    part = np.zeros(4 * 64)
    nb = dev.devnum_sweep_dense_box(ndim, SOLVER_ID[solver], IP3(*ext), IP3(*shell), nblocks, orc.dptr(uin), orc.dptr(uout), dt,
                                    2.0 ** -level, st, 1.3, 0.8, 1.4, 1e-10, 1e-10, 10, orc.dptr(part), 0)
    _check_box_result(c, uout, act, slot, unew, part, nb, ndim)


@pytest.mark.parametrize("coarse,level,bound,r1d,r2d,st", [
    ((3, 2, 1), 3, (0,) * 6, "roe", "llf", 1),                   # 24 x 16 x 8
    ((3, 2, 1), 3, (0,) * 6, "hlld", "hlld", 2),
    ((1, 3, 2), 3, (0,) * 6, "llf", "hll", 1),                   # 8 x 24 x 16
    ((1, 2, 1), 3, (2, 2, 0, 0, 0, 0), "hlld", "hlld", 1),       # 8 x 16 x 8 between zero-gradient x ends
    ((8, 4, 1), 1, (0,) * 6, "hlld", "hlld", 2),                 # 16 x 8 x 2: 2-cell periodic z
    ((1, 4, 2), 2, (0,) * 6, "roe", "llf", 1),                   # 4 x 16 x 8: 4-cell periodic x
])
def test_mhd_six_pass_kernels_emulated_on_non_cubic_boxes(orc, dev, coarse, level, bound, r1d, r2d, st):
    """the six MHD passes of mhd_dense.cuh (cells decoded with ncx / ncy, W indexed [ncz][ncy][ncx]) on boxes of several coarse
    cells with different extents per axis, periodic or between zero-gradient x ends: the owned cells equal set_unew + godunov_fine
    of the oracle, bit for bit (both copies of every face field)."""
    from helpers import MhdCase, level_slots, mhd_box_state
    c = MhdCase(level, riemann=r1d, riemann2d=r2d, slope_type=st, bound=bound, coarse=coarse, boxlen=float(coarse[0]), order=2,
                seed=3)
    ext = c.mesh.extent(level)
    d0 = mhd_box_state(ext)
    d0[0] *= 1 + 0.2 * (np.random.default_rng(4).standard_normal(d0[0].shape) > 1.3)
    c.init_dense(d0)
    dt, _ = c.oracle_courant()
    dt *= 0.7
    unew = c.oracle_godunov(dt, nthreads=2)
    shell = [int(bound[2 * d] > 0) for d in range(3)]
    uin, act, slot = level_slots(c.mesh, level, c.u, 11)
    uout = np.zeros_like(uin)
    dev.devnum_mhd_sweep_box(IP3(*ext), IP3(*shell), orc.MHD_RIEMANN[r1d], orc.MHD_RIEMANN2D[r2d], 0 if st == 0 else 1,
                             orc.dptr(uin), orc.dptr(uout), dt, 2.0 ** -level, c.p.gamma, c.p.smallr, c.p.smallc, st, st,
                             c.p.slope_theta, c.p.courant_factor)
    _check_box_result(c, uout, act, slot, unew, None, 0, 3)


@pytest.mark.parametrize("coarse,bound", [((3, 2, 1), (0,) * 6), ((1, 3, 2), (0,) * 6), ((3, 2, 2), (1, 1, 0, 0, 2, 2))])
def test_amr_tree_walks_across_coarse_cells_equal_oracle(orc, dev, coarse, bound):
    """amr_get3cubefather / amr_getnborfather of amr_kernels.cuh on a domain of several coarse cells (with and without boundary
    coarse cells): the level-1 walks decode coarse cells with nx, ny, nz and wrap over the coarse grid; every oct of levels 1-3
    and every cell of levels 0-2 give the oracle's neighbour cells"""
    from helpers import Case
    lev = 3
    m = Case(3, lev, bound=bound, coarse=coarse, order=2, seed=5).mesh
    s = m.s
    assert (s.nx, s.ny, s.nz) == tuple(coarse[d] + (bound[2 * d] > 0) + (bound[2 * d + 1] > 0) for d in range(3))
    son = np.ascontiguousarray(m.son()[1:], dtype=np.int32)
    father = np.ascontiguousarray(m.father()[1:], dtype=np.int32)
    nbor = np.ascontiguousarray(m.nbor()[:, 1:], dtype=np.int32)
    geo = (3, s.ncoarse, s.ngridmax, s.nx, s.ny, s.nz)
    L = orc.lib()
    L.orc_getnborfather.argtypes = [C.POINTER(orc.MeshS), C.c_int, C.c_int, C.POINTER(C.c_int)]
    buf27, buf7 = (C.c_int * 27)(), (C.c_int * 7)()
    for l in range(1, lev + 1):
        act = np.ascontiguousarray(m.active(l), dtype=np.int32)
        got = np.zeros((len(act), 27), dtype=np.int32)
        dev.devnum_amr_get3cubefather(*geo, orc.iptr(son), orc.iptr(father), orc.iptr(nbor), len(act), orc.iptr(act), l, orc.iptr(got))
        ref = np.zeros_like(got)
        for i, g in enumerate(act):
            L.orc_get3cubefather(m.ptr, int(father[g - 1]), l, buf27, None)
            ref[i] = buf27[:27]
        assert (ref > 0).all() and np.array_equal(got, ref)
        if l == 1:   # the coarse cells of the domain: the level-1 branch of getnborfather
            cells = np.arange(1, s.ncoarse + 1, dtype=np.int32)
        else:
            prev = m.active(l - 1).astype(np.int64)
            cells = np.array([s.ncoarse + ind * s.ngridmax + g for g in prev for ind in range(8)], dtype=np.int32)
        got = np.zeros((len(cells), 7), dtype=np.int32)
        dev.devnum_amr_getnborfather(*geo, orc.iptr(son), orc.iptr(father), orc.iptr(nbor), len(cells), orc.iptr(cells), l,
                                     orc.iptr(got))
        ref = np.zeros_like(got)
        for i, c in enumerate(cells):
            L.orc_getnborfather(m.ptr, int(c), l, buf7)
            ref[i] = buf7[:7]
        assert np.array_equal(got, ref)


@pytest.mark.parametrize("coarse,bound,solver,nblocks", [((3, 2, 1), (0,) * 6, "hllc", 5), ((1, 2, 3), (2, 2, 0, 0, 0, 0), "llf", 7)])
def test_dense_sweep_amr_variant_emulated_on_non_cubic_boxes(orc, dev, coarse, bound, solver, nblocks):
    """sweep_dense_kernel<..., AMRV=true> on a 48x32x16 periodic base level and on a 16x32x48 base level between outflow x ends, a
    scattered tenth of its cells marked refined (son > 0): fluxes through refined faces reset, the update accumulated into a unew
    that already holds the finer level's refluxes -- equals set_unew + godunov_fine of the oracle on that level, bit for bit"""
    _dense_amr_box_compare(orc, dev, coarse, bound, solver, nblocks)


def _dense_amr_box_compare(orc, dev, coarse, bound, solver, nblocks, floors=None):
    """the body of the test above; floors = a key of helpers.FLOORS: a floor_state under those floors in place of the box_state"""
    from helpers import FLOORS, Case, box_state, floor_state, level_slots
    smallr, smallc = FLOORS[floors] if floors else (1e-10, 1e-10)
    dev.devnum_sweep_dense_amr_box.argtypes = [C.c_int, IP3, IP3, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double),
                                               C.POINTER(C.c_ubyte), C.c_double, C.c_double, C.c_int, C.c_double, C.c_double,
                                               C.c_double, C.c_double, C.c_int]
    lev = 4
    c = Case(3, lev, riemann=solver, slope_type=1, bound=bound, coarse=coarse, boxlen=float(coarse[0]), order=2, seed=8,
             smallr=smallr, smallc=smallc)
    ext = c.mesh.extent(lev)
    c.init_dense(floor_state(3, ext, 8, smallr, smallc) if floors else box_state(3, ext))
    s = c.mesh.s
    act = c.mesh.active(lev).astype(np.int64)
    cells = np.concatenate([s.ncoarse + ind * s.ngridmax + act for ind in range(8)])        # 1-based
    son = c.mesh.son()
    rng = np.random.default_rng(3)
    ref_cells = cells[rng.random(len(cells)) < 0.1]
    son[ref_cells] = 1                                     # marked refined: godfine1 only tests son > 0 on its own level
    try:
        dt, _ = c.oracle_courant()
        L = orc.lib()
        unew = np.zeros_like(c.u)
        L.orc_set_unew(C.byref(c.p), c.mesh.ptr, lev, orc.dptr(c.u), orc.dptr(unew))
        U = unew.reshape(5, s.ncell)
        U[:, cells - 1] += 1e-3 * rng.standard_normal((5, len(cells))) * (son[cells] == 0)    # refluxes of a finer level
        start = unew.copy()
        L.orc_godunov_fine(C.byref(c.p), c.mesh.ptr, lev, dt, orc.dptr(c.u), orc.dptr(unew), 1)
    finally:
        son[ref_cells] = 0
    uin, act_, slot = level_slots(c.mesh, lev, c.u, 5)
    uout, _, _ = level_slots(c.mesh, lev, start, 5)
    refined = np.zeros(uin.shape[1:], dtype=np.uint8)
    for ind in range(8):
        refined[ind, slot] = np.isin(s.ncoarse + ind * s.ngridmax + act, ref_cells)
    assert refined.sum() == len(ref_cells) > 0
    shell = [int(bound[2 * d] > 0) for d in range(3)]
    unmasked = uout.copy()
    for mask, out in ((refined, uout), (np.zeros_like(refined), unmasked)):
        dev.devnum_sweep_dense_amr_box(SOLVER_ID[solver], IP3(*ext), IP3(*shell), nblocks, orc.dptr(uin), orc.dptr(out),
                                       mask.ctypes.data_as(C.POINTER(C.c_ubyte)), dt, 2.0 ** -lev, 1, 1.5, 1.4, smallr, smallc, 10)
    assert not np.array_equal(unmasked, uout)              # the marks matter
    assert np.isfinite(unew).all()
    Un, Us = unew.reshape(5, s.ncell), start.reshape(5, s.ncell)
    moved = 0.0
    for ind in range(8):
        cc = s.ncoarse + ind * s.ngridmax + act - 1
        moved = max(moved, np.abs(Un[:, cc] - Us[:, cc]).max())
        assert np.array_equal(uout[:, ind, slot], Un[:, cc]), (ind, float(np.abs(uout[:, ind, slot] - Un[:, cc]).max()))
    assert moved > 1e-5


# ---- the floors: near-vacuum and cold hypersonic states on which smallr / smalle fire (helpers.floor_state) ----
def _floor_case(ndim, ext, solver, st, floors, seed, bound=(0,) * 6):
    """oracle level step on a floor_state of ext cells (one coarse cell per 16 cells in x: dx = 1/16) under the floors
    helpers.FLOORS[floors]; asserts the state makes the ctoprim floors fire and the oracle stays finite"""
    from helpers import FLOORS, Case, floor_counts, floor_state
    smallr, smallc = FLOORS[floors]
    level = 4 if ext[0] >= 16 else int(np.log2(ext[0]))
    coarse = tuple(max(e >> level, 1) for e in ext)
    c = Case(ndim, level, riemann=solver, slope_type=st, slope_theta=1.3, bound=bound, coarse=coarse, boxlen=float(coarse[0]),
             order=1, seed=2, smallr=smallr, smallc=smallc)
    assert tuple(c.mesh.extent(level))[:ndim] == tuple(ext)[:ndim]
    d0 = floor_state(ndim, c.mesh.extent(level), seed, smallr, smallc)
    nrho, neint = floor_counts(d0, ndim, smallr, smallc)
    ncell = d0[0].size
    assert min(nrho, neint) >= max(2, 0.02 * ncell), (nrho, neint)
    c.init_dense(d0)
    dt, _ = c.oracle_courant()
    unew = c.oracle_godunov(dt, nthreads=1)
    assert np.isfinite(dt) and dt > 0 and np.isfinite(unew).all()
    return c, c.mesh.extent(level), dt, unew


@pytest.mark.parametrize("floors", ["default", "raised"])
@pytest.mark.parametrize("solver,st,nblocks,by,vec", [("llf", 1, 3, 12, 1), ("exact", 2, 2, 12, 1), ("acoustic", 8, 3, 12, 1),
                                                      ("hllc", 1, 5, 12, 0), ("hll", 2, 3, 16, 2), ("hllc", 8, 3, 12, 12),
                                                      ("exact", 1, 4, 12, 40), ("hllc", 2, 5, 12, 41), ("llf", 8, 3, 12, 42),
                                                      ("hll", 1, 4, 8, 41)])
def test_sweep3_kernel_emulated_at_the_floors(orc, dev, floors, solver, st, nblocks, by, vec):
    """sweep3_kernel (solver forms 0 / 1 / 2, the 12 form) and sweep4_kernel (40-42) on a 16^3 floor_state: near-vacuum cells
    whose six face densities the predictor drives below smallr (the y face passing through shared memory), densities below
    smallr and cold hypersonic cells with E/rho - ekin below smalle, under the RAMSES floors and raised ones -- the new state and
    the fused Courant partials equal the oracle's, bit for bit"""
    from helpers import level_slots
    c, ext, dt, unew = _floor_case(3, (16, 16, 16), solver, st, floors, 11 + vec)
    uin, act, slot = level_slots(c.mesh, c.level, c.u, 5)
    uout = np.zeros_like(uin)
    part = np.zeros(4 * 64)
    nb = dev.devnum_sweep3_box(SOLVER_ID[solver], IP3(*ext), IP3(0, 0, 0), nblocks, orc.dptr(uin), orc.dptr(uout), dt,
                               2.0 ** -c.level, st, 1.3, 0.8, 1.4, c.p.smallr, c.p.smallc, 10, orc.dptr(part), by, vec)
    _check_box_result(c, uout, act, slot, unew, part, nb, 3)


@pytest.mark.parametrize("floors", ["default", "raised"])
@pytest.mark.parametrize("ndim,ext,bound,solver,st,nblocks", [
    (1, (64, 1, 1), (0,) * 6, "hllc", 2, 2),
    (1, (64, 1, 1), (1, 1, 0, 0, 0, 0), "exact", 1, 1),
    (2, (32, 32, 1), (0,) * 6, "llf", 8, 3),
    (2, (32, 32, 1), (0, 0, 2, 2, 0, 0), "acoustic", 1, 2),
    (3, (16, 16, 16), (0,) * 6, "hll", 2, 3),
    (3, (16, 16, 16), (0,) * 6, "exact", 8, 4),
    (3, (16, 16, 16), (1, 1, 0, 0, 0, 0), "hllc", 1, 5),
])
def test_dense_sweep_kernel_emulated_at_the_floors(orc, dev, floors, ndim, ext, bound, solver, st, nblocks):
    """sweep_dense_kernel (1-D, 2-D and 3-D forms) on a floor_state, periodic or with a wall / outflow shell: ctoprim's density and
    internal-energy floors and the face-density resets of the predictor fire; the owned cells and the fused Courant partials
    equal the oracle's, bit for bit"""
    from helpers import level_slots
    c, ext, dt, unew = _floor_case(ndim, ext, solver, st, floors, 5 + nblocks, bound=bound)
    shell = [int(bound[2 * d] > 0) for d in range(3)]
    uin, act, slot = level_slots(c.mesh, c.level, c.u, ndim + 2)
    uout = np.zeros_like(uin)
    part = np.zeros(4 * 64)
    nb = dev.devnum_sweep_dense_box(ndim, SOLVER_ID[solver], IP3(*ext), IP3(*shell), nblocks, orc.dptr(uin), orc.dptr(uout), dt,
                                    2.0 ** -c.level, st, 1.3, 0.8, 1.4, c.p.smallr, c.p.smallc, 10, orc.dptr(part), 0)
    _check_box_result(c, uout, act, slot, unew, part, nb, ndim)


@pytest.mark.parametrize("floors", ["default", "raised"])
@pytest.mark.parametrize("solver", ["hllc", "exact"])
def test_dense_sweep_amr_variant_emulated_at_the_floors(orc, dev, floors, solver):
    """sweep_dense_kernel<..., AMRV=true> on a 48x32x16 base level holding a floor_state, a tenth of its cells marked refined:
    equals set_unew + godunov_fine of the oracle, bit for bit"""
    _dense_amr_box_compare(orc, dev, (3, 2, 1), (0,) * 6, solver, 5, floors=floors)


# ---- MHD at the floors and where the field degenerates (helpers.mhd_floor_state, helpers.fill_mhd_floor_cells) ----
MHD_FLOOR_PAIRS = [("roe", "llf", 0, 0), ("hlld", "hlld", 1, 1), ("llf", "llf", 2, 2), ("hll", "hll", 1, 1), ("hlld", "roe", 2, 2),
                   ("upwind", "upwind", 1, 1), ("hydro", "hlla", 1, 1), ("hlld", "hlld", 3, 1), ("roe", "llf", 7, 2),
                   ("hll", "hlld", 8, 1)]


def _mhd_floor_case(coarse, level, bound, r1d, r2d, st, smt, floors, seed):
    """MhdCase on `coarse` domain cells (dx = 2^-level) holding an mhd_floor_state under helpers.FLOORS[floors]: asserts the
    density / pressure floors fire, field-free and field-aligned (vA > c_s) cells are present, and the oracle's level step is
    finite; returns the case, dt and the oracle's unew"""
    from helpers import FLOORS, MhdCase, mhd_floor_counts, mhd_floor_state
    smallr, smallc = FLOORS[floors]
    c = MhdCase(level, riemann=r1d, riemann2d=r2d, slope_type=st, slope_mag_type=smt, bound=bound, coarse=coarse,
                boxlen=float(coarse[0]), order=2, seed=3, smallr=smallr, smallc=smallc)
    ext = c.mesh.extent(level)
    d0 = mhd_floor_state(ext, seed, smallr, smallc, slab_vt=0.3 if r2d == "hlla" else 0.0)
    nrho, npr, nfree, nfast = mhd_floor_counts(d0, smallr, smallc)
    ncell = d0[0].size
    assert min(nrho, npr) >= 0.02 * ncell and nfree >= 0.05 * ncell and nfast >= 10, (nrho, npr, nfree, nfast)
    c.init_dense(d0)
    dt, _ = c.oracle_courant()
    assert np.isfinite(dt) and dt > 0
    dt *= 0.7
    unew = c.oracle_godunov(dt, nthreads=4)
    assert np.isfinite(unew).all()
    return c, ext, dt, unew


@pytest.mark.parametrize("floors", ["default", "raised"])
@pytest.mark.parametrize("box", ["cube", "shell"])
@pytest.mark.parametrize("r1d,r2d,st,smt", MHD_FLOOR_PAIRS)
def test_mhd_six_pass_kernels_emulated_at_the_floors(orc, dev, floors, box, r1d, r2d, st, smt):
    """the six MHD passes of mhd_dense.cuh on an mhd_floor_state -- a periodic 16^3 box, and a 24x16x8 box between zero-gradient
    x ends -- under the RAMSES floors and raised ones: ctoprim's pressure floor, the density / pressure clamps of every traced
    face and edge state, the field-free sub-box (1-D solvers reduce to hydro, the smallc floor of the 2-D HLLD Alfven speeds) and
    the field-aligned slab (HLLD's degenerate star state, Roe's bt = 0 branch) are all at work; the owned cells equal set_unew +
    godunov_fine of the oracle, bit for bit (both copies of every face field)"""
    from helpers import level_slots
    coarse, level, bound = ((1, 1, 1), 4, (0,) * 6) if box == "cube" else ((3, 2, 1), 3, (2, 2, 0, 0, 0, 0))
    c, ext, dt, unew = _mhd_floor_case(coarse, level, bound, r1d, r2d, st, smt, floors, 21 + st)
    shell = [int(bound[2 * d] > 0) for d in range(3)]
    uin, act, slot = level_slots(c.mesh, level, c.u, 11)
    uout = np.zeros_like(uin)
    dev.devnum_mhd_sweep_box(IP3(*ext), IP3(*shell), orc.MHD_RIEMANN[r1d], orc.MHD_RIEMANN2D[r2d], 0 if st == 0 else 1,
                             orc.dptr(uin), orc.dptr(uout), dt, 2.0 ** -level, c.p.gamma, c.p.smallr, c.p.smallc, st, smt,
                             c.p.slope_theta, c.p.courant_factor)
    s = c.mesh.s
    U, U0 = unew.reshape(11, s.ncell), c.u.reshape(11, s.ncell)
    moved = 0.0
    for ind in range(8):
        cells = s.ncoarse + ind * s.ngridmax + act - 1
        moved = max(moved, float(np.abs(U[:, cells] - U0[:, cells]).max()))
        assert np.array_equal(uout[:, ind, slot], U[:, cells]), (ind, float(np.abs(uout[:, ind, slot] - U[:, cells]).max()))
    assert moved > 0


def _mhd_box_floor_case(coarse, level, bound, floors, seed):
    """MhdCase (hlld / hlld, slope_type 1) holding an mhd_floor_state under helpers.FLOORS[floors], with the floors and the
    degenerate-field cells asserted present; returns the case and the owned extent"""
    from helpers import FLOORS, MhdCase, mhd_floor_counts, mhd_floor_state
    smallr, smallc = FLOORS[floors]
    c = MhdCase(level, riemann="hlld", riemann2d="hlld", slope_type=1, bound=bound, coarse=coarse, boxlen=float(coarse[0]), order=2,
                seed=3, smallr=smallr, smallc=smallc)
    ext = c.mesh.extent(level)
    d0 = mhd_floor_state(ext, seed, smallr, smallc)
    nrho, npr, nfree, nfast = mhd_floor_counts(d0, smallr, smallc)
    assert min(nrho, npr) >= 0.02 * d0[0].size and nfree > 0 and nfast > 0, (nrho, npr, nfree, nfast)
    c.init_dense(d0)
    return c, ext


@pytest.mark.parametrize("floors", ["default", "raised"])
@pytest.mark.parametrize("coarse,level,bound,nblocks", [((1, 1, 1), 4, (0,) * 6, 3), ((3, 2, 1), 3, (2, 2, 0, 0, 0, 0), 5),
                                                        ((1, 2, 1), 4, (1, 1, 2, 2, 0, 0), 2)])
def test_mhd_courant_kernel_emulated_at_the_floors(orc, dev, floors, coarse, level, bound, nblocks):
    """the stand-alone MHD Courant scan (mhd_courant_kernel: grid-stride loop over the owned cells, cmpdt with its density and
    pressure floors, warp and block reductions) on mhd_floor_state boxes, periodic or with a wall / outflow shell, under both
    helpers.FLOORS settings: the reduced time step equals orc_mhd_courant_fine's bit for bit, the mass / energy / internal /
    magnetic sums agree to 1e-12"""
    from helpers import level_slots
    c, ext = _mhd_box_floor_case(coarse, level, bound, floors, 51 + nblocks)
    dt_ref, sums = c.oracle_courant()
    assert np.isfinite(dt_ref) and dt_ref > 0 and np.isfinite(sums).all()
    uin, _, _ = level_slots(c.mesh, level, c.u, 11)
    shell = [int(bound[2 * d] > 0) for d in range(3)]
    part = np.zeros(5 * nblocks)
    dx = 2.0 ** -level
    dev.devnum_mhd_courant.argtypes = [IP3, IP3, C.c_int, C.POINTER(C.c_double), C.c_double, C.c_double, C.c_double, C.c_double,
                                       C.c_double, C.POINTER(C.c_double)]
    dev.devnum_mhd_courant(IP3(*ext), IP3(*shell), nblocks, orc.dptr(np.ascontiguousarray(uin)), dx, c.p.gamma, c.p.smallr,
                           c.p.smallc, c.p.courant_factor, orc.dptr(part))
    p5 = part.reshape(5, nblocks)
    assert min(p5[0].min(), c.p.courant_factor * dx / c.p.smallc, c.p.boxlen / c.p.smallc) == dt_ref
    got = p5[1:].sum(axis=1) * dx ** 3
    assert np.all(np.abs(got - sums) <= 1e-12 * np.abs(sums).max()), (got, sums)


def _oct_slots(mesh, l):
    """{oct index: slot} of the active and boundary octs of level l in the dense-box layout of level_slots"""
    act = mesh.active(l).astype(np.int64)
    ig = np.concatenate([act] + [mesh.bound(b, l).astype(np.int64) for b in range(mesh.s.nboundary)])
    pos = mesh._pos_fast(l, ig)
    q = pos - pos.min(axis=0)
    no = pos.max(axis=0) - pos.min(axis=0) + 1
    return dict(zip(ig.tolist(), (q[:, 0] + no[0] * (q[:, 1] + no[1] * q[:, 2])).tolist()))


@pytest.mark.parametrize("floors", ["default", "raised"])
@pytest.mark.parametrize("bound", [(2, 2, 0, 0, 0, 0), (1, 1, 2, 2, 0, 0), (2, 1, 1, 2, 1, 1), (2, 2, 2, 2, 2, 2)])
def test_mhd_boundary_kernel_emulated_at_the_floors(orc, dev, floors, bound):
    """make_boundary_hydro of the dense MHD path (mhd_boundary_kernel, one launch per boundary region in the reference's order)
    on a 16^3 mhd_floor_state between reflexive walls and zero-gradient ends, corner octs included: the ghost octs are scrambled
    first, then refilled by one pass; the zero-gradient branch removes and restores ekin with the density floored at smallr, which the
    near-vacuum cells next to the boundary take.  Every ghost oct equals orc_mhd_make_boundary_hydro's, bit for bit."""
    c, ext = _mhd_box_floor_case((1, 1, 1), 4, bound, floors, 61)
    m, s, lev = c.mesh, c.mesh.s, 4
    U = c.u.reshape(11, s.ncell)
    edge = np.zeros(tuple(ext[::-1]), dtype=bool)
    for d in range(3):
        if 2 in bound[2 * d:2 * d + 2]:
            edge[(slice(None),) * (2 - d) + ([0, -1],)] = True
    d0 = c.dense()
    assert (d0[0][edge] < c.p.smallr).sum() > 0                  # floored densities next to a zero-gradient face
    ghost = []
    for b in range(s.nboundary):
        for g in m.bound(b, lev).astype(np.int64):
            for ind in range(8):
                ghost.append(s.ncoarse + ind * s.ngridmax + g - 1)
    ghost = np.array(ghost)
    U[:, ghost] = 9.0
    from helpers import level_slots
    uin, _, _ = level_slots(m, lev, c.u, 11)
    uin = np.ascontiguousarray(uin)
    ref = c.u.copy()
    orc.lib().orc_mhd_make_boundary_hydro(C.byref(c.p), m.ptr, lev, orc.dptr(ref))
    slots = _oct_slots(m, lev)
    shell = [int(bound[2 * d] > 0) for d in range(3)]
    dev.devnum_mhd_boundary.argtypes = [IP3, IP3, C.c_int, C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_double), C.c_double]
    types = m.boundary_types()
    assert any(t // 10 == 1 for t in types)
    for b in range(s.nboundary):
        lst = np.array([slots[g] for g in m.bound(b, lev).astype(np.int64).tolist()], dtype=np.int32)
        if len(lst):
            dev.devnum_mhd_boundary(IP3(*ext), IP3(*shell), int(types[b]), orc.iptr(lst), len(lst), orc.dptr(uin), c.p.smallr)
    R = ref.reshape(11, s.ncell)
    refilled = ~(R[:, ghost] == 9.0).all(axis=0)      # corner octs that read a not yet refilled neighbour need a second pass
    assert np.isfinite(R[:, ghost]).all() and refilled.mean() > 0.5
    for b in range(s.nboundary):
        for g in m.bound(b, lev).astype(np.int64).tolist():
            for ind in range(8):
                got, exp = uin[:, ind, slots[g]], R[:, s.ncoarse + ind * s.ngridmax + g - 1]
                assert np.array_equal(got, exp), (b, g, ind, got - exp)


def _mhd_amr_floor_run(orc, ndim, r1, r2, slope_type, floors, field_scale, seed):
    """the refined meshes of the MHD AMR tests above (imhd-tube 1-D, Orszag-Tang 2-D, the nested 3-D mesh) with every cell
    overwritten by fill_mhd_floor_cells; returns the run and its godfine / upload / courant / boundary routines"""
    from helpers import fill_mhd_floor_cells
    L = orc.lib()
    if ndim == 1:
        from oracle.amr_mhd import MhdAmrRun
        from test_oracle_golden import IMHD
        r = MhdAmrRun(5, 9, (2, 2, 0, 0, 0, 0), 3.5, nsubcycle=[1, 1, 1, 1], riemann=r1, slope_type=slope_type, gamma=1.6666667,
                      courant_factor=0.8, err_grad_d=0.01, err_grad_u=0.05, err_grad_p=0.05, interpol_type=2, regions=IMHD,
                      tout=[1e9], ngridmax=10000)
        r.run(max_coarse=10)
        fns = (L.orc_mhd1_godunov_fine, L.orc_mhd1_upload_fine, L.orc_mhd1_courant_fine, L.orc_mhd1_make_boundary_hydro)
    elif ndim == 2:
        from oracle.amr_mhd import MhdAmrRun2D
        r = MhdAmrRun2D(4, 6, 1.0, nsubcycle=[1], riemann=r1, riemann2d=r2, slope_type=slope_type, gamma=1.6666667,
                        courant_factor=0.8, err_grad_p=0.1, interpol_type=2, tout=[1e9], nexpand=1, ngridmax=20000)
        r.run(max_coarse=6)
        fns = (L.orc_mhd2_godunov_fine, L.orc_mhdn_upload_fine, L.orc_mhdn_courant_fine, None)
    else:
        r = _mhd3_static_run(r1, r2, slope_type)
        fns = (L.orc_mhd3_godunov_fine, L.orc_mhdn_upload_fine, L.orc_mhdn_courant_fine, None)
    fill_mhd_floor_cells(r, floors, seed, field_scale)
    # a stable step for the new state: _mhd_amr_compare_levels advances level l by 0.5 dtnew(levelmin) / 2^(l - levelmin)
    dts = [fns[2](C.byref(r.pm), r.mp, l, r.p.boxlen / r.p.smallc, orc.dptr(r.uold)) * 2.0 ** (l - r.levelmin)
           for l in range(r.levelmin, r.nlevelmax + 1) if len(r.active[l])]
    r.dtnew[r.levelmin] = min(dts)
    return r, fns


@pytest.mark.parametrize("ndim,r1,r2,slope_type,field_scale,floors", [
    (1, "hlld", "llf", 1, 1.0, "default"), (1, "roe", "llf", 2, 1.0, "default"), (1, "hydro", "llf", 1, 0.0, "default"),
    (1, "hlld", "llf", 1, 1.0, "raised"), (1, "roe", "llf", 2, 1.0, "raised"), (1, "hydro", "llf", 1, 0.0, "raised"),
    (2, "hlld", "hlld", 2, 1.0, "raised"), (2, "roe", "llf", 1, 1.0, "raised"), (2, "hlld", "hlld", 1, 0.0, "raised"),
    (2, "llf", "roe", 2, 1.0, "raised"), (3, "hlld", "hlld", 2, 1.0, "raised"), (3, "roe", "roe", 1, 0.0, "raised")])
def test_mhd_amr_kernels_emulated_at_the_floors(orc, dev, ndim, r1, r2, slope_type, field_scale, floors):
    """the MHD AMR kernels (mhd_amr.cuh) in 1-D, 2-D and 3-D on refined meshes whose every cell holds floor-state draws
    (helpers.fill_mhd_floor_cells: densities down to 0.1 smallr, cold magnetised and cold hypersonic cells, magnetically dominated
    near-vacuum) with the mesh's own divergence-free face fields, or none (field_scale = 0: a field-free tree): ctoprim's
    floors, the trace resets, prolongation of floored father cells, upload_fine, cmpdt and (1-D) the outflow boundaries equal the
    oracle bit for bit on every level, refluxed coarse cells included.  (The 2-D and 3-D trees under the RAMSES floors are left
    out: there the oracle's own update is not finite -- NaN face fields from the corner EMFs of near-vacuum cells.)"""
    r, (god, upl, cour, bnd) = _mhd_amr_floor_run(orc, ndim, r1, r2, slope_type, floors, field_scale, 31 + ndim)
    if field_scale == 0:
        assert (r.uold.reshape(11, -1)[5:] == 0).all()
    nlev, nrefl, moved = _mhd_amr_compare_levels(orc, dev, r, ndim, r1, r2, slope_type, 2, god, upl, cour, boundary=bnd)
    assert nlev >= 3 and nrefl > 0 and moved > 0
