"""pressure_fix on levelmin=levelmax levels outside AMR mode, on the GPU: rgpu_level_steps and the per-level calls run the plain
PFIX form of the dense sweep and the dense set_unew / set_uold passes in 1-D, 2-D and 3-D.  Every run is compared with the oracle
under orc_set_pressure_fix in the state, divu, enew and the time steps, bit for bit ('exact': 1e-12, CUDA pow vs libm pow), and
with the same box through AMR mode."""
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import FLOORS, Case, box_state, fill_floor_state, max_rel_err
from test_gpu_pfix_dense import Sources

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu():
    from ramses_b200 import lib
    lib.load()
    return lib


def _case(ndim, coarse, level, bound, riemann, slope_type, seed=4, scale=1.0, floors=None, dense=None):
    from oracle import orc
    import ctypes as C
    smallr, smallc = FLOORS[floors] if floors else (1e-10, 1e-10)
    c = Case(ndim, level, riemann=riemann, slope_type=slope_type, bound=bound, coarse=coarse, boxlen=scale * coarse[0], order=2,
             seed=seed, smallr=smallr, smallc=smallc)
    c.init_dense(box_state(ndim, c.mesh.extent(level), seed=seed) if dense is None else dense)
    if floors:
        fill_floor_state(c.u, ndim, ndim + 2, c.mesh.s.ncell, floors, 50 + seed)
        orc.lib().orc_make_boundary_hydro(C.byref(c.p), c.mesh.ptr, level, orc.dptr(c.u))
    return c


def _oracle(c, nstep, beta_fix=0.5):
    with Sources(c.mesh.s.ncell, beta_fix) as src:
        ref, dts = c.oracle_steps(nstep, nthreads=1)
    return ref.reshape(c.nvar, -1), np.asarray(dts), src.divu, src.enew


def _gpu(c, nstep, mode="fused", beta_fix=0.5, fast=False):
    """nstep level steps with pressure_fix: 'fused' rgpu_level_steps, 'split' the per-level calls in amr_step order, 'amr' the
    per-level calls in AMR mode; returns (state, dts, divu, enew, level_info)"""
    from ramses_b200.hydro import HydroGPU
    a = c.amr_commons()
    a.pressure_fix, a.beta_fix, a.fast = True, beta_fix, fast
    level = c.level
    h = HydroGPU(a, amr_mode=(mode == "amr"))
    try:
        if mode == "amr":
            for l in range(1, level + 1):
                h.bind_level(l)
            h.upload_state(0)
            h.make_boundary_hydro(level)
        else:
            h.bind_level(level)
            h.upload_state(level)
        info = h.level_info(level)
        if mode == "fused":
            dts, _ = h.level_steps(level, nstep)
        else:
            dts = []
            for _ in range(nstep):
                a.dtnew[level] = a.boxlen / a.smallc
                dts.append(h.courant_fine(level))
                h.set_unew(level); h.godunov_fine_dev(level); h.set_uold(level)
                h.make_virtual_fine(level); h.make_boundary_hydro(level)
        h.download_state(0 if mode == "amr" else level)
        divu, enew = h.download_pressure_fix()
    finally:
        h.finalize()
    return a.uold.copy(), np.asarray(dts), divu, enew, info


def _check_oracle(c, got, want):
    u, dts, divu, enew = got[:4]
    ref, dts_ref, rdivu, renew = want
    idx = c.active_cells()
    g = np.concatenate([u[:, idx], divu[None, idx], enew[None, idx]])
    w = np.concatenate([ref[:, idx], rdivu[None, idx], renew[None, idx]])
    assert np.isfinite(w).all()
    assert np.abs(ref[:, idx] - c.u.reshape(c.nvar, -1)[:, idx]).max() > 1e-4
    assert np.abs(rdivu[idx]).max() > 0
    if c.riemann == "exact":
        assert np.allclose(dts, dts_ref, rtol=1e-12, atol=0)
        assert max_rel_err(g, w) <= 1e-12
    else:
        assert np.array_equal(dts, dts_ref), (dts, dts_ref)
        assert np.array_equal(g, w), [float(np.abs(g[n] - w[n]).max()) for n in range(len(g))]


ROWS = [   # ndim, coarse, level, bound, riemann, slope_type
    (1, (5, 1, 1), 5, (0,) * 6, "hllc", 2),
    (1, (3, 1, 1), 5, (1, 1, 0, 0, 0, 0), "exact", 1),
    (1, (3, 1, 1), 5, (2, 2, 0, 0, 0, 0), "llf", 8),
    (2, (3, 2, 1), 4, (0,) * 6, "hll", 7),
    (2, (3, 2, 1), 4, (0, 0, 1, 1, 0, 0), "llf", 3),
    (2, (2, 2, 1), 4, (2, 2, 0, 0, 0, 0), "acoustic", 1),
    (3, (3, 2, 1), 3, (0,) * 6, "hllc", 1),
    (3, (1, 2, 3), 3, (2, 2, 0, 0, 0, 0), "exact", 2),
    (3, (3, 2, 1), 3, (1, 1, 0, 0, 0, 0), "acoustic", 3),
    (3, (2, 2, 2), 3, (0, 0, 0, 0, 1, 1), "hll", 8),
    (3, (3, 2, 1), 3, (0,) * 6, "llf", 7),
]


@pytest.mark.parametrize("ndim,coarse,level,bound,riemann,slope_type", ROWS)
def test_level_steps_with_pressure_fix_equal_oracle(gpu, ndim, coarse, level, bound, riemann, slope_type):
    """rgpu_level_steps with pressure_fix: per step set_unew's divu / enew, the plain PFIX sweep, set_uold's pdV source and energy
    switch and the Courant scan of the switched state; the dt history, the state and divu / enew of the last step equal the
    oracle's set_unew + godunov_fine + set_uold under orc_set_pressure_fix; the 3-D level binds the round-1 kernel"""
    c = _case(ndim, coarse, level, bound, riemann, slope_type)
    got = _gpu(c, 3)
    assert got[4].dense == 1 and got[4].sweep_variant == 0
    _check_oracle(c, got, _oracle(c, 3))


@pytest.mark.parametrize("ndim,coarse,level,bound,riemann,slope_type", [ROWS[0], ROWS[4], ROWS[7], ROWS[8]])
def test_per_level_calls_equal_oracle_and_level_steps(gpu, ndim, coarse, level, bound, riemann, slope_type):
    """courant_fine, set_unew, godunov_fine_dev, set_uold, make_virtual_fine, make_boundary_hydro in amr_step order equal the
    oracle and rgpu_level_steps bit for bit (state, divu, enew, dt)"""
    c = _case(ndim, coarse, level, bound, riemann, slope_type)
    split, fused = _gpu(c, 3, "split"), _gpu(c, 3, "fused")
    _check_oracle(c, split, _oracle(c, 3))
    for x, y in zip(split[:4], fused[:4]):
        assert np.array_equal(x, y)


@pytest.mark.parametrize("ndim,coarse,level,bound,riemann,slope_type", [ROWS[0], ROWS[2], ROWS[3], ROWS[5], ROWS[6], ROWS[8]])
def test_same_box_through_amr_mode_equals_the_dense_path(gpu, ndim, coarse, level, bound, riemann, slope_type):
    """the same levelmin=levelmax box through AMR mode (the PFIX AMR variant in 3-D, the oct-batch kernel in 1-D / 2-D, the list
    passes of set_unew / set_uold) gives the state, divu, enew and dt of the new path, bit for bit"""
    c = _case(ndim, coarse, level, bound, riemann, slope_type)
    amr, dense = _gpu(c, 3, "amr"), _gpu(c, 3, "fused")
    assert amr[4].dense == (1 if ndim == 3 else 0)
    idx = c.active_cells()
    assert np.array_equal(amr[1], dense[1])
    assert np.array_equal(amr[0][:, idx], dense[0][:, idx])
    assert np.array_equal(amr[2][idx], dense[2][idx]) and np.array_equal(amr[3][idx], dense[3][idx])


def test_fast_flag_and_tile_override_keep_the_strict_bits(gpu, monkeypatch):
    """fast = 1 and RGPU_BY3 / RGPU_SWEEP select kernels of the plain sweep; with pressure_fix the level binds the round-1 PFIX
    kernel (sweep_variant 0) and gives the strict bits"""
    c = _case(*ROWS[6])
    strict = _gpu(c, 3)
    monkeypatch.setenv("RGPU_BY3", "16")
    monkeypatch.setenv("RGPU_SWEEP", "31201")
    fast = _gpu(c, 3, fast=True)
    assert fast[4].sweep_variant == 0
    for x, y in zip(strict[:4], fast[:4]):
        assert np.array_equal(x, y)


def _cold_hypersonic(ndim, ext, seed=3):
    """a shear flow at |v| ~ 3 on a sound speed ~ 0.005 (Mach ~600), density contrasts of 1.5; dense [ndim+2][nz][ny][nx]"""
    rng = np.random.default_rng(seed)
    shape = (ext[2], ext[1], ext[0])
    Z, Y, X = np.meshgrid(*[np.arange(n) + 0.5 for n in shape], indexing="ij")
    axes = [X / ext[0], Y / ext[1], Z / ext[2]]
    rho = 1.0 + 0.5 * rng.random(shape)
    u = np.zeros((ndim + 2,) + shape)
    u[0] = rho
    ekin = 0.0
    for d in range(ndim):
        v = 3.0 * np.sin(2 * np.pi * axes[(d + 1) % ndim]) + 0.3 * rng.standard_normal(shape)
        u[1 + d] = rho * v
        ekin = ekin + 0.5 * rho * v ** 2
    u[ndim + 1] = 1e-5 * (1 + rng.random(shape)) / 0.4 + ekin
    return u


@pytest.mark.parametrize("kind,ndim,coarse,level,riemann", [("floors", 3, (2, 2, 1), 3, "hllc"), ("floors", 2, (2, 2, 1), 4, "llf"),
                                                            ("hypersonic", 3, (2, 2, 1), 3, "hll"),
                                                            ("hypersonic", 1, (4, 1, 1), 5, "hllc")])
def test_switch_fires_at_the_floors_and_in_cold_hypersonic_flow(gpu, kind, ndim, coarse, level, riemann):
    """the regime pressure_fix exists for: every cell a floor_state cell under the raised floors, or a cold hypersonic shear flow.
    rgpu_level_steps equals the oracle, and the energy switch fired (the state differs from the oracle's run without
    pressure_fix in the total energy of some cells, and only there)"""
    if kind == "floors":
        c = _case(ndim, coarse, level, (0,) * 6, riemann, 1, seed=6, floors="raised")
    else:
        ext = tuple(coarse[d] << level if d < ndim else 1 for d in range(3))
        c = _case(ndim, coarse, level, (0,) * 6, riemann, 1, dense=_cold_hypersonic(ndim, ext))
    got = _gpu(c, 2)
    want = _oracle(c, 2)
    _check_oracle(c, got, want)
    ref_plain, _ = c.oracle_steps(2, nthreads=1)
    ref_plain = ref_plain.reshape(c.nvar, -1)
    idx = c.active_cells()
    # after the first step the two runs differ everywhere downstream of a switched cell; the first step pins the switch itself
    one, _ = c.oracle_steps(1, nthreads=1)
    with Sources(c.mesh.s.ncell, 0.5):
        one_pfix, _ = c.oracle_steps(1, nthreads=1)
    one, one_pfix = one.reshape(c.nvar, -1)[:, idx], one_pfix.reshape(c.nvar, -1)[:, idx]
    assert np.array_equal(one[:-1], one_pfix[:-1])
    fired = one[-1] != one_pfix[-1]
    assert 0 < fired.sum() < fired.size, (int(fired.sum()), fired.size)
    assert not np.array_equal(ref_plain[:, idx], got[0][:, idx])


def test_sweep_without_set_unew_and_host_array_call_are_refused(gpu):
    """godunov_fine_dev sweeps only divu / enew that set_unew initialised since the last sweep (RGPU_EINVAL otherwise), and the
    host-array rgpu_godunov_fine keeps refusing pressure_fix (divu / enew have no host arguments), outside and inside AMR mode"""
    from ramses_b200 import lib
    from ramses_b200.hydro import HydroGPU
    c = _case(*ROWS[6])
    for amr_mode in (False, True):
        a = c.amr_commons()
        a.pressure_fix, a.beta_fix = True, 0.5
        a.dtnew[c.level] = 1e-3
        h = HydroGPU(a, amr_mode=amr_mode)
        try:
            for l in (range(1, c.level + 1) if amr_mode else [c.level]):
                h.bind_level(l)
            h.upload_state(0 if amr_mode else c.level)
            if not amr_mode:
                with pytest.raises(lib.RgpuError) as e:
                    h.godunov_fine_dev(c.level)
                assert e.value.code == -1
                h.set_unew(c.level)
                h.godunov_fine_dev(c.level)
                with pytest.raises(lib.RgpuError) as e:       # divu / enew already hold this sweep's fluxes
                    h.godunov_fine_dev(c.level)
                assert e.value.code == -1
                h.set_uold(c.level)
                with pytest.raises(lib.RgpuError) as e:
                    h.godunov_fine_dev(c.level)
                assert e.value.code == -1
            with pytest.raises(lib.RgpuError) as e:
                h.godunov_fine(c.level)
            assert e.value.code == -3
        finally:
            h.finalize()


@pytest.mark.parametrize("level,overlap", [(5, "0"), (7, "1")], ids=["32^3-serial", "128^3-overlap"])
def test_multi_gpu_pressure_fix_matches_single_gpu(gpu, level, overlap):
    """rgpu_level_steps with pressure_fix on 2+ GPUs (32^3 per rank with the serial exchange, 128^3 per rank with the exchange
    overlapping the interior of the next sweep) equals one GPU in the dt history, the state, divu and enew, bit for bit
    (tests/mgpu_pfix_check.py)"""
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    n = 2 if n < 4 else (4 if n < 8 else 8)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", str(29671 + level), os.path.join(root, "tests", "mgpu_pfix_check.py"), str(level), "4", "hllc", overlap]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "state identical=True" in r.stdout and "divu/enew identical=True" in r.stdout
