"""Cost of poisson in the dense sweep, one GPU, CUDA events around the timed calls after a warm-up.

(a) levelmin=levelmax, 3-D 256^3 hllc: rgpu_level_steps with a fixed, non-uniform acceleration f (GRAV instantiation of the
    round-1 kernel, source term and gravity Courant term fused) against the same run without gravity on the round-1 kernel
    (RGPU_SWEEP=old) -- the price of gravity on one kernel.
(b) AMR mode, the config-4 nested tree (build_nested_tree, levels 7-10, hllc, interpol_type=2) with poisson through
    rgpu_amr_steps, dense base box and patches (RGPU_AMR_DENSE=1) against the oct-batch kernel (RGPU_AMR_DENSE=0); the two
    final states must be bit-identical.

Prints one JSON line with the card name and power limit read in the same run.  Usage: python profiles/gravity_dense.py"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                       text=True)
    name, plim = [s.strip() for s in q.stdout.strip().split(",")[:2]] if q.returncode == 0 else ("unknown", "unknown")
    return name, plim


def force(ndim, ncell, seed=5):
    rng = np.random.default_rng(seed)
    return np.ascontiguousarray(5.0 * (np.array([0.8, -0.5, 0.3])[:ndim, None] + 0.4 * rng.standard_normal((ndim, ncell))))


def uniform(gravity, steps, warmup):
    from ramses_b200.hydro import HydroGPU
    from ramses_b200.tree import build_uniform_tree, fill_state
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from mgpu_check import state_fn
    level = 8
    os.environ["RGPU_SWEEP"] = "old"           # the round-1 kernel for both runs
    a = build_uniform_tree(3, level, order="lattice")
    a.riemann, a.slope_type, a.courant_factor = "hllc", 1, 0.8
    a.poisson = gravity
    fill_state(a, level, state_fn((1, 1, 1)))
    h = HydroGPU(a, device=0)
    h.bind_level(level)
    assert h.level_info(level).sweep_variant == 0
    h.upload_state(level)
    if gravity:
        h.upload_force(force(3, a.ncell))
    h.level_steps(level, warmup)
    h.level_steps(level, steps)
    ms = h.level_info(level).last_steps_ms
    h.finalize()
    del os.environ["RGPU_SWEEP"]
    ncell = (1 << level) ** 3
    return dict(ms_per_step=ms / steps, cell_updates_per_s=ncell * steps / (ms * 1e-3))


def nested(dense, steps, warmup):
    from ramses_b200.hydro import HydroGPU
    from ramses_b200.tree import build_nested_tree, cell_centers
    os.environ["RGPU_AMR_DENSE"] = "1" if dense else "0"
    levelmin, levelmax, gamma = 7, 10, 1.4
    a = build_nested_tree(levelmin, levelmax, half_width=16, boxlen=1.0)
    a.gamma, a.courant_factor, a.slope_type, a.riemann = gamma, 0.8, 1, "hllc"
    a.poisson = True
    dxf = 0.5 ** levelmax
    for l in range(levelmin, levelmax + 1):    # the config-4 Sedov blast at the box centre
        ig, cc = cell_centers(a, l)
        for ind in range(8):
            x, y, z = cc[ind][:, 0] - 0.5, cc[ind][:, 1] - 0.5, cc[ind][:, 2] - 0.5
            r = np.maximum(1 - np.abs(x) / dxf, 0) * np.maximum(1 - np.abs(y) / dxf, 0) * np.maximum(1 - np.abs(z) / dxf, 0)
            u = np.zeros((5, len(x)))
            u[0] = 1.0
            u[4] = (1e-5 + 0.4 * r / dxf ** 3) / (gamma - 1.0)
            a.uold[:, a.ncoarse + ind * a.ngridmax + ig - 1] = u
    h = HydroGPU(a, device=0, amr_mode=True, interpol_type=2)
    for l in range(1, levelmax + 1):
        h.bind_level(l)
    kernels = [h.level_info(l).dense for l in range(levelmin, levelmax + 1)]
    h.upload_state(0)
    h.upload_force(force(3, a.ncell))
    for l in range(levelmax - 1, 0, -1):
        h.upload_fine(l)
    nsub = [1] * levelmin + [2] * 64
    h.amr_steps(levelmin, nsub, warmup)
    h.amr_steps(levelmin, nsub, steps)
    ms = h.level_info(levelmin).last_steps_ms
    h.download_state(0)
    h.finalize()
    del os.environ["RGPU_AMR_DENSE"]
    return dict(ms_per_coarse_step=ms / steps, dense_levels=kernels), a.uold.copy()


def main():
    from ramses_b200 import lib
    lib.load()
    name, plim = card()
    out = dict(gpu=name, power_limit=plim)
    out["a_uniform_256_hllc"] = dict(gravity=uniform(True, 10, 3), no_gravity=uniform(False, 10, 3))
    g, n = out["a_uniform_256_hllc"]["gravity"], out["a_uniform_256_hllc"]["no_gravity"]
    out["a_uniform_256_hllc"]["gravity_cost"] = g["ms_per_step"] / n["ms_per_step"]
    rd, ud = nested(True, 4, 2)
    ro, uo = nested(False, 4, 2)
    out["b_nested_7_10_hllc_poisson"] = dict(dense=rd, octbatch=ro, speedup=ro["ms_per_coarse_step"] / rd["ms_per_coarse_step"],
                                             bit_identical=bool(np.array_equal(ud, uo)))
    print(json.dumps(out))
    if not out["b_nested_7_10_hllc_poisson"]["bit_identical"]:
        raise SystemExit("dense and oct-batch runs differ")


if __name__ == "__main__":
    main()
