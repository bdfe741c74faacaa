"""Cost of pressure_fix on the dense sweep, one GPU, CUDA events around the timed calls after a warm-up.

AMR mode, the config-4 nested tree (build_nested_tree, levels 7-10, hllc, interpol_type=2) with pressure_fix through
rgpu_amr_steps: dense base box and patches on the PFIX AMR variant (RGPU_AMR_DENSE=1) against the oct-batch kernel on every
level (RGPU_AMR_DENSE=0).  The two configurations are run alternately, twice each, in the same process; the final state, divu
and enew of every run must be bit-identical.

Prints one JSON line with the card name and power limit read in the same run.  Usage: python profiles/pfix_dense.py"""
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


def nested(dense, steps, warmup):
    from ramses_b200.hydro import HydroGPU
    from ramses_b200.tree import build_nested_tree, cell_centers
    os.environ["RGPU_AMR_DENSE"] = "1" if dense else "0"
    levelmin, levelmax, gamma = 7, 10, 1.4
    a = build_nested_tree(levelmin, levelmax, half_width=16, boxlen=1.0)
    a.gamma, a.courant_factor, a.slope_type, a.riemann = gamma, 0.8, 1, "hllc"
    a.pressure_fix, a.beta_fix = True, 0.5
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
    for l in range(levelmax - 1, 0, -1):
        h.upload_fine(l)
    nsub = [1] * levelmin + [2] * 64
    h.amr_steps(levelmin, nsub, warmup)
    h.amr_steps(levelmin, nsub, steps)
    ms = h.level_info(levelmin).last_steps_ms
    h.download_state(0)
    divu, enew = h.download_pressure_fix()
    h.finalize()
    del os.environ["RGPU_AMR_DENSE"]
    return dict(ms_per_coarse_step=ms / steps, dense_levels=kernels), (a.uold.copy(), divu, enew)


def main():
    from ramses_b200 import lib
    lib.load()
    name, plim = card()
    out = dict(gpu=name, power_limit=plim)
    steps, warmup = 4, 2
    runs = {"dense": [], "octbatch": []}
    for _ in range(2):                         # alternate the two configurations
        runs["dense"].append(nested(True, steps, warmup))
        runs["octbatch"].append(nested(False, steps, warmup))
    ref = runs["dense"][0][1]
    same = all(all(np.array_equal(x, y) for x, y in zip(r[1], ref)) for rs in runs.values() for r in rs)
    res = {k: dict(ms_per_coarse_step=[r[0]["ms_per_coarse_step"] for r in rs], dense_levels=rs[0][0]["dense_levels"])
           for k, rs in runs.items()}
    res["speedup"] = min(res["octbatch"]["ms_per_coarse_step"]) / min(res["dense"]["ms_per_coarse_step"])
    res["bit_identical"] = bool(same)
    out["nested_7_10_hllc_pressure_fix"] = res
    print(json.dumps(out))
    if not same:
        raise SystemExit("dense and oct-batch runs differ")


if __name__ == "__main__":
    main()
