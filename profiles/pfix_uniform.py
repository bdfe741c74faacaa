"""Cost of pressure_fix on a levelmin=levelmax box, one GPU, CUDA events around the timed calls after a warm-up.

A 256^3 periodic box (level 8, hllc, minmod, the Sedov blast of bench.py) timed three ways:
  (a) rgpu_level_steps without pressure_fix on the round-1 kernel (RGPU_SWEEP=old: the kernel the PFIX form extends);
  (b) rgpu_level_steps with pressure_fix: per step set_unew's divu / enew, the plain PFIX sweep, the pdV and energy-switch passes
      and a Courant scan of the switched state;
  (c) the same box with pressure_fix through AMR mode (rgpu_amr_steps, levelmin = levelmax): the PFIX AMR variant with divu /
      enew gathered and scattered per call and the set_unew / set_uold list kernels over the tree.
The three configurations run alternately, twice each, in the same process, every one from the same initial state for the same
number of steps; (b) and (c) must give identical states, divu, enew and dt histories.

Prints one JSON line (ms per step and cell updates per second) with the card name and power limit read in the same run.
Usage: python profiles/pfix_uniform.py [steps] [warmup]"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LEVEL = 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                       text=True)
    name, plim = [s.strip() for s in q.stdout.strip().split(",")[:2]] if q.returncode == 0 else ("unknown", "unknown")
    return name, plim


def tree(pfix):
    from bench import sedov_ic
    from ramses_b200.tree import build_uniform_tree, fill_state
    a = build_uniform_tree(3, LEVEL, order="creation", boxlen=0.5)
    a.gamma, a.courant_factor, a.slope_type, a.riemann = 1.4, 0.8, 1, "hllc"
    a.pressure_fix, a.beta_fix = pfix, 0.5
    fill_state(a, LEVEL, sedov_ic(0.5, 1, LEVEL))
    return a


def run(kind, steps, warmup):
    """kind 'a', 'b' or 'c' (module docstring); returns (ms per step, (state, divu, enew, dts) for b and c)"""
    from ramses_b200.hydro import HydroGPU
    if kind == "a":
        os.environ["RGPU_SWEEP"] = "old"
    a = tree(kind != "a")
    h = HydroGPU(a, device=0, amr_mode=(kind == "c"))
    try:
        if kind == "c":
            for l in range(1, LEVEL + 1):
                h.bind_level(l)
            h.upload_state(0)
            nsub = [1] * (LEVEL + 1) + [2] * 64
            dts = list(h.amr_steps(LEVEL, nsub, warmup))
            dts += list(h.amr_steps(LEVEL, nsub, steps))
        else:
            h.bind_level(LEVEL)
            h.upload_state(LEVEL)
            d0, _ = h.level_steps(LEVEL, warmup)
            d1, _ = h.level_steps(LEVEL, steps)
            dts = list(d0) + list(d1)
        ms = h.level_info(LEVEL).last_steps_ms / steps
        out = None
        if kind != "a":
            h.download_state(0 if kind == "c" else LEVEL)
            divu, enew = h.download_pressure_fix()
            ig = a.active[LEVEL].astype(np.int64)
            cc = np.concatenate([a.ncoarse + ind * a.ngridmax + ig - 1 for ind in range(8)])
            out = (a.uold[:, cc].copy(), divu[cc], enew[cc], np.array(dts))
    finally:
        h.finalize()
        os.environ.pop("RGPU_SWEEP", None)
    return ms, out


def main():
    from ramses_b200 import lib
    lib.load()
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    warmup = int(sys.argv[2]) if len(sys.argv) > 2 else 2
    name, plim = card()
    cells = float(8 ** LEVEL)
    ms = {"a": [], "b": [], "c": []}
    outs = []
    for _ in range(2):                         # alternate the three configurations
        for k in ("a", "b", "c"):
            t, o = run(k, steps, warmup)
            ms[k].append(t)
            if o is not None:
                outs.append(o)
    same = all(all(np.array_equal(x, y) for x, y in zip(o, outs[0])) for o in outs)
    res = {k: dict(ms_per_step=v, cell_updates_per_s=cells / (min(v) * 1e-3)) for k, v in ms.items()}
    out = dict(gpu=name, power_limit=plim, box="256^3 hllc sedov, level 8", steps=steps, warmup=warmup,
               a_level_steps_round1=res["a"], b_level_steps_pfix=res["b"], c_amr_steps_pfix=res["c"],
               b_over_c_speedup=min(ms["c"]) / min(ms["b"]), pfix_cost_b_over_a=min(ms["b"]) / min(ms["a"]),
               b_c_identical=bool(same))
    print(json.dumps(out))
    if not same:
        raise SystemExit("the level-steps and AMR-mode runs with pressure_fix differ")


if __name__ == "__main__":
    main()
