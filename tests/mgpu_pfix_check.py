#!/usr/bin/env python
"""Multi-GPU parity check of pressure_fix outside AMR mode, run under torchrun:
    torchrun --nproc-per-node N tests/mgpu_pfix_check.py [level] [steps] [riemann] [overlap]

Every rank owns one coarse cell of an (nx,ny,nz) periodic coarse grid refined to `level` (level 5: 32^3 cells per rank, level 7:
128^3); K fused level steps with pressure_fix run with the NCCL ghost-oct exchange, serial (overlap 0) or overlapped with the
interior of the next sweep (overlap 1, RGPU_OVERLAP).  The flow is cold and hypersonic in part of the box, so the energy switch
fires there.  Rank 0 then repeats the same global problem on one GPU and compares cell by cell: the dt history, the state, divu
and enew of the decomposed run must be bit-identical."""
import ctypes as C
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from mgpu_check import keys_and_state                  # noqa: E402
from ramses_b200 import lib as _l                      # noqa: E402
from ramses_b200.hydro import HydroGPU                 # noqa: E402
from ramses_b200.tree import build_uniform_tree, coarse_dims_for_ranks, fill_state  # noqa: E402


def cold_state_fn(coarse):
    """smooth periodic flow at speeds ~0.3 whose pressure drops to 1e-5 over part of the box (Mach ~100 there)"""
    def fn(x, y, z):
        tw = 2 * np.pi
        xs, ys, zs = x / coarse[0], y / coarse[1], z / coarse[2]
        rho = 1 + 0.2 * np.sin(tw * xs) * np.cos(tw * ys)
        vx, vy, vz = 0.3 * np.sin(tw * ys), 0.3 * np.sin(tw * zs), 0.3 * np.sin(tw * xs)
        p = 1e-5 + 0.1 * np.maximum(0.0, np.cos(tw * (xs + ys + zs))) ** 2
        u = np.zeros((5, len(x)))
        u[0] = rho
        u[1], u[2], u[3] = rho * vx, rho * vy, rho * vz
        u[4] = p / 0.4 + 0.5 * rho * (vx ** 2 + vy ** 2 + vz ** 2)
        return u
    return fn


def pfix_at(a, l, divu, enew):
    """divu, enew of the active cells in the order of keys_and_state"""
    ig = a.active[l].astype(np.int64)
    cc = np.concatenate([a.ncoarse + ind * a.ngridmax + ig - 1 for ind in range(8)])
    return np.stack([divu[cc], enew[cc]])


def main():
    level = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 4
    riemann = sys.argv[3] if len(sys.argv) > 3 else "hllc"
    os.environ["RGPU_OVERLAP"] = sys.argv[4] if len(sys.argv) > 4 else "0"
    rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(lr)
    dist.init_process_group("nccl", device_id=torch.device("cuda", lr))
    coarse = coarse_dims_for_ranks(3, world)

    def configure(t):
        t.riemann, t.slope_type, t.courant_factor = riemann, 1, 0.8
        t.pressure_fix, t.beta_fix = True, 0.5
        fill_state(t, level, cold_state_fn(coarse))
    a = build_uniform_tree(3, level, coarse=coarse, myid=rank + 1, ncpu=world, order="random", seed=rank + 5)
    configure(a)
    h = HydroGPU(a, device=lr)
    uid = torch.zeros(128, dtype=torch.uint8, device="cuda")
    if rank == 0:
        buf = (C.c_ubyte * 128)()
        _l.check(h.L.rgpu_comm_unique_id(buf))
        uid = torch.tensor(list(buf), dtype=torch.uint8, device="cuda")
    dist.broadcast(uid, 0)
    buf = (C.c_ubyte * 128)(*uid.cpu().tolist())
    _l.check(h.L.rgpu_comm_init(world, rank, buf))
    h.bind_level(level)
    h.upload_state(level)
    dts, _ = h.level_steps(level, steps)
    h.download_state(level)
    divu, enew = h.download_pressure_fix()
    h.finalize()
    k, u = keys_and_state(a, level)
    u = np.concatenate([u, pfix_at(a, level, divu, enew)])
    kt = torch.from_numpy(k).cuda()
    ut = torch.from_numpy(np.ascontiguousarray(u)).cuda()
    ks = [torch.zeros_like(kt) for _ in range(world)]
    us = [torch.zeros_like(ut) for _ in range(world)]
    dist.all_gather(ks, kt)
    dist.all_gather(us, ut)
    ok = True
    if rank == 0:
        kk = torch.cat(ks).cpu().numpy()
        uu = torch.cat(us, dim=1).cpu().numpy()
        order = np.argsort(kk)
        kk, uu = kk[order], uu[:, order]
        os.environ["RGPU_OVERLAP"] = "0"
        g = build_uniform_tree(3, level, coarse=coarse, myid=1, ncpu=1, order="creation")
        configure(g)
        hg = HydroGPU(g, device=lr)
        hg.bind_level(level)
        hg.upload_state(level)
        dts1, _ = hg.level_steps(level, steps)
        hg.download_state(level)
        divu1, enew1 = hg.download_pressure_fix()
        hg.finalize()
        k1, u1 = keys_and_state(g, level)
        u1 = np.concatenate([u1, pfix_at(g, level, divu1, enew1)])
        o1 = np.argsort(k1)
        k1, u1 = k1[o1], u1[:, o1]
        same_dt = np.array_equal(dts, dts1)
        same_u = np.array_equal(kk, k1) and np.array_equal(uu[:5], u1[:5])
        same_p = np.array_equal(uu[5:], u1[5:])
        moved = bool(np.abs(u1[5]).max() > 0)
        print(f"mgpu_pfix_check world={world} level={level} steps={steps} riemann={riemann} overlap={sys.argv[4] if len(sys.argv) > 4 else '0'}: "
              f"dt identical={same_dt} state identical={same_u} divu/enew identical={same_p} divu moved={moved}")
        ok = same_dt and same_u and same_p and moved
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.broadcast(flag, 0)
    dist.destroy_process_group()
    sys.exit(0 if flag.item() == 1 else 1)


if __name__ == "__main__":
    main()
