"""ORACLE (test infrastructure): the NDIM=1 ideal-MHD build of the AMR driver, on top of oracle/amr.py.

`MhdAmrRun` reuses the mesh-adaptation control flow of `AmrRun` (init_refine, flag_fine, refine_fine, amr_step with sub-cycling,
newdt_fine, update_time: amr/*.f90 are shared by the hydro and the MHD builds) and swaps every floating-point routine for its
MHD version restated in oracle/ramses_oracle_mhd.c: godfine1 (mhd/godunov_fine.f90:538) with trace1d, interpol_hydro +
interpol_mag (mhd/interpol_hydro.f90:612,990), upload_fine (:5,233), courant_fine/cmpdt, make_boundary_hydro, hydro_refine
(mhd/godunov_utils.f90:113), condinit/region_condinit (mhd/condinit.f90, mhd/init_flow_fine.f90:465), the output fields of
mhd/output_hydro.f90:60-175.  It exists to reproduce tests/mhd/imhd-tube/imhd-tube-ref.dat (tests/test_oracle_golden.py).
"""
import ctypes as C
import math

import numpy as np

from . import orc
from .amr import AmrRun, FastAmrRun

NV, NVS = 8, 11


class MhdAmrRun(AmrRun):
    def __init__(self, levelmin, levelmax, bound_type, boxlen, nsubcycle, riemann="hlld", slope_type=1, gamma=1.4,
                 courant_factor=0.8, err_grad_d=-1.0, err_grad_u=-1.0, err_grad_p=-1.0, err_grad_A=-1.0, err_grad_B=-1.0,
                 err_grad_C=-1.0, err_grad_B2=-1.0, interpol_type=1, regions=(), tout=(), nexpand=1, ngridmax=2000, nvector=32,
                 smallr=1e-10, smallc=1e-10):
        super().__init__(1, levelmin, levelmax, bound_type, boxlen, nsubcycle, nexpand=nexpand, ngridmax=ngridmax,
                         riemann="llf", slope_type=slope_type, gamma=gamma, courant_factor=courant_factor,
                         err_grad_d=err_grad_d, err_grad_u=err_grad_u, err_grad_p=err_grad_p, interpol_type=interpol_type,
                         interpol_var=0, regions=regions, tout=tout, nvector=nvector)
        self.pm = orc.make_mhd_params(slope_type=slope_type, riemann=riemann, riemann2d="llf", gamma=gamma,
                                      courant_factor=courant_factor, boxlen=boxlen, smallr=smallr, smallc=smallc)
        self.p.smallr, self.p.smallc = smallr, smallc      # the driver's own floors (dtnew = boxlen / smallc, region fill)
        self.nvar = NVS                                   # stored variables (nvar+3 of the MHD build)
        self.uold = np.zeros(NVS * self.ncell)
        self.unew = np.zeros(NVS * self.ncell)
        self.err_grad_A, self.err_grad_B, self.err_grad_C, self.err_grad_B2 = err_grad_A, err_grad_B, err_grad_C, err_grad_B2
        self.floor_A = self.floor_B = self.floor_C = self.floor_b2 = 1e-10
        L, mp, pp, dp = self.L, C.POINTER(orc.MeshS), C.POINTER(orc.MhdParams), C.POINTER(C.c_double)
        L.orc_mhd1_interpol_cell.argtypes = [mp, C.c_int, C.c_int, dp, dp]
        L.orc_mhd1_godunov_fine.argtypes = [pp, mp, C.c_int, C.c_int, C.c_int, C.c_double, dp, dp]
        L.orc_mhdn_set_unew.argtypes = [mp, C.c_int, dp, dp]
        L.orc_mhdn_set_uold.argtypes = [mp, C.c_int, dp, dp]
        L.orc_mhd1_courant_fine.restype = C.c_double
        L.orc_mhd1_courant_fine.argtypes = [pp, mp, C.c_int, C.c_double, dp]
        L.orc_mhd1_make_boundary_hydro.argtypes = [pp, mp, C.c_int, dp]
        L.orc_mhd1_upload_fine.argtypes = [pp, mp, C.c_int, dp]

    # ---- floating-point routines -------------------------------------------------------------------------------------
    def c_set_unew(self, l):
        self.L.orc_mhdn_set_unew(self.mp, l, orc.dptr(self.uold), orc.dptr(self.unew))

    def c_godunov_fine(self, l):
        self.L.orc_mhd1_godunov_fine(C.byref(self.pm), self.mp, l, self.levelmin, self.nvector, self.dtnew[l], orc.dptr(self.uold),
                                     orc.dptr(self.unew))

    def c_set_uold(self, l):
        self.L.orc_mhdn_set_uold(self.mp, l, orc.dptr(self.uold), orc.dptr(self.unew))

    def c_interpol_cell(self, c, lnew):
        u2 = np.zeros(2 * NVS)
        self.L.orc_mhd1_interpol_cell(self.mp, c, lnew, orc.dptr(self.uold), orc.dptr(u2))
        return u2

    def make_boundary_hydro(self, l):
        self.L.orc_mhd1_make_boundary_hydro(C.byref(self.pm), self.mp, l, orc.dptr(self.uold))

    def upload_fine(self, l):
        self.L.orc_mhd1_upload_fine(C.byref(self.pm), self.mp, l, orc.dptr(self.uold))

    def newdt_fine(self, l):
        self.dtold[l] = self.dtnew[l]
        self.dtnew[l] = self.p.boxlen / self.p.smallc
        self.dtnew[l] = self.L.orc_mhd1_courant_fine(C.byref(self.pm), self.mp, l, self.dtnew[l], orc.dptr(self.uold))

    # ---- initial conditions: mhd/init_flow_fine.f90:465 region_condinit + mhd/condinit.f90 ------------------------------------
    def init_flow_fine(self, l):
        if self.numbtot(l) == 0:
            return
        p = self.p
        U = self.uold.reshape(NVS, self.ncell)
        nx_loc = self.m.icoarse_max - self.m.icoarse_min + 1
        scale = p.boxlen / nx_loc
        dx = 0.5 ** l
        for ig in self.active[l]:
            for ind in range(2):
                x = (self.xg[0, ig] + (ind - 0.5) * dx - self.m.icoarse_min) * scale
                q = [p.smallr, 0.0, 0.0, 0.0, p.smallr * p.smallc ** 2 / p.gamma, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0]
                for r in self.regions:
                    if r.get("type", "square") != "square":
                        raise NotImplementedError("point regions")
                    en = float(r.get("exp_region", 2.0))
                    xn = 2.0 * abs(x - r["x_center"]) / r["length_x"]
                    rr = (xn ** en + 0.0 ** en + 0.0 ** en) ** (1.0 / en) if en < 10 else max(xn, 0.0, 0.0)
                    if rr < 1.0:
                        q = [r.get("d", 0.0), r.get("u", 0.0), r.get("v", 0.0), r.get("w", 0.0), r.get("p", 0.0), r.get("A", 0.0),
                             r.get("B", 0.0), r.get("C", 0.0), r.get("A", 0.0), r.get("B", 0.0), r.get("C", 0.0)]
                u = [0.0] * NVS
                u[0] = q[0]
                u[1], u[2], u[3] = q[0] * q[1], q[0] * q[2], q[0] * q[3]
                e = 0.0
                e = e + 0.5 * q[0] * q[1] ** 2
                e = e + 0.5 * q[0] * q[2] ** 2
                e = e + 0.5 * q[0] * q[3] ** 2
                e = e + q[4] / (p.gamma - 1.0)
                e = e + 0.125 * (q[5] + q[8]) ** 2
                e = e + 0.125 * (q[6] + q[9]) ** 2
                e = e + 0.125 * (q[7] + q[10]) ** 2
                u[4] = e
                u[5:8] = q[5:8]
                u[8:11] = q[8:11]
                U[:, self.cell(ind, ig) - 1] = u

    # ---- refinement criteria: mhd/godunov_utils.f90:113 hydro_refine ------------------------------------------------------
    def hydro_refine_ok(self, ug, um, ud):
        p = self.p
        prim, emag = [], []
        for u in (ug, um, ud):
            u = list(u)
            u[0] = max(u[0], p.smallr)
            for d in range(3):
                u[d + 1] = u[d + 1] / u[0]
            ek = 0.0
            for d in range(3):
                ek = ek + 0.5 * u[0] * u[d + 1] ** 2
            em = 0.0
            for d in range(3):
                em = em + 0.5 * (0.5 * (u[5 + d] + u[NV + d])) ** 2
            u[4] = (p.gamma - 1.0) * (u[4] - ek - em)
            prim.append(u); emag.append(em)
        g, m_, d_ = prim
        ok = False
        if self.err_grad_d >= 0.0:
            err = 2.0 * max(abs((d_[0] - m_[0]) / (d_[0] + m_[0] + self.floor_d)), abs((m_[0] - g[0]) / (m_[0] + g[0] + self.floor_d)))
            ok = ok or err > self.err_grad_d
        if self.err_grad_p >= 0.0:
            err = 2.0 * max(abs((d_[4] - m_[4]) / (d_[4] + m_[4] + self.floor_p)), abs((m_[4] - g[4]) / (m_[4] + g[4] + self.floor_p)))
            ok = ok or err > self.err_grad_p
        if self.err_grad_B2 >= 0.0:
            pg, pm, pd = emag
            err = 2.0 * max(abs((pd - pm) / (pd + pm + self.floor_b2)), abs((pm - pg) / (pm + pg + self.floor_b2)))
            ok = ok or err > self.err_grad_B2
        for k, (eg, fl) in enumerate(((self.err_grad_A, self.floor_A), (self.err_grad_B, self.floor_B), (self.err_grad_C, self.floor_C))):
            if eg >= 0.0:
                vg, vm, vd = (0.5 * (u[5 + k] + u[NV + k]) for u in (g, m_, d_))
                cg, cm, cd = (math.sqrt(e) for e in emag)
                err = 2.0 * max(abs((vd - vm) / (cd + cm + fl)), abs((vm - vg) / (cm + cg + fl)))
                ok = ok or err > eg
        if self.err_grad_u >= 0.0:
            for d in range(3):
                vg, vm, vd = g[d + 1], m_[d + 1], d_[d + 1]
                cg = math.sqrt(max(p.gamma * g[4] / g[0], self.floor_u ** 2))
                cm = math.sqrt(max(p.gamma * m_[4] / m_[0], self.floor_u ** 2))
                cd = math.sqrt(max(p.gamma * d_[4] / d_[0], self.floor_u ** 2))
                err = 2.0 * max(abs((vd - vm) / (cd + cm + abs(vd) + abs(vm) + self.floor_u)),
                                abs((vm - vg) / (cm + cg + abs(vm) + abs(vg) + self.floor_u)))
                ok = ok or err > self.err_grad_u
        return ok

    def hydro_flag(self, l):
        """hydro/hydro_flag.f90:1 (SOLVERmhd branches)"""
        if l == self.nlevelmax or self.numbtot(l) == 0:
            return
        if all(e == -1.0 for e in (self.err_grad_d, self.err_grad_p, self.err_grad_u, self.err_grad_A, self.err_grad_B,
                                   self.err_grad_C, self.err_grad_B2)):
            return
        super_all = self.err_grad_d, self.err_grad_p, self.err_grad_u
        # AmrRun.hydro_flag returns early when d,p,u criteria are all off; route around it
        if all(e == -1.0 for e in super_all):
            self.err_grad_d = -2.0
            try:
                AmrRun.hydro_flag(self, l)
            finally:
                self.err_grad_d = -1.0
        else:
            AmrRun.hydro_flag(self, l)

    # ---- output: mhd/output_hydro.f90:60-175 -----------------------------------------------------------------------------
    def dump(self):
        U = self.uold.reshape(NVS, self.ncell)
        p = self.p
        nx_loc = self.m.icoarse_max - self.m.icoarse_min + 1
        scale = p.boxlen / nx_loc
        rows = []
        for l in range(1, self.nlevelmax + 1):
            dx = 0.5 ** l
            for ig in self.active[l]:
                for ind in range(2):
                    c = self.cell(ind, ig)
                    if self.son[c] != 0:
                        continue
                    u_ = U[:, c - 1]
                    d = max(u_[0], p.smallr)
                    vx, vy, vz = u_[1] / d, u_[2] / d, u_[3] / d
                    A, B, Cc = 0.5 * (u_[5] + u_[8]), 0.5 * (u_[6] + u_[9]), 0.5 * (u_[7] + u_[10])
                    e = u_[4] - 0.5 * d * (vx ** 2 + vy ** 2 + vz ** 2) - 0.5 * (A ** 2 + B ** 2 + Cc ** 2)
                    x = (self.xg[0, ig] + (ind - 0.5) * dx - self.m.icoarse_min) * scale
                    rows.append(dict(level=l, x=x, dx=dx * scale, density=u_[0], velocity_x=vx, velocity_y=vy, velocity_z=vz,
                                     pressure=(p.gamma - 1.0) * e, B_x_left=u_[5], B_y_left=u_[6], B_z_left=u_[7],
                                     B_x_right=u_[8], B_y_right=u_[9], B_z_right=u_[10]))
        return rows


def check_sums_mhd(rows, threshold=2.0e-14, norm_min=1.0e-30, min_variance=1.0e-14):
    """tests/visu/visu_ramses.py:495-557 check_solution on the MHD output fields (one dict per leaf cell)."""
    keys = sorted(rows[0].keys())
    data = {k: np.array([r[k] for r in rows], dtype=float) for k in keys}
    norms = {k: 1.0 for k in keys}
    for k in keys:
        if k[-2:] in ("_x", "_y", "_z"):
            raw = k[:-2]
            others = [raw + s for s in ("_x", "_y", "_z") if s != k[-2:]]
            if all(o in data for o in others):
                n = np.sqrt(data[k] ** 2 + data[others[0]] ** 2 + data[others[1]] ** 2)
                norms[k] = np.where(n < norm_min, norm_min, n)
    out = {"ncells": float(len(rows))}
    for k in keys:
        av = np.average(data[k])
        kd = data[k] if av == 0.0 else np.where(np.abs(data[k] - av) / abs(av) < min_variance, av, data[k])
        if k in ("density", "pressure"):
            sol = np.log10(np.abs(kd))
        else:
            sol = np.where(np.abs(kd) < threshold * norms[k], 0.0, np.abs(kd))
        out[k] = math.fsum(sol)
    return out


class MhdAmrRun2D(FastAmrRun):
    """NDIM=2 ideal-MHD build of the AMR driver (periodic box): the control flow of oracle/amr.py (C flag / scan passes) with
    every floating-point routine from the NDIM=2 section of oracle/ramses_oracle_mhd.c -- godfine1 with trace2d, the E_z corner
    EMF, constrained transport, divergence-free prolongation (interpol_mag), EMF refluxing, face-centred restriction.  Exists to
    reproduce tests/mhd/orszag-tang/orszag-tang-ref.dat."""

    NDIM = 2

    def __init__(self, levelmin, levelmax, boxlen, nsubcycle, riemann="hlld", riemann2d="hlld", slope_type=2, gamma=1.4,
                 courant_factor=0.8, err_grad_d=-1.0, err_grad_u=-1.0, err_grad_p=-1.0, err_grad_A=-1.0, err_grad_B=-1.0,
                 err_grad_C=-1.0, err_grad_B2=-1.0, interpol_type=2, tout=(), nexpand=1, ngridmax=100000, nvector=32,
                 ic="orszag_tang", nthreads=None, smallr=1e-10, smallc=1e-10):
        super().__init__(self.NDIM, levelmin, levelmax, (0, 0, 0, 0, 0, 0), boxlen, nsubcycle, nexpand=nexpand, ngridmax=ngridmax,
                         riemann="llf", slope_type=slope_type, gamma=gamma, courant_factor=courant_factor,
                         err_grad_d=err_grad_d, err_grad_u=err_grad_u, err_grad_p=err_grad_p, interpol_type=interpol_type,
                         interpol_var=0, regions=(), tout=tout, nvector=nvector, nthreads=nthreads)
        self.pm = orc.make_mhd_params(slope_type=slope_type, riemann=riemann, riemann2d=riemann2d, gamma=gamma,
                                      courant_factor=courant_factor, boxlen=boxlen, smallr=smallr, smallc=smallc)
        self.p.smallr, self.p.smallc = smallr, smallc
        self.nvar = NVS
        self.uold = np.zeros(NVS * self.ncell)
        self.unew = np.zeros(NVS * self.ncell)
        self.ic = ic
        self.err7 = np.array([err_grad_d, err_grad_p, err_grad_B2, err_grad_A, err_grad_B, err_grad_C, err_grad_u], dtype=float)
        self.flo7 = np.full(7, 1e-10)
        L, mp, pp, dp, ip = self.L, C.POINTER(orc.MeshS), C.POINTER(orc.MhdParams), C.POINTER(C.c_double), C.POINTER(C.c_int)
        L.orc_mhd_set_interpol.argtypes = [C.c_int, C.c_int]
        L.orc_mhd_set_interpol(interpol_type, -1)
        import os
        L.orc_mhd_set_threads.argtypes = [C.c_int]      # flux phase of a batch only; results do not depend on it
        L.orc_mhd_set_threads(int(nthreads) if nthreads else min(8, os.cpu_count() or 1))
        L.orc_mhd2_interpol_cell.argtypes = [mp, C.c_int, C.c_int, dp, dp]
        L.orc_mhd2_godunov_fine.argtypes = [pp, mp, C.c_int, C.c_int, C.c_int, C.c_double, dp, dp]
        L.orc_mhdn_set_unew.argtypes = [mp, C.c_int, dp, dp]
        L.orc_mhdn_set_uold.argtypes = [mp, C.c_int, dp, dp]
        L.orc_mhdn_courant_fine.restype = C.c_double
        L.orc_mhdn_courant_fine.argtypes = [pp, mp, C.c_int, C.c_double, dp]
        L.orc_mhdn_upload_fine.argtypes = [pp, mp, C.c_int, dp]
        L.orc_mhd2_condinit_orszag_tang.argtypes = [pp, mp, C.c_int, dp]
        L.orc_amr_mhd_hydro_flag.argtypes = [pp, mp, C.c_int, dp, ip, dp, dp]
        L.orc_mhd3_interpol_cell.argtypes = [mp, C.c_int, C.c_int, dp, dp]
        L.orc_mhd3_godunov_fine.argtypes = [pp, mp, C.c_int, C.c_int, C.c_int, C.c_double, dp, dp]
        L.orc_mhd3_condinit_orszag_tang.argtypes = [pp, mp, C.c_int, dp]
        self._godunov = L.orc_mhd2_godunov_fine if self.NDIM == 2 else L.orc_mhd3_godunov_fine
        self._interpol = L.orc_mhd2_interpol_cell if self.NDIM == 2 else L.orc_mhd3_interpol_cell
        self._condinit = L.orc_mhd2_condinit_orszag_tang if self.NDIM == 2 else L.orc_mhd3_condinit_orszag_tang

    def c_set_unew(self, l):
        self.L.orc_mhdn_set_unew(self.mp, l, orc.dptr(self.uold), orc.dptr(self.unew))

    def c_godunov_fine(self, l):
        self._godunov(C.byref(self.pm), self.mp, l, self.levelmin, self.nvector, self.dtnew[l], orc.dptr(self.uold),
                                     orc.dptr(self.unew))

    def c_set_uold(self, l):
        self.L.orc_mhdn_set_uold(self.mp, l, orc.dptr(self.uold), orc.dptr(self.unew))

    def c_interpol_cell(self, c, lnew):
        u2 = np.zeros(self.T * NVS)
        self._interpol(self.mp, c, lnew, orc.dptr(self.uold), orc.dptr(u2))
        return u2

    def make_boundary_hydro(self, l):
        assert self.m.nboundary == 0               # periodic box only

    def upload_fine(self, l):
        self.L.orc_mhdn_upload_fine(C.byref(self.pm), self.mp, l, orc.dptr(self.uold))

    def newdt_fine(self, l):
        self.dtold[l] = self.dtnew[l]
        self.dtnew[l] = self.p.boxlen / self.p.smallc
        self.dtnew[l] = self.L.orc_mhdn_courant_fine(C.byref(self.pm), self.mp, l, self.dtnew[l], orc.dptr(self.uold))

    def init_flow_fine(self, l):
        if self.numbtot(l) == 0:
            return
        assert self.ic == "orszag_tang"
        self._condinit(C.byref(self.pm), self.mp, l, orc.dptr(self.uold))

    def hydro_flag(self, l):
        if l == self.nlevelmax or self.numbtot(l) == 0:
            return
        if np.all(self.err7 == -1.0):
            return
        self.L.orc_amr_mhd_hydro_flag(C.byref(self.pm), self.mp, l, orc.dptr(self.uold), self._f1, orc.dptr(self.err7),
                                      orc.dptr(self.flo7))

    def leaf_cells(self):
        """(level, cell index) of every leaf cell, level by level in active-list order"""
        out = []
        for l in range(1, self.nlevelmax + 1):
            act = np.asarray(self.active[l], dtype=np.int64)
            if len(act) == 0:
                continue
            for ind in range(self.T):
                c = self.ncoarse + ind * self.ngridmax + act
                leaf = c[self.son[c] == 0]
                if len(leaf):
                    out.append((l, ind, act[self.son[c] == 0], leaf))
        return out

    def dump(self):
        """mhd/output_hydro.f90:60-175 fields of the leaf cells (vectorised; one dict of arrays)"""
        U = self.uold.reshape(NVS, self.ncell)
        p = self.p
        scale = p.boxlen / (self.m.icoarse_max - self.m.icoarse_min + 1)
        cols = {k: [] for k in ("level", "x", "y", "z", "dx", "density", "velocity_x", "velocity_y", "velocity_z", "pressure",
                                "B_x_left", "B_y_left", "B_z_left", "B_x_right", "B_y_right", "B_z_right")}
        for l, ind, ig, c in self.leaf_cells():
            dx = 0.5 ** l
            u_ = U[:, c - 1]
            d = np.maximum(u_[0], p.smallr)
            vx, vy, vz = u_[1] / d, u_[2] / d, u_[3] / d
            A, B, Cc = 0.5 * (u_[5] + u_[8]), 0.5 * (u_[6] + u_[9]), 0.5 * (u_[7] + u_[10])
            e = u_[4] - 0.5 * d * (vx ** 2 + vy ** 2 + vz ** 2) - 0.5 * (A ** 2 + B ** 2 + Cc ** 2)
            n = len(c)
            cols["level"].append(np.full(n, float(l)))
            cols["x"].append((self.xg[0, ig] + ((ind & 1) - 0.5) * dx - self.m.icoarse_min) * scale)
            cols["y"].append((self.xg[1, ig] + (((ind >> 1) & 1) - 0.5) * dx - self.m.jcoarse_min) * scale)
            cols["z"].append(np.zeros(n) if self.NDIM == 2 else
                             (self.xg[2, ig] + (((ind >> 2) & 1) - 0.5) * dx - self.m.kcoarse_min) * scale)
            cols["dx"].append(np.full(n, dx * scale))
            cols["density"].append(u_[0].copy())
            cols["velocity_x"].append(vx); cols["velocity_y"].append(vy); cols["velocity_z"].append(vz)
            cols["pressure"].append((p.gamma - 1.0) * e)
            for k, name in enumerate(("B_x_left", "B_y_left", "B_z_left", "B_x_right", "B_y_right", "B_z_right")):
                cols[name].append(u_[5 + k].copy())
        return {k: np.concatenate(v) for k, v in cols.items()}

    def divb_max(self):
        """max |div B| * dx over the leaf cells (face fields)"""
        U = self.uold.reshape(NVS, self.ncell)
        worst = 0.0
        for l, ind, ig, c in self.leaf_cells():
            u_ = U[:, c - 1]
            d = (u_[8] - u_[5]) + (u_[9] - u_[6])
            if self.NDIM == 3:
                d = d + (u_[10] - u_[7])
            worst = max(worst, float(np.max(np.abs(d))))
        return worst


class MhdAmrRun3D(MhdAmrRun2D):
    """NDIM=3 ideal-MHD AMR driver on the NDIM=3 AMR routines of oracle/ramses_oracle_mhd.c (the initial condition is the
    z-invariant Orszag-Tang state, so that a run can be compared with the golden-pinned NDIM=2 run)."""
    NDIM = 3

    def __init__(self, *a, courant_ndim=0, **kw):
        super().__init__(*a, **kw)
        self.courant_ndim = courant_ndim            # bit mask of the cmpdt directions (test hook; 0 = all three)

    def newdt_fine(self, l):
        self.L.orc_mhd_set_courant_ndim.argtypes = [C.c_int]
        self.L.orc_mhd_set_courant_ndim(self.courant_ndim)
        try:
            super().newdt_fine(l)
        finally:
            self.L.orc_mhd_set_courant_ndim(0)


def check_sums_cols(data, threshold=2.0e-14, norm_min=1.0e-30, min_variance=1.0e-14):
    """check_solution (tests/visu/visu_ramses.py:495-557) on a dict of column arrays"""
    keys = sorted(data.keys())
    norms = {k: 1.0 for k in keys}
    for k in keys:
        if k[-2:] in ("_x", "_y", "_z"):
            raw = k[:-2]
            others = [raw + s for s in ("_x", "_y", "_z") if s != k[-2:]]
            if all(o in data for o in others):
                n = np.sqrt(data[k] ** 2 + data[others[0]] ** 2 + data[others[1]] ** 2)
                norms[k] = np.where(n < norm_min, norm_min, n)
    out = {"ncells": float(len(data[keys[0]]))}
    for k in keys:
        av = np.average(data[k])
        kd = data[k] if av == 0.0 else np.where(np.abs(data[k] - av) / abs(av) < min_variance, av, data[k])
        if k in ("density", "pressure"):
            sol = np.log10(np.abs(kd))
        else:
            sol = np.where(np.abs(kd) < threshold * norms[k], 0.0, np.abs(kd))
        out[k] = math.fsum(sol)
    return out
