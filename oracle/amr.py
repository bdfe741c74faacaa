"""AMR driver of the CPU ORACLE (test infrastructure, NOT product code).

A restatement of the reference's mesh-adaptation control flow -- init_refine, flag_fine (init_flag / smooth_fine /
hydro_flag / ensure_ref_rules), refine_fine (make_grid_fine / kill_grid), amr_step with sub-cycling -- operating on the
SAME tree arrays (son, father, nbor, xg, active / boundary lists) as oracle/ramses_oracle.c, whose routines do all the
floating-point work (godunov_fine with interpol_hydro ghost prolongation and coarse refluxing, courant_fine, set_unew /
set_uold, upload_fine, make_boundary_hydro, condinit).  Serial (ncpu=1).

Purpose: turn the reference's golden sums of AMR runs (tests/hydro/sod-tube/sod-tube-ref.dat, tolerance 3e-13) into
real pins of the oracle.  Citations are reference file:line.
"""
import ctypes as C
import math

import numpy as np

from . import orc


class AmrRun:
    def __init__(self, ndim, levelmin, levelmax, bound_type, boxlen, nsubcycle, nexpand=1, ngridmax=2000,
                 riemann="hllc", slope_type=2, gamma=1.4, courant_factor=0.8, err_grad_d=-1.0, err_grad_u=-1.0,
                 err_grad_p=-1.0, interpol_type=1, interpol_var=0, regions=(), tout=(), nvector=32,
                 floor_d=1e-10, floor_u=1e-10, floor_p=1e-10, bound_regions=None, coarse=(1, 1, 1), nvar=None):
        """coarse = (nx, ny, nz) domain coarse cells (orc_mesh_new_box); the mesh-adaptation driver itself is exercised with
        one domain coarse cell, several are for trees fabricated elsewhere and loaded into son / father / nbor / lists.
        nvar = ndim+2 (default) + the number of passive scalars; the initial conditions (regions) leave the scalars at 0."""
        self.ndim, self.levelmin, self.nlevelmax = ndim, levelmin, levelmax
        self.T, self.twondim = 1 << ndim, 2 * ndim
        L = self.L = orc.lib()
        L.orc_mesh_new.restype = C.POINTER(orc.MeshS)
        L.orc_mesh_new.argtypes = [C.c_int, C.POINTER(C.c_int), C.c_int, C.c_int]
        L.orc_mesh_new_box.restype = C.POINTER(orc.MeshS)
        L.orc_mesh_new_box.argtypes = [C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int, C.c_int]
        L.orc_mesh_set_list.argtypes = [C.POINTER(orc.MeshS), C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)]
        L.orc_interpol_cell.argtypes = [C.POINTER(orc.Params), C.POINTER(orc.MeshS), C.c_int, C.c_int,
                                        C.POINTER(C.c_double), C.POINTER(C.c_double)]
        L.orc_upload_fine.argtypes = [C.POINTER(orc.Params), C.POINTER(orc.MeshS), C.c_int, C.POINTER(C.c_double)]
        L.orc_set_interpol.argtypes = [C.c_int, C.c_int]
        L.orc_set_interpol(interpol_type, interpol_var)
        bt = (C.c_int * 6)(*bound_type)
        if tuple(coarse) == (1, 1, 1):
            self.mp = L.orc_mesh_new(ndim, bt, ngridmax, levelmax)
        else:
            if any(coarse[d] != 1 for d in range(ndim, 3)) or min(coarse) < 1:
                raise ValueError(f"coarse={coarse} does not fit ndim={ndim}")
            self.mp = L.orc_mesh_new_box(ndim, (C.c_int * 3)(*coarse), bt, ngridmax, levelmax)
        self.m = self.mp.contents
        m = self.m
        self.ncoarse, self.ngridmax, self.ncell = m.ncoarse, m.ngridmax, m.ncell
        self.son = np.ctypeslib.as_array(m.son, shape=(m.ncell + 1,))
        self.father = np.ctypeslib.as_array(m.father, shape=(m.ngridmax + 1,))
        self.nbor = np.ctypeslib.as_array(m.nbor, shape=(2 * ndim, m.ngridmax + 1))
        self.xg = np.ctypeslib.as_array(m.xg, shape=(ndim, m.ngridmax + 1))
        self.p = orc.make_params(ndim=ndim, riemann=riemann, slope_type=slope_type, gamma=gamma,
                                 courant_factor=courant_factor, boxlen=boxlen, nvector=nvector, nvar=nvar)
        self.nvar = self.p.nvar
        self.uold = np.zeros(self.nvar * m.ncell)
        self.unew = np.zeros(self.nvar * m.ncell)
        self.flag1 = np.zeros(m.ncell + 1, dtype=np.int32)
        self.flag2 = np.zeros(m.ncell + 1, dtype=np.int32)
        self.active = {l: [] for l in range(1, levelmax + 2)}
        self.bound = {b: {l: [] for l in range(1, levelmax + 2)} for b in range(m.nboundary)}
        self.free = list(range(1, ngridmax + 1))          # headf free list, init_amr.f90
        self.nvector = nvector
        # level dependent arrays rearranged like amr/read_params.f90:441-470
        ns = list(nsubcycle) + [2] * 64
        self.nsubcycle = {l: (ns[l - levelmin] if l >= levelmin else 1) for l in range(1, levelmax + 2)}
        # a scalar applies to every level; a list is the namelist array (`nexpand=4` in a namelist sets element 1 only,
        # i.e. pass [4]): level l >= levelmin takes element l-levelmin+1, missing elements and coarser levels are 1
        ne = (list(nexpand) + [1] * 64) if hasattr(nexpand, "__len__") else [nexpand] * 64
        self.nexpand = {l: (ne[l - levelmin] if l >= levelmin else 1) for l in range(1, levelmax + 2)}
        # boundary regions in the coarse-cell ranges of hydro/read_hydro_params.f90:316-407.  Default: one region per
        # non-periodic face covering that face only (no edge/corner cells).  bound_regions = [(boundary_type, (imin,
        # imax), (jmin, jmax), (kmin, kmax)), ...] in namelist order restates BOUNDARY_PARAMS blocks whose regions include
        # the corner cells (tests/hydro/implosion/implosion.nml:17-24); ranges are coarse-grid indices incl. boundary cells
        self.bound_regions = None
        if bound_regions is not None:
            assert len(bound_regions) == m.nboundary
            self.bound_regions = [(int(t), tuple(ri), tuple(rj), tuple(rk)) for t, ri, rj, rk in bound_regions]
            for b, reg in enumerate(self.bound_regions):
                m.boundary_type[b] = reg[0]
        self.err_grad_d, self.err_grad_u, self.err_grad_p = err_grad_d, err_grad_u, err_grad_p
        self.floor_d, self.floor_u, self.floor_p = floor_d, floor_u, floor_p
        self.regions = list(regions)
        self.tout = list(tout)
        self.dtnew = {l: 0.0 for l in range(0, levelmax + 2)}
        self.dtold = {l: 0.0 for l in range(0, levelmax + 2)}
        self.t, self.nstep, self.nstep_coarse = 0.0, 0, 0
        self.nstep_coarse_old = 0
        self.init = False
        self.done = False
        self.snapshot = None
        self.iout = 0
        self.log = []
        self.static = False      # static=.true. (amr_parameters): no regridding inside amr_step

    # ------------------------------------------------------------------ helpers
    def cell(self, ind, ig):
        return self.ncoarse + ind * self.ngridmax + ig

    def numbtot(self, l):
        return len(self.active[l]) if l <= self.nlevelmax else 0

    def push_lists(self, l):
        for kind, b, lst in [(0, 0, self.active[l])] + [(1, b, self.bound[b][l]) for b in range(self.m.nboundary)]:
            arr = np.asarray(lst, dtype=np.int32)
            self.L.orc_mesh_set_list(self.mp, kind, b, l, len(lst), orc.iptr(np.ascontiguousarray(arr)) if len(lst) else None)

    def push_all(self):
        for l in range(1, self.nlevelmax + 1):
            self.push_lists(l)

    def nbor_grids(self, ig):
        """getnborgrids amr/nbors_utils.f90:530: [ig, son(nbor(ig,1)), ...]"""
        return [ig] + [int(self.son[self.nbor[j, ig]]) if self.nbor[j, ig] > 0 else 0 for j in range(self.twondim)]

    def nbor_cells(self, igridn, ind):
        """getnborcells amr/nbors_utils.f90:363 (ggg/hhh tables generated): neighbour cell in every direction, 0 if absent."""
        out = []
        for d in range(self.ndim):
            for s in range(2):
                bit = (ind >> d) & 1
                ind2 = ind ^ (1 << d)
                g = igridn[0] if bit != s else igridn[2 * d + s + 1]
                out.append(self.cell(ind2, g) if g > 0 else 0)
        return out

    def all_lists(self, l):
        return [(0, -1, self.active[l])] + [(1, b, self.bound[b][l]) for b in range(self.m.nboundary)]

    # ------------------------------------------------------------------ boundaries of integer maps
    def make_boundary_flag(self, l):
        """amr/physical_boundaries.f90:259"""
        m = self.m
        for b in range(m.nboundary):
            bt = m.boundary_type[b]
            bdir = bt - 10 * (bt // 10)
            inbor = {1: 2, 2: 1, 3: 4, 4: 3, 5: 6, 6: 5}[bdir]
            d = (bdir - 1) // 2
            for ig in self.bound[b][l]:
                gref = int(self.son[self.nbor[inbor - 1, ig]])
                for ind in range(self.T):
                    if bt // 10 == 0:
                        indr = ind ^ (1 << d)                               # reflexive: mirror cell
                    else:
                        indr = (ind & ~(1 << d)) | ((0 if bdir % 2 == 1 else 1) << d)
                    self.flag1[self.cell(ind, ig)] = self.flag1[self.cell(indr, gref)] if gref > 0 else 0

    # ------------------------------------------------------------------ flag_utils.f90
    def flag_coarse(self):
        m = self.m
        self.flag1[0:self.ncoarse + 1] = 0
        for iz in range(m.kcoarse_min, m.kcoarse_max + 1):
            for iy in range(m.jcoarse_min, m.jcoarse_max + 1):
                for ix in range(m.icoarse_min, m.icoarse_max + 1):
                    self.flag1[1 + ix + iy * m.nx + iz * m.nx * m.ny] = 1
        # make_boundary_coarse (physical_boundaries.f90:213): boundary coarse cells mirror the interior flag
        for c in range(1, self.ncoarse + 1):
            self.flag1[c] = 1

    def init_flag(self, l):
        for ig in self.active[l]:
            for ind in range(self.T):
                self.flag1[self.cell(ind, ig)] = 0
        if l >= self.levelmin:
            # test_flag :166-195
            for ind in range(self.T):
                for ig in self.active[l]:
                    c = self.cell(ind, ig)
                    gs = int(self.son[c])
                    ok = False
                    if gs > 0:
                        for inds in range(self.T):
                            cs = self.cell(inds, gs)
                            ok = ok or self.son[cs] > 0 or self.flag1[cs] == 1
                    if ok:
                        self.flag1[c] = 1
        else:
            for ig in self.active[l]:
                for ind in range(self.T):
                    self.flag1[self.cell(ind, ig)] = 1
        self.make_boundary_flag(l)

    def smooth_fine(self, l):
        """:556-632"""
        if l == self.nlevelmax or self.numbtot(l) == 0:
            return
        n_nbor = [1, 2, 2]
        self.flag1[0] = 0
        for ismooth in range(self.ndim):
            for ig in self.active[l]:
                for ind in range(self.T):
                    self.flag2[self.cell(ind, ig)] = 0
            for ig in self.active[l]:
                gn = self.nbor_grids(ig)
                for ind in range(self.T):
                    cnt = sum(int(self.flag1[c]) for c in self.nbor_cells(gn, ind))
                    if cnt >= n_nbor[ismooth]:
                        self.flag2[self.cell(ind, ig)] = 1
            for ig in self.active[l]:
                for ind in range(self.T):
                    c = self.cell(ind, ig)
                    if self.flag1[c] == 1:
                        self.flag2[c] = 0
                    if self.flag2[c] == 1:
                        self.flag1[c] = 1
            self.make_boundary_flag(l)

    def hydro_refine_ok(self, ug, um, ud):
        """hydro_refine hydro/godunov_utils.f90:125-263 for one cell and one direction pair"""
        p, nd = self.p, self.ndim
        prim = []
        for u in (ug, um, ud):
            u = list(u)
            u[0] = max(u[0], p.smallr)
            ek = 0.0
            for d in range(nd):
                u[d + 1] = u[d + 1] / u[0]
            for d in range(nd):
                ek = ek + 0.5 * u[0] * u[d + 1] ** 2
            u[nd + 1] = (p.gamma - 1.0) * (u[nd + 1] - ek)
            prim.append(u)
        g, m_, d_ = prim
        ok = False
        if self.err_grad_d >= 0.0:
            err = 2.0 * max(abs((d_[0] - m_[0]) / (d_[0] + m_[0] + self.floor_d)), abs((m_[0] - g[0]) / (m_[0] + g[0] + self.floor_d)))
            ok = ok or err > self.err_grad_d
        if self.err_grad_p >= 0.0:
            ip = nd + 1
            err = 2.0 * max(abs((d_[ip] - m_[ip]) / (d_[ip] + m_[ip] + self.floor_p)), abs((m_[ip] - g[ip]) / (m_[ip] + g[ip] + self.floor_p)))
            ok = ok or err > self.err_grad_p
        if self.err_grad_u >= 0.0:
            ip = nd + 1
            for d in range(nd):
                vg, vm, vd = g[d + 1], m_[d + 1], d_[d + 1]
                cg = math.sqrt(max(p.gamma * g[ip] / g[0], self.floor_u ** 2))
                cm = math.sqrt(max(p.gamma * m_[ip] / m_[0], self.floor_u ** 2))
                cd = math.sqrt(max(p.gamma * d_[ip] / d_[0], self.floor_u ** 2))
                err = 2.0 * max(abs((vd - vm) / (cd + cm + abs(vd) + abs(vm) + self.floor_u)),
                                abs((vm - vg) / (cm + cg + abs(vm) + abs(vg) + self.floor_u)))
                ok = ok or err > self.err_grad_u
        return ok

    def hydro_flag(self, l):
        """hydro/hydro_flag.f90:1"""
        if l == self.nlevelmax or self.numbtot(l) == 0:
            return
        if self.err_grad_d == -1.0 and self.err_grad_p == -1.0 and self.err_grad_u == -1.0:
            return
        U = self.uold.reshape(self.nvar, self.ncell)
        for ig in self.active[l]:
            gn = self.nbor_grids(ig)
            for ind in range(self.T):
                c = self.cell(ind, ig)
                indn = self.nbor_cells(gn, ind)
                for j in range(self.twondim):
                    if indn[j] == 0:
                        indn[j] = int(self.nbor[j, ig])
                ok = False
                for d in range(self.ndim):
                    ok = ok or self.hydro_refine_ok(U[:, indn[2 * d] - 1], U[:, c - 1], U[:, indn[2 * d + 1] - 1])
                if ok:
                    self.flag1[c] = 1

    def ensure_ref_rules(self, l):
        """:197-255"""
        n3 = 3 ** self.ndim
        nfc = (C.c_int * 27)()
        for ig in self.active[l]:
            self.L.orc_get3cubefather(self.mp, int(self.father[ig]), l, nfc, None)
            ok = True
            for j in range(n3):
                if nfc[j] == 0 or self.son[nfc[j]] == 0:
                    ok = False
            if not ok:
                for ind in range(self.T):
                    self.flag1[self.cell(ind, ig)] = 0
        self.make_boundary_flag(l)

    def flag_fine(self, l, icount):
        """:56-104"""
        if l == self.nlevelmax or self.numbtot(l) == 0:
            return
        self.init_flag(l)
        if l < self.levelmin:
            return
        self.smooth_fine(l)
        self.hydro_flag(l)          # userflag_fine :257-375 (m_refine = -1)
        self.make_boundary_flag(l)
        for _ in range(self.nexpand[l]):
            self.smooth_fine(l)
        if l > self.levelmin and icount < self.nsubcycle[l - 1]:
            self.ensure_ref_rules(l)

    def flag(self):
        for l in range(self.nlevelmax - 1, 0, -1):
            self.flag_fine(l, 2)
        self.flag_coarse()

    # ------------------------------------------------------------------ refine_utils.f90
    def authorize_fine(self, l):
        """amr/virtual_boundaries.f90:34 (serial) + init_boundary_fine amr/physical_boundaries.f90:106"""
        if l == self.nlevelmax:
            return
        for ig in self.active[l]:
            for ind in range(self.T):
                self.flag2[self.cell(ind, ig)] = 1
        self.flag2[0] = 0
        for b in range(self.m.nboundary):
            for ig in self.bound[b][l]:
                for ind in range(self.T):
                    self.flag2[self.cell(ind, ig)] = 0
        if self.numbtot(l) > 0:
            n_nbor = [1, 2, 3]
            for ismooth in range(self.ndim):
                for b in range(self.m.nboundary):
                    for ig in self.bound[b][l]:
                        for ind in range(self.T):
                            self.flag1[self.cell(ind, ig)] = 0
                for b in range(self.m.nboundary):
                    for ig in self.bound[b][l]:
                        gn = self.nbor_grids(ig)
                        for ind in range(self.T):
                            cnt = sum(int(self.flag2[c]) for c in self.nbor_cells(gn, ind))
                            if cnt >= n_nbor[ismooth]:
                                self.flag1[self.cell(ind, ig)] = 1
                for b in range(self.m.nboundary):
                    for ig in self.bound[b][l]:
                        for ind in range(self.T):
                            c = self.cell(ind, ig)
                            if self.flag1[c] == 1:
                                self.flag2[c] = 1
        self.make_boundary_flag(l)

    def make_grid_coarse(self, ind, b):
        """:165-330"""
        m = self.m
        ig = self.free.pop(0)
        nxny = m.nx * m.ny
        iz = (ind - 1) // nxny
        iy = (ind - 1 - iz * nxny) // m.nx
        ix = ind - 1 - iy * m.nx - iz * nxny
        pos = [ix, iy, iz]
        nn = [m.nx, m.ny, m.nz]
        strd = [1, m.nx, nxny]
        for d in range(self.ndim):
            self.xg[d, ig] = pos[d] + 0.5
        self.son[ind] = ig
        self.father[ig] = ind
        for d in range(self.ndim):
            self.nbor[2 * d, ig] = ind - strd[d] if pos[d] > 0 else ind + (nn[d] - 1) * strd[d]
            self.nbor[2 * d + 1, ig] = ind + strd[d] if pos[d] < nn[d] - 1 else ind - (nn[d] - 1) * strd[d]
        (self.active[1] if b < 0 else self.bound[b][1]).append(ig)

    def refine_coarse(self):
        """:25-160 (level-1 octs exist for every coarse cell, domain and boundary regions)"""
        m = self.m
        nxny = m.nx * m.ny
        dom = set()
        for k in range(m.kcoarse_min, m.kcoarse_max + 1):
            for j in range(m.jcoarse_min, m.jcoarse_max + 1):
                for i in range(m.icoarse_min, m.icoarse_max + 1):
                    ind = 1 + i + j * m.nx + k * nxny
                    dom.add(ind)
                    if self.flag1[ind] == 1 and self.son[ind] == 0:
                        self.make_grid_coarse(ind, -1)
        # boundary regions (:93-150): by default one slab of coarse cells per boundary face
        for b in range(m.nboundary):
            bt = m.boundary_type[b]
            bdir = bt - 10 * (bt // 10)
            d, s = (bdir - 1) // 2, (bdir - 1) % 2
            cmin = [m.icoarse_min, m.jcoarse_min, m.kcoarse_min]
            cmax = [m.icoarse_max, m.jcoarse_max, m.kcoarse_max]
            rng = [range(cmin[x], cmax[x] + 1) for x in range(3)]
            rng[d] = [cmin[d] - 1] if s == 0 else [cmax[d] + 1]
            if self.bound_regions is not None:
                rng = [range(lo, hi + 1) for lo, hi in self.bound_regions[b][1:]]
            for k in rng[2]:
                for j in rng[1]:
                    for i in rng[0]:
                        ind = 1 + i + j * m.nx + k * nxny
                        if self.flag1[ind] == 1 and self.son[ind] == 0:
                            self.make_grid_coarse(ind, b)

    def make_grid_fine(self, ig_father, ind, lnew, b):
        """:590-948 for one new oct: father cell = cell `ind` of oct ig_father (level lnew-1)"""
        c = self.cell(ind, ig_father)
        ig = self.free.pop(0)
        dx = 0.5 ** (lnew - 1)
        for d in range(self.ndim):
            self.xg[d, ig] = self.xg[d, ig_father] + (((ind >> d) & 1) - 0.5) * dx
        self.son[c] = ig
        self.father[ig] = c
        indn = self.nbor_cells(self.nbor_grids(ig_father), ind)
        for j in range(self.twondim):
            self.nbor[j, ig] = indn[j]
            if indn[j] == 0 and b < 0:
                raise RuntimeError("Fatal error in make_grid_fine")          # :612-626
        (self.active[lnew] if b < 0 else self.bound[b][lnew]).append(ig)
        if not self.init:
            u2 = self.c_interpol_cell(c, lnew)
            U = self.uold.reshape(self.nvar, self.ncell)
            for j in range(self.T):
                U[:, self.cell(j, ig) - 1] = u2[j * self.nvar:(j + 1) * self.nvar]

    def kill_grid(self, c, lkill, b):
        """:953-1100"""
        ig = int(self.son[c])
        self.son[c] = 0
        (self.active[lkill] if b < 0 else self.bound[b][lkill]).remove(ig)
        for d in range(self.ndim):
            self.xg[d, ig] = 0.0
        self.father[ig] = 0
        self.nbor[:, ig] = 0
        self.free.insert(0, ig)      # killed octs go back to the head of the free list

    def refine_fine(self, l):
        """:332-585"""
        if l == self.nlevelmax or self.numbtot(l) == 0:
            return
        self.authorize_fine(l)
        nv = self.nvector
        for kind, b, lst in self.all_lists(l):
            snapshot = list(lst)
            for i0 in range(0, len(snapshot), nv):
                chunk = snapshot[i0:i0 + nv]
                for ind in range(self.T):
                    for ig in chunk:
                        c = self.cell(ind, ig)
                        if self.flag2[c] == 1 and self.flag1[c] == 1 and self.son[c] == 0:
                            self.make_grid_fine(ig, ind, l + 1, b)
        for kind, b, lst in self.all_lists(l):
            snapshot = list(lst)
            for i0 in range(0, len(snapshot), nv):
                chunk = snapshot[i0:i0 + nv]
                for ind in range(self.T):
                    for ig in chunk:
                        c = self.cell(ind, ig)
                        if self.flag1[c] == 0 and self.son[c] > 0:
                            self.kill_grid(c, l + 1, b)
        self.push_lists(l + 1)

    def refine(self):
        self.refine_coarse()
        self.push_lists(1)
        for l in range(1, self.nlevelmax):
            self.refine_fine(l)

    # ------------------------------------------------------------------ hydro passes (C oracle)
    # ---- the floating-point routines (C oracle); the MHD driver (oracle/amr_mhd.py) overrides these -------------------
    def c_set_unew(self, l):
        self.L.orc_set_unew(C.byref(self.p), self.mp, l, orc.dptr(self.uold), orc.dptr(self.unew))

    def c_godunov_fine(self, l):
        self.L.orc_godunov_fine(C.byref(self.p), self.mp, l, self.dtnew[l], orc.dptr(self.uold), orc.dptr(self.unew), 1)

    def c_set_uold(self, l):
        self.L.orc_set_uold(C.byref(self.p), self.mp, l, orc.dptr(self.uold), orc.dptr(self.unew))

    def c_interpol_cell(self, c, lnew):
        u2 = np.zeros(self.T * self.nvar)
        self.L.orc_interpol_cell(C.byref(self.p), self.mp, c, lnew, orc.dptr(self.uold), orc.dptr(u2))
        return u2

    def make_boundary_hydro(self, l):
        self.L.orc_make_boundary_hydro(C.byref(self.p), self.mp, l, orc.dptr(self.uold))

    def upload_fine(self, l):
        self.L.orc_upload_fine(C.byref(self.p), self.mp, l, orc.dptr(self.uold))

    def init_flow_fine(self, l):
        if self.numbtot(l) == 0:
            return
        orc.condinit_regions(self.p, _MeshView(self), l, self.uold, self.regions)

    def init_flow(self):
        """hydro/init_flow_fine.f90:5-23"""
        for l in range(self.nlevelmax, 0, -1):
            if l >= self.levelmin:
                self.init_flow_fine(l)
            self.upload_fine(l)
            self.make_boundary_hydro(l)

    # ------------------------------------------------------------------ init_refine.f90
    def init_refine(self):
        self.init = True
        for _ in range(1, self.levelmin + 1):
            self.flag()
            self.refine()
        for l in range(self.levelmin + 1, self.nlevelmax + 1):
            self.init_flow()
            self.flag()
            self.refine()
            if self.numbtot(l) == 0:
                break
        self.init = False
        self.init_flow()

    def init_refine_2(self):
        for _ in range(self.levelmin, self.nlevelmax + 2):
            self.refine_coarse()
            self.push_lists(1)
            for l in range(1, self.nlevelmax + 1):
                self.refine_fine(l)
                self.init_flow_fine(l)
            for l in range(self.nlevelmax, self.levelmin - 1, -1):
                self.upload_fine(l)
                self.make_boundary_hydro(l)
            for l in range(self.nlevelmax, 0, -1):
                self.flag_fine(l, 2)
            self.flag_coarse()

    # ------------------------------------------------------------------ time stepping
    def update_time(self, l):
        """amr/update_time.f90 (the parts that steer the run)"""
        dt = self.dtnew[l]
        if self.nstep_coarse != self.nstep_coarse_old:
            if self.t >= self.tout[-1]:
                self.done = True          # clean_end
                return
        self.nstep_coarse_old = self.nstep_coarse
        self.t = self.t + dt
        self.nstep += 1

    def newdt_fine(self, l):
        """pm/newdt_fine.f90:47-51,177 + hydro/courant_fine.f90"""
        self.dtold[l] = self.dtnew[l]
        self.dtnew[l] = self.p.boxlen / self.p.smallc
        sums = np.zeros(3)
        self.dtnew[l] = self.L.orc_courant_fine(C.byref(self.p), self.mp, l, self.dtnew[l], orc.dptr(self.uold), orc.dptr(sums))

    def dump(self):
        """leaf cells of the domain as output_hydro.f90 writes them (primitive variables)"""
        U = self.uold.reshape(self.nvar, self.ncell)
        p = self.p
        nx_loc = self.m.icoarse_max - self.m.icoarse_min + 1
        scale = p.boxlen / nx_loc
        rows = []
        for l in range(1, self.nlevelmax + 1):
            dx = 0.5 ** l
            for ig in self.active[l]:
                for ind in range(self.T):
                    c = self.cell(ind, ig)
                    if self.son[c] == 0:
                        d = max(U[0, c - 1], p.smallr)
                        vel = [U[1 + k, c - 1] / d for k in range(self.ndim)]
                        e = U[self.ndim + 1, c - 1]                      # output_hydro.f90:108-115
                        for k in range(self.ndim):
                            e = e - 0.5 * U[1 + k, c - 1] ** 2 / d
                        pr = (p.gamma - 1.0) * e
                        x = [(self.xg[k, ig] + (((ind >> k) & 1) - 0.5) * dx - [self.m.icoarse_min, self.m.jcoarse_min, self.m.kcoarse_min][k]) * scale
                             for k in range(self.ndim)]
                        rows.append((l, x, U[0, c - 1], vel, pr))
        return rows

    def amr_step(self, l, icount):
        """amr/amr_step.f90"""
        if self.numbtot(l) == 0 or self.done:
            return
        if self.levelmin < self.nlevelmax and not self.static:
            if l == self.levelmin or icount > 1:
                for i in range(l, self.nlevelmax + 1):
                    if i > self.levelmin:
                        self.make_boundary_hydro(i)                 # :50-70 (build_comm + boundaries)
                    self.refine_fine(i)                             # :92
        if l == self.levelmin:                                     # :141-175 output
            if self.iout < len(self.tout) and self.t >= self.tout[self.iout]:
                self.snapshot = dict(t=self.t, rows=self.dump(), nstep=self.nstep, nstep_coarse=self.nstep_coarse,
                                     grids={k: len(self.active[k]) for k in range(1, self.nlevelmax + 1)}, dt=self.dtnew[self.levelmin])
                self.iout += 1
        self.newdt_fine(l)                                         # :326
        if l > self.levelmin:
            self.dtnew[l] = min(self.dtnew[l - 1] / float(self.nsubcycle[l - 1]), self.dtnew[l])
        self.c_set_unew(l)                                         # :333
        if l < self.nlevelmax:
            if self.numbtot(l + 1) > 0:
                if self.nsubcycle[l] == 2:
                    self.amr_step(l + 1, 1)
                    self.amr_step(l + 1, 2)
                else:
                    self.amr_step(l + 1, 1)
            else:
                self.dtold[l + 1] = self.dtnew[l] / float(self.nsubcycle[l])
                self.dtnew[l + 1] = self.dtnew[l] / float(self.nsubcycle[l])
                self.update_time(l)
        else:
            self.update_time(l)
        if self.done:
            return
        self.c_godunov_fine(l)                                     # :388
        self.c_set_uold(l)                                         # :423
        self.upload_fine(l)                                                                                  # :441
        self.make_boundary_hydro(l)                                                                          # :514
        if not self.static:
            self.flag_fine(l, icount)                                                                        # :531
        if l > self.levelmin:
            if self.nsubcycle[l - 1] == 1:
                self.dtnew[l - 1] = self.dtnew[l]
            if icount == 2:
                self.dtnew[l - 1] = self.dtold[l] + self.dtnew[l]

    def run(self, max_coarse=100000):
        """amr/adaptive_loop.f90"""
        self.flag_coarse()
        self.init_refine()
        self.init_refine_2()
        self.initial_grids = {k: len(self.active[k]) for k in range(1, self.nlevelmax + 1)}
        self.nstep_coarse_old = self.nstep_coarse
        while not self.done and self.nstep_coarse < max_coarse:
            if self.levelmin < self.nlevelmax:
                self.refine_coarse()
                self.push_lists(1)
                for l in range(1, self.levelmin + 1):
                    self.make_boundary_hydro(l)
                    if l < self.levelmin:
                        self.refine_fine(l)
            self.amr_step(self.levelmin, 1)
            if self.done:
                break
            if self.levelmin < self.nlevelmax:
                for l in range(self.levelmin - 1, 0, -1):
                    self.upload_fine(l)
                    self.make_boundary_hydro(l)
                for l in range(self.levelmin - 1, 0, -1):
                    self.flag_fine(l, 2)
                self.flag_coarse()
            self.nstep_coarse += 1
        return self.snapshot


class FastAmrRun(AmrRun):
    """AmrRun with the per-cell flag / scan passes done by oracle/ramses_oracle_amr.c (same passes, same visiting order; the
    Python methods of AmrRun remain the readable statement and the cross-check).  Needed for the 2-D golden run."""

    def __init__(self, *a, nthreads=None, **kw):
        super().__init__(*a, **kw)
        L = self.L
        import os
        L.orc_set_amr_threads.argtypes = [C.c_int]     # flux phase only; bit-identical to the serial routine for any count
        L.orc_set_amr_threads(int(nthreads) if nthreads else min(8, os.cpu_count() or 1))
        MP, ip, dp = C.POINTER(orc.MeshS), C.POINTER(C.c_int), C.POINTER(C.c_double)
        L.orc_amr_make_boundary_flag.argtypes = [MP, C.c_int, ip]
        L.orc_amr_init_flag.argtypes = [MP, C.c_int, C.c_int, ip]
        L.orc_amr_smooth_fine.argtypes = [MP, C.c_int, ip, ip]
        L.orc_amr_hydro_flag.argtypes = [C.POINTER(orc.Params), MP, C.c_int, dp, ip, dp, dp]
        L.orc_amr_ensure_ref_rules.argtypes = [MP, C.c_int, ip]
        L.orc_amr_authorize_fine.argtypes = [MP, C.c_int, ip, ip]
        L.orc_amr_refine_scan.argtypes = [MP, C.c_int, C.c_int, C.c_int, C.c_int, ip, ip, C.c_int, ip, C.c_int]
        self._f1, self._f2 = orc.iptr(self.flag1), orc.iptr(self.flag2)
        self._scan = np.zeros(2 * self.T * (self.ngridmax + 1), dtype=np.int32)

    def make_boundary_flag(self, l):
        self.L.orc_amr_make_boundary_flag(self.mp, l, self._f1)

    def init_flag(self, l):
        self.L.orc_amr_init_flag(self.mp, l, self.levelmin, self._f1)

    def smooth_fine(self, l):
        if l == self.nlevelmax or self.numbtot(l) == 0:
            return
        self.L.orc_amr_smooth_fine(self.mp, l, self._f1, self._f2)

    def hydro_flag(self, l):
        if l == self.nlevelmax or self.numbtot(l) == 0:
            return
        if self.err_grad_d == -1.0 and self.err_grad_p == -1.0 and self.err_grad_u == -1.0:
            return
        err = np.array([self.err_grad_d, self.err_grad_u, self.err_grad_p])
        flo = np.array([self.floor_d, self.floor_u, self.floor_p])
        self.L.orc_amr_hydro_flag(C.byref(self.p), self.mp, l, orc.dptr(self.uold), self._f1, orc.dptr(err), orc.dptr(flo))

    def ensure_ref_rules(self, l):
        self.L.orc_amr_ensure_ref_rules(self.mp, l, self._f1)

    def authorize_fine(self, l):
        if l == self.nlevelmax:
            return
        self.L.orc_amr_authorize_fine(self.mp, l, self._f1, self._f2)

    def refine_fine(self, l):
        if l == self.nlevelmax or self.numbtot(l) == 0:
            return
        self.authorize_fine(l)
        cap = len(self._scan) // 2
        for mode in (0, 1):
            for kind, b, lst in self.all_lists(l):
                n = self.L.orc_amr_refine_scan(self.mp, l, kind, max(b, 0), self.nvector, self._f1, self._f2, mode,
                                               orc.iptr(self._scan), cap)
                assert n <= cap
                for ig, ind in self._scan[:2 * n].reshape(n, 2).tolist():
                    if mode == 0:
                        self.make_grid_fine(ig, ind, l + 1, b)
                    else:
                        self.kill_grid(self.cell(ind, ig), l + 1, b)
        self.push_lists(l + 1)


class _MeshView:
    """duck-typed stand-in for orc.Mesh in orc.condinit_regions"""

    def __init__(self, run):
        self.ptr = run.mp


def check_sums(rows, ndim, boxlen=1.0):
    """tests/visu/visu_ramses.py:495-557 check_solution sums for the hydro fields.  Vector components are thresholded
    against 2e-14 x norm, where the norm is the vector length only if all three components exist in the snapshot (true
    for x,y,z -- never binding -- and for NDIM=3 velocities) and 1 otherwise."""
    lev = np.array([r[0] for r in rows], dtype=float)

    def filt(a):
        av = np.average(a)
        if av == 0.0:
            return a
        return np.where(np.abs(a - av) / abs(av) < 1.0e-14, av, a)
    dens = np.array([r[2] for r in rows])
    pres = np.array([r[4] for r in rows])
    out = {"ncells": float(len(rows)), "level": math.fsum(np.abs(filt(lev))), "dx": math.fsum(np.abs(filt(0.5 ** lev * boxlen))),
           "density": math.fsum(np.log10(np.abs(filt(dens)))), "pressure": math.fsum(np.log10(np.abs(filt(pres))))}
    vel = [np.array([r[3][k] for r in rows]) for k in range(ndim)]
    norm = np.sqrt(sum(v * v for v in vel)) if ndim == 3 else 1.0
    for k in range(ndim):
        out["xyz"[k]] = math.fsum(np.abs(filt(np.array([r[1][k] for r in rows]))))
        kd = filt(vel[k])
        out["velocity_" + "xyz"[k]] = math.fsum(np.where(np.abs(kd) < 2.0e-14 * norm, 0.0, np.abs(kd)))
    return out
