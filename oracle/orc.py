"""ctypes binding of the CPU ORACLE (oracle/ramses_oracle.c).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline / --impl reference legs.  Never imported by ramses_b200/.
"""
import ctypes as C
import os
import subprocess
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(_HERE, "libramses_oracle.so")

RIEMANN = {"llf": 0, "exact": 1, "acoustic": 2, "hllc": 3, "hll": 4}
MAXBOUND = 6


def build(force=False):
    srcs = [os.path.join(_HERE, f) for f in ("ramses_oracle.c", "ramses_oracle.h", "ramses_oracle_mhd.c", "ramses_oracle_mhd.h",
                                              "ramses_oracle_amr.c")]
    if force or not os.path.exists(_LIB) or os.path.getmtime(_LIB) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["make", "-C", _HERE, "-s", "-B", "libramses_oracle.so"])
    return _LIB


class Params(C.Structure):
    _fields_ = [("ndim", C.c_int), ("nvar", C.c_int), ("nvector", C.c_int), ("slope_type", C.c_int),
                ("niter_riemann", C.c_int), ("scheme", C.c_int), ("riemann", C.c_int), ("pad_", C.c_int),
                ("gamma", C.c_double), ("smallr", C.c_double), ("smallc", C.c_double),
                ("slope_theta", C.c_double), ("difmag", C.c_double), ("courant_factor", C.c_double),
                ("boxlen", C.c_double)]


class MeshS(C.Structure):
    _fields_ = [("ndim", C.c_int), ("nx", C.c_int), ("ny", C.c_int), ("nz", C.c_int),
                ("icoarse_min", C.c_int), ("icoarse_max", C.c_int), ("jcoarse_min", C.c_int),
                ("jcoarse_max", C.c_int), ("kcoarse_min", C.c_int), ("kcoarse_max", C.c_int),
                ("ncoarse", C.c_int), ("ngridmax", C.c_int), ("ncell", C.c_int), ("nlevelmax", C.c_int),
                ("nboundary", C.c_int), ("boundary_type", C.c_int * MAXBOUND),
                ("son", C.POINTER(C.c_int)), ("father", C.POINTER(C.c_int)), ("nbor", C.POINTER(C.c_int)),
                ("xg", C.POINTER(C.c_double)), ("cpu_map", C.POINTER(C.c_int)),
                ("nactive", C.POINTER(C.c_int)), ("active", C.POINTER(C.POINTER(C.c_int))),
                ("nrecv", C.POINTER(C.c_int)), ("recv", C.POINTER(C.POINTER(C.c_int))),
                ("nbound", C.POINTER(C.c_int) * MAXBOUND),
                ("bound", C.POINTER(C.POINTER(C.c_int)) * MAXBOUND),
                ("ngrid_used", C.c_int)]


class MhdParams(C.Structure):
    _fields_ = [("slope_type", C.c_int), ("slope_mag_type", C.c_int), ("riemann", C.c_int), ("riemann2d", C.c_int),
                ("gamma", C.c_double), ("smallr", C.c_double), ("smallc", C.c_double), ("slope_theta", C.c_double),
                ("courant_factor", C.c_double), ("boxlen", C.c_double)]


MHD_RIEMANN = {"llf": 0, "roe": 1, "hll": 2, "hlld": 3, "upwind": 4, "hydro": 5}
MHD_RIEMANN2D = {"llf": 0, "roe": 1, "upwind": 2, "hll": 3, "hlla": 4, "hlld": 5}
MHD_NVAR = 8          # nvar of the MHD build; 11 = nvar+3 variables are stored (right-face B in 9..11)

_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB)
        dp = C.POINTER(C.c_double)
        ip = C.POINTER(C.c_int)
        pp = C.POINTER(Params)
        mp = C.POINTER(MeshS)
        L.orc_mesh_build_uniform.restype = mp
        L.orc_mesh_build_uniform.argtypes = [C.c_int, C.c_int, ip, C.c_int, C.c_uint]
        L.orc_mesh_build_box.restype = mp
        L.orc_mesh_build_box.argtypes = [C.c_int, C.c_int, ip, ip, C.c_int, C.c_uint]
        L.orc_mesh_free.argtypes = [mp]
        L.orc_mesh_oct_pos.argtypes = [mp, C.c_int, C.c_int, ip]
        L.orc_get3cubefather.argtypes = [mp, C.c_int, C.c_int, ip, ip]
        L.orc_getindices3cube.argtypes = [C.c_int, C.c_int, ip, ip]
        L.orc_dx.restype = C.c_double
        L.orc_dx.argtypes = [pp, mp, C.c_int]
        L.orc_condinit_regions.argtypes = [pp, mp, C.c_int, dp, C.c_int, ip] + [dp] * 12
        L.orc_set_unew.argtypes = [pp, mp, C.c_int, dp, dp]
        L.orc_set_uold.argtypes = [pp, mp, C.c_int, dp, dp]
        L.orc_godunov_fine.argtypes = [pp, mp, C.c_int, C.c_double, dp, dp, C.c_int]
        L.orc_courant_fine.restype = C.c_double
        L.orc_courant_fine.argtypes = [pp, mp, C.c_int, C.c_double, dp, dp]
        L.orc_make_boundary_hydro.argtypes = [pp, mp, C.c_int, dp]
        L.orc_run_uniform.argtypes = [pp, mp, C.c_int, C.c_int, dp, dp, dp, dp, C.c_int]
        for nm in ("llf", "hll", "hllc", "acoustic", "approx"):
            getattr(L, "orc_riemann_" + nm).argtypes = [pp, dp, dp, dp, C.c_int]
        L.orc_cmpdt.argtypes = [pp, dp, dp, C.c_double, dp, C.c_int]
        L.orc_work_new.restype = C.c_void_p
        L.orc_work_new.argtypes = [pp]
        L.orc_work_free.argtypes = [C.c_void_p]
        L.orc_unsplit.argtypes = [pp, C.c_void_p, dp, dp, dp, dp] + [C.c_double] * 4 + [C.c_int]
        # ideal-MHD variant (oracle/ramses_oracle_mhd.c)
        mpp = C.POINTER(MhdParams)
        L.orc_mhd_work_new.restype = C.c_void_p
        L.orc_mhd_work_free.argtypes = [C.c_void_p]
        for nm in ("uloc", "flux"):
            getattr(L, "orc_mhd_work_" + nm).restype = dp
            getattr(L, "orc_mhd_work_" + nm).argtypes = [C.c_void_p]
        L.orc_mhd_work_emf.restype = dp
        L.orc_mhd_work_emf.argtypes = [C.c_void_p, C.c_int]
        L.orc_mhd_riemann.argtypes = [mpp, dp, dp, dp]
        L.orc_mhd_emf.restype = C.c_double
        L.orc_mhd_emf.argtypes = [mpp, dp, dp, dp, dp, C.c_int]
        L.orc_mhd_unsplit.argtypes = [mpp, C.c_void_p, C.c_double, C.c_double]
        L.orc_mhd_cmpdt_cell.restype = C.c_double
        L.orc_mhd_cmpdt_cell.argtypes = [mpp, dp, C.c_double]
        L.orc_mhd_set_unew.argtypes = [mp, C.c_int, dp, dp]
        L.orc_mhd_set_uold.argtypes = [mp, C.c_int, dp, dp]
        L.orc_mhd_godunov_fine.argtypes = [mpp, mp, C.c_int, C.c_double, dp, dp, C.c_int]
        L.orc_mhd_courant_fine.restype = C.c_double
        L.orc_mhd_courant_fine.argtypes = [mpp, mp, C.c_int, C.c_double, dp, dp]
        L.orc_mhd_make_boundary_hydro.argtypes = [mpp, mp, C.c_int, dp]
        L.orc_mhd_run_uniform.argtypes = [mpp, mp, C.c_int, C.c_int, dp, dp, dp, dp, C.c_int]
        L.orc_mhd_set_threads.argtypes = [C.c_int]
        _lib = L
    return _lib


def dptr(a):
    assert a.dtype == np.float64 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.POINTER(C.c_double))


def iptr(a):
    assert a.dtype == np.int32 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.POINTER(C.c_int))


def make_params(ndim=3, nvar=None, nvector=32, slope_type=1, niter_riemann=10, riemann="llf", gamma=1.4,
                smallr=1e-10, smallc=1e-10, slope_theta=1.5, difmag=0.0, courant_factor=0.8, boxlen=1.0):
    p = Params()
    p.ndim = ndim
    p.nvar = nvar if nvar else ndim + 2
    p.nvector = nvector
    p.slope_type = slope_type
    p.niter_riemann = niter_riemann
    p.scheme = 0
    p.riemann = RIEMANN[riemann] if isinstance(riemann, str) else riemann
    p.gamma, p.smallr, p.smallc = gamma, smallr, smallc
    p.slope_theta, p.difmag, p.courant_factor, p.boxlen = slope_theta, difmag, courant_factor, boxlen
    return p


class Mesh:
    """Fully refined oct tree (levels 1..levelmax) fabricated by the oracle's builder.  coarse = (nx, ny, nz): the domain
    coarse cells (boundary coarse cells are added around them for every face with a boundary type)."""

    def __init__(self, ndim, levelmax, bound_type=(0,) * 6, order=0, seed=1, coarse=(1, 1, 1)):
        bt = (C.c_int * 6)(*bound_type)
        if tuple(coarse) == (1, 1, 1):
            self.ptr = lib().orc_mesh_build_uniform(ndim, levelmax, bt, order, seed)
        else:
            if any(coarse[d] != 1 for d in range(ndim, 3)) or min(coarse) < 1:
                raise ValueError(f"coarse={coarse} does not fit ndim={ndim}")
            self.ptr = lib().orc_mesh_build_box(ndim, levelmax, (C.c_int * 3)(*coarse), bt, order, seed)
        self.s = self.ptr.contents
        self.ndim, self.levelmax = ndim, levelmax

    def __del__(self):
        try:
            lib().orc_mesh_free(self.ptr)
        except Exception:
            pass

    # numpy views (1-based arrays: element 0 unused) -------------------------------
    @property
    def ncell(self): return self.s.ncell
    @property
    def ncoarse(self): return self.s.ncoarse
    @property
    def ngridmax(self): return self.s.ngridmax

    def son(self): return np.ctypeslib.as_array(self.s.son, shape=(self.s.ncell + 1,))
    def father(self): return np.ctypeslib.as_array(self.s.father, shape=(self.s.ngridmax + 1,))
    def nbor(self): return np.ctypeslib.as_array(self.s.nbor, shape=(2 * self.ndim, self.s.ngridmax + 1))
    def xg(self): return np.ctypeslib.as_array(self.s.xg, shape=(self.ndim, self.s.ngridmax + 1))
    def active(self, l): return np.ctypeslib.as_array(self.s.active[l], shape=(max(self.s.nactive[l], 1),))[:self.s.nactive[l]]
    def bound(self, b, l):
        n = self.s.nbound[b][l]
        return np.ctypeslib.as_array(self.s.bound[b][l], shape=(max(n, 1),))[:n]
    def boundary_types(self): return [self.s.boundary_type[b] for b in range(self.s.nboundary)]

    def oct_pos(self, l, igrid):
        pos = (C.c_int * 3)()
        lib().orc_mesh_oct_pos(self.ptr, l, int(igrid), pos)
        return tuple(pos)

    def coarse(self):
        """domain coarse cells per axis (icoarse_max - icoarse_min + 1 etc.)"""
        s = self.s
        return (s.icoarse_max - s.icoarse_min + 1, s.jcoarse_max - s.jcoarse_min + 1, s.kcoarse_max - s.kcoarse_min + 1)

    def extent(self, l):
        """(nx, ny, nz) cells of the domain at level l (1 along the unused axes)"""
        return tuple(self.coarse()[d] << l if d < self.ndim else 1 for d in range(3))

    def new_state(self, nvar):
        return np.zeros(nvar * self.s.ncell, dtype=np.float64)

    def cell_index(self, igrid, ind):
        """1-based cell index of cell `ind` (0-based position) of oct igrid."""
        return self.s.ncoarse + ind * self.s.ngridmax + igrid

    def level_to_dense(self, u, l, nvar):
        """Gather the active cells of level l into a dense [nvar][nz][ny][nx] array (domain only)."""
        nd = self.ndim
        ig = self.active(l).astype(np.int64)
        pos = np.array([self.oct_pos(l, g) for g in ig], dtype=np.int64) if len(ig) < 5000 else self._pos_fast(l, ig)
        cmin = np.array([self.s.icoarse_min, self.s.jcoarse_min, self.s.kcoarse_min]) * (1 << (l - 1))
        pos = pos - cmin[None, :]
        shape = self.extent(l)
        out = np.zeros((nvar, shape[2], shape[1], shape[0]))
        uu = u.reshape(nvar, self.s.ncell)
        for ind in range(1 << nd):
            cx = 2 * pos[:, 0] + (ind & 1)
            cy = 2 * pos[:, 1] + ((ind >> 1) & 1) if nd > 1 else np.zeros_like(cx)
            cz = 2 * pos[:, 2] + ((ind >> 2) & 1) if nd > 2 else np.zeros_like(cx)
            ic = self.s.ncoarse + ind * self.s.ngridmax + ig - 1
            out[:, cz, cy, cx] = uu[:, ic]
        return out

    def dense_to_level(self, dense, u, l, nvar):
        nd = self.ndim
        ext = self.extent(l)
        assert dense.shape[1:] == (ext[2], ext[1], ext[0]), (dense.shape, ext)
        ig = self.active(l).astype(np.int64)
        pos = self._pos_fast(l, ig)
        cmin = np.array([self.s.icoarse_min, self.s.jcoarse_min, self.s.kcoarse_min]) * (1 << (l - 1))
        pos = pos - cmin[None, :]
        uu = u.reshape(nvar, self.s.ncell)
        for ind in range(1 << nd):
            cx = 2 * pos[:, 0] + (ind & 1)
            cy = 2 * pos[:, 1] + ((ind >> 1) & 1) if nd > 1 else np.zeros_like(cx)
            cz = 2 * pos[:, 2] + ((ind >> 2) & 1) if nd > 2 else np.zeros_like(cx)
            ic = self.s.ncoarse + ind * self.s.ngridmax + ig - 1
            uu[:, ic] = dense[:, cz, cy, cx]

    def _pos_fast(self, l, ig):
        """Vectorised father-chain walk: integer oct positions (units of oct size at level l)."""
        father = self.father().astype(np.int64)
        nc, ng = self.s.ncoarse, self.s.ngridmax
        chain = []
        g = ig.copy()
        for lev in range(l, 1, -1):
            ic = father[g]
            ind = (ic - nc - 1) // ng
            g = ic - nc - ind * ng
            chain.append(ind)
        ic = father[g]
        nxny = self.s.nx * self.s.ny
        pz = (ic - 1) // nxny
        py = (ic - 1 - pz * nxny) // self.s.nx
        px = ic - 1 - py * self.s.nx - pz * nxny
        pos = np.stack([px, py, pz], axis=1)
        for ind in reversed(chain):
            pos = 2 * pos + np.stack([ind & 1, (ind >> 1) & 1, (ind >> 2) & 1], axis=1)
        return pos


def condinit_regions(p, mesh, l, u, regions):
    """regions: list of dicts like the INIT_PARAMS namelist (hydro/init_flow_fine.f90:475)."""
    n = len(regions)
    rt = np.array([0 if r.get("type", "square") == "square" else 1 for r in regions], dtype=np.int32)
    def arr(key, default):
        return np.array([float(r.get(key, default)) for r in regions], dtype=np.float64)
    args = [arr("x_center", 0), arr("y_center", 0), arr("z_center", 0), arr("length_x", 1e10), arr("length_y", 1e10),
            arr("length_z", 1e10), arr("exp_region", 2.0), arr("d", 0), arr("u", 0), arr("v", 0), arr("w", 0), arr("p", 0)]
    lib().orc_condinit_regions(C.byref(p), mesh.ptr, l, dptr(u), n, iptr(rt), *[dptr(a) for a in args])


def run_uniform(p, mesh, l, nstep, uold, nthreads=1):
    unew = np.zeros_like(uold)
    dts = np.zeros(nstep)
    t = C.c_double(0.0)
    lib().orc_run_uniform(C.byref(p), mesh.ptr, l, nstep, dptr(uold), dptr(unew), dptr(dts), C.byref(t), nthreads)
    return dts, t.value


# ---------------------------------------------------------------------------------------------------------
# ideal MHD (NDIM=3, nvar=8 stored as 11)
def make_mhd_params(slope_type=1, slope_mag_type=-1, riemann="llf", riemann2d="llf", gamma=1.4, smallr=1e-10, smallc=1e-10,
                    slope_theta=1.5, courant_factor=0.8, boxlen=1.0):
    p = MhdParams()
    p.slope_type = slope_type
    p.slope_mag_type = slope_type if slope_mag_type == -1 else slope_mag_type     # hydro/read_hydro_params.f90:528
    p.riemann = MHD_RIEMANN[riemann] if isinstance(riemann, str) else riemann
    p.riemann2d = MHD_RIEMANN2D[riemann2d] if isinstance(riemann2d, str) else riemann2d
    p.gamma, p.smallr, p.smallc = gamma, smallr, smallc
    p.slope_theta, p.courant_factor, p.boxlen = slope_theta, courant_factor, boxlen
    return p


def mhd_run_uniform(p, mesh, l, nstep, uold, nthreads=1):
    unew = np.zeros_like(uold)
    dts = np.zeros(nstep)
    t = C.c_double(0.0)
    lib().orc_mhd_run_uniform(C.byref(p), mesh.ptr, l, nstep, dptr(uold), dptr(unew), dptr(dts), C.byref(t), nthreads)
    return dts, t.value


def mhd_state_from_primitives(d, vel, P, bface, gamma):
    """Dense conservative MHD state [11][nz][ny][nx] from cell primitives and the three staggered face fields.
    bface[c] has one extra layer along axis c: bface[0] is [nz][ny][nx+1] etc. (left face of cell i = index i).
    E includes 0.5*B_c^2 with B_c the face average (mhd/condinit.f90:60-75)."""
    nz, ny, nx = d.shape
    u = np.zeros((11, nz, ny, nx))
    u[0] = d
    for c in range(3):
        u[1 + c] = d * vel[c]
    u[5] = bface[0][:, :, :-1]; u[8] = bface[0][:, :, 1:]
    u[6] = bface[1][:, :-1, :]; u[9] = bface[1][:, 1:, :]
    u[7] = bface[2][:-1, :, :]; u[10] = bface[2][1:, :, :]
    ekin = 0.5 * d * (vel[0] ** 2 + vel[1] ** 2 + vel[2] ** 2)
    emag = 0.125 * ((u[5] + u[8]) ** 2 + (u[6] + u[9]) ** 2 + (u[7] + u[10]) ** 2)
    u[4] = P / (gamma - 1.0) + ekin + emag
    return u
