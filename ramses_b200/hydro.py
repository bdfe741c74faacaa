"""Host-side mirror of the reference's driver interface for the hydro sweep.

The reference keeps all state in module globals (amr_commons, hydro_commons,
hydro_parameters) and its routines take only `ilevel`:

    call courant_fine(ilevel)   ! hydro/courant_fine.f90:1
    call set_unew(ilevel)       ! hydro/godunov_fine.f90:40
    call godunov_fine(ilevel)   ! hydro/godunov_fine.f90:5
    call set_uold(ilevel)       ! hydro/godunov_fine.f90:135
    call make_boundary_hydro(ilevel)  ! hydro/hydro_boundary.f90:5

`AmrCommons` plays the role of those modules (same array names, shapes and 1-based
index conventions, stored as Fortran-ordered numpy arrays) and `HydroGPU` exposes the
routines under the same names, forwarding to the C-ABI (include/ramses_gpu.h).
"""
import ctypes as C
import numpy as np
from . import lib as _lib


class AmrCommons:
    """amr_commons + hydro_commons + hydro_parameters of one rank (amr/amr_commons.f90, hydro/hydro_commons.f90).

    son(1:ncell), father(1:ngridmax), nbor(1:ngridmax,1:twondim) are int32 numpy arrays holding the Fortran
    arrays element for element (index i of Fortran = index i-1 here); uold/unew(1:ncell,1:nvar) are float64
    arrays of shape (nvar, ncell) (= column-major (ncell,nvar)).  active[l] / boundary[b][l] / reception[c][l] /
    emission[c][l] are the %igrid lists (1-based oct indices).
    """

    def __init__(self, ndim, nvar, ncoarse, ngridmax, nx, ny, nz, icoarse=(0, 0), jcoarse=(0, 0), kcoarse=(0, 0),
                 nlevelmax=1, boxlen=1.0, myid=1, ncpu=1, mhd=False):
        self.ndim, self.nvar = ndim, nvar
        self.mhd = bool(mhd)                     # SOLVER=mhd build: uold(1:ncell,1:nvar+3), mhd/hydro_commons.f90
        self.nvar_store = nvar + 3 if mhd else nvar
        self.ncoarse, self.ngridmax = ncoarse, ngridmax
        self.twotondim, self.twondim = 1 << ndim, 2 * ndim
        self.ncell = ncoarse + self.twotondim * ngridmax
        self.nx, self.ny, self.nz = nx, ny, nz
        self.icoarse_min, self.icoarse_max = icoarse
        self.jcoarse_min, self.jcoarse_max = jcoarse
        self.kcoarse_min, self.kcoarse_max = kcoarse
        self.nlevelmax, self.boxlen = nlevelmax, boxlen
        self.myid, self.ncpu = myid, ncpu
        self.son = np.zeros(self.ncell, dtype=np.int32)
        self.father = np.zeros(ngridmax, dtype=np.int32)
        self.nbor = np.zeros((self.twondim, ngridmax), dtype=np.int32)   # Fortran nbor(1:ngridmax,1:twondim)
        self.uold = np.zeros((self.nvar_store, self.ncell), dtype=np.float64)
        self.unew = np.zeros((self.nvar_store, self.ncell), dtype=np.float64)
        self.active = {}       # ilevel -> int32 array of igrid
        self.boundary = {}     # ilevel -> list of int32 arrays, one per ibound
        self.boundary_type = []
        self.reception = {}    # ilevel -> list (per cpu) of int32 arrays
        self.emission = {}
        self.dtnew = {}
        # hydro_parameters defaults (hydro/hydro_parameters.f90:75-85)
        self.gamma, self.courant_factor = 1.4, 0.5
        self.smallr, self.smallc = 1e-10, 1e-10
        self.slope_type, self.slope_theta = 1, 1.5
        self.niter_riemann, self.difmag = 10, 0.0
        self.scheme, self.riemann = "muscl", "llf"
        self.nvector = 32
        self.pressure_fix = False
        self.mass_tot = self.ekin_tot = self.eint_tot = self.emag_tot = 0.0
        self.riemann2d, self.slope_mag_type = "llf", -1          # mhd/hydro_parameters.f90:93,104

    def dx(self, ilevel):
        nx_loc = self.icoarse_max - self.icoarse_min + 1
        return 0.5 ** ilevel * self.boxlen / nx_loc


def _ip(a):
    return a.ctypes.data_as(C.POINTER(C.c_int))


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def make_params(amr):
    """struct rgpu_params from the module variables (what the Fortran shim fills after read_params)."""
    p = _lib.Params()
    p.ndim, p.nvar, p.nvector = amr.ndim, amr.nvar, amr.nvector
    p.slope_type, p.niter_riemann = amr.slope_type, amr.niter_riemann
    if amr.scheme not in ("muscl", "plmde"):
        raise ValueError("unknown scheme")
    p.scheme = 0 if amr.scheme == "muscl" else 1
    if getattr(amr, "mhd", False):
        if amr.riemann not in _lib.MHD_RIEMANN:
            raise ValueError("unknown riemann solver")      # mhd/umuscl.f90:1435
        if amr.riemann2d not in _lib.MHD_RIEMANN2D:
            raise ValueError("unknown 2D riemann solver")   # mhd/umuscl.f90:1886
        p.riemann, p.riemann2d = _lib.MHD_RIEMANN[amr.riemann], _lib.MHD_RIEMANN2D[amr.riemann2d]
        p.mhd, p.slope_mag_type = 1, amr.slope_mag_type
    else:
        if amr.riemann not in _lib.RIEMANN:
            raise ValueError("unknown Riemann solver")      # hydro/umuscl.f90:801-803
        p.riemann = _lib.RIEMANN[amr.riemann]
    p.pressure_fix = int(bool(amr.pressure_fix))
    p.poisson = int(bool(getattr(amr, "poisson", False)))   # f(1:ncell,1:ndim) is an input: HydroGPU.upload_force
    p.beta_fix = float(getattr(amr, "beta_fix", 0.0))
    p.fast = int(bool(getattr(amr, "fast", False)))        # rgpu_params.fast: FAST arithmetic of the 3-D dense sweep
    p.gamma, p.smallr, p.smallc = amr.gamma, amr.smallr, amr.smallc
    p.slope_theta, p.difmag, p.courant_factor, p.boxlen = amr.slope_theta, amr.difmag, amr.courant_factor, amr.boxlen
    p.nx, p.ny, p.nz = amr.nx, amr.ny, amr.nz
    p.icoarse_min, p.icoarse_max = amr.icoarse_min, amr.icoarse_max
    p.jcoarse_min, p.jcoarse_max = amr.jcoarse_min, amr.jcoarse_max
    p.kcoarse_min, p.kcoarse_max = amr.kcoarse_min, amr.kcoarse_max
    p.nlevelmax = amr.nlevelmax
    return p


def _level_lists(a, ilevel, keep):
    """ctypes views of the communicator lists of one level, in the argument order of rgpu_bind_level."""
    act = np.ascontiguousarray(a.active[ilevel], dtype=np.int32)
    bl = [np.ascontiguousarray(x, dtype=np.int32) for x in a.boundary.get(ilevel, [])]
    nb = len(bl)
    btype = (C.c_int * max(nb, 1))(*a.boundary_type[:nb])
    nbnd = (C.c_int * max(nb, 1))(*[len(x) for x in bl])
    bptr = (C.POINTER(C.c_int) * max(nb, 1))(*[_ip(x) for x in bl])
    ncpu = a.ncpu
    if ncpu > 1:
        rl = [np.ascontiguousarray(x, dtype=np.int32) for x in a.reception[ilevel]]
        el = [np.ascontiguousarray(x, dtype=np.int32) for x in a.emission[ilevel]]
        nr = (C.c_int * ncpu)(*[len(x) for x in rl])
        ne = (C.c_int * ncpu)(*[len(x) for x in el])
        rp = (C.POINTER(C.c_int) * ncpu)(*[_ip(x) for x in rl])
        ep = (C.POINTER(C.c_int) * ncpu)(*[_ip(x) for x in el])
        keep.append((rl, el))
    else:
        nr = ne = rp = ep = None
    keep.append((act, bl))
    return (len(act), _ip(act), ncpu, nr, rp, ne, ep, nb, btype, nbnd, bptr)


def plan_level(amr, ilevel):
    """Host-only dry run of bind_level (rgpu_plan_level): returns (LevelInfo, slot_igrid array).  No GPU needed."""
    L = _lib.load()
    p = make_params(amr)
    keep = []
    args = _level_lists(amr, ilevel, keep)
    info = _lib.LevelInfo()
    cap = 8 * max(len(amr.active[ilevel]), 1) + 64
    for _ in range(2):
        slots = np.zeros(cap, dtype=np.int32)
        rc = L.rgpu_plan_level(C.byref(p), amr.myid, amr.ncoarse, amr.ngridmax, _ip(amr.father), ilevel, *args,
                               C.byref(info), _ip(slots), cap)
        if rc == 0 or info.nslot <= cap:
            break
        cap = int(info.nslot)
    _lib.check(rc)
    return info, slots[:info.nslot].copy()


class HydroGPU:
    """The patched routines of hydro/godunov_fine.f90 & friends, running on the GPU through the C-ABI."""

    def __init__(self, amr: AmrCommons, device=-1, amr_mode=False, interpol_type=1, interpol_var=0, interpol_mag_type=-1):
        self.a = amr
        self.L = _lib.load()
        p = make_params(amr)
        self.params = p
        _lib.check(self.L.rgpu_init(C.byref(p), amr.myid, amr.ncpu, device))
        if amr_mode:      # levelmin < nlevelmax: oct-list kernels on mirrored arrays
            _lib.check(self.L.rgpu_set_amr(1, interpol_type, interpol_var))
            self.set_interpol_mag(interpol_mag_type)
        self._keep = []
        self.bind_tree()

    def set_interpol_mag(self, interpol_mag_type):
        """interpol_mag_type of the MHD build (face-field prolongation limiter; -1 = interpol_type), rgpu_set_interpol_mag"""
        _lib.check(self.L.rgpu_set_interpol_mag(int(interpol_mag_type)))

    # -- bookkeeping the Fortran shim performs after build_comm / refine ------------------------------
    def bind_tree(self):
        a = self.a
        assert a.son.dtype == np.int32 and a.father.dtype == np.int32 and a.nbor.dtype == np.int32
        assert a.nbor.flags["C_CONTIGUOUS"]
        _lib.check(self.L.rgpu_bind_tree(a.ncoarse, a.ngridmax, _ip(a.son), _ip(a.father), _ip(a.nbor)))

    def bind_level(self, ilevel):
        args = _level_lists(self.a, ilevel, self._keep)
        _lib.check(self.L.rgpu_bind_level(ilevel, *args))

    def level_info(self, ilevel):
        info = _lib.LevelInfo()
        _lib.check(self.L.rgpu_get_level_info(ilevel, C.byref(info)))
        return info

    # -- Level-0 contract: the drop-in godunov_fine(ilevel) on host arrays --------------------------------
    def godunov_fine(self, ilevel):
        """godunov_fine(ilevel): unew(active cells) = uold + flux differences, dt = dtnew(ilevel)."""
        a = self.a
        _lib.check(self.L.rgpu_godunov_fine(ilevel, float(a.dtnew[ilevel]), _dp(a.uold), _dp(a.unew)))

    # -- Level-1 contract: device resident ----------------------------------------------------------------
    def upload_state(self, ilevel):
        _lib.check(self.L.rgpu_upload_state(ilevel, _dp(self.a.uold)))

    def download_state(self, ilevel):
        _lib.check(self.L.rgpu_download_state(ilevel, _dp(self.a.uold)))

    def set_unew(self, ilevel):
        _lib.check(self.L.rgpu_set_unew(ilevel))

    def godunov_fine_dev(self, ilevel):
        _lib.check(self.L.rgpu_godunov_fine_dev(ilevel, float(self.a.dtnew[ilevel])))

    def set_uold(self, ilevel):
        _lib.check(self.L.rgpu_set_uold(ilevel))

    def courant_fine(self, ilevel):
        """courant_fine(ilevel): dtnew(ilevel) = min(dtnew(ilevel), CFL dt); mass_tot etc. accumulated."""
        a = self.a
        dt = C.c_double(a.dtnew[ilevel])
        sums = (C.c_double * 4)(0.0, 0.0, 0.0, 0.0)
        _lib.check(self.L.rgpu_courant_fine(ilevel, C.byref(dt), sums))
        a.dtnew[ilevel] = dt.value
        a.mass_tot += sums[0]; a.ekin_tot += sums[1]; a.eint_tot += sums[2]; a.emag_tot += sums[3]
        return dt.value

    def make_boundary_hydro(self, ilevel):
        _lib.check(self.L.rgpu_make_boundary_hydro(ilevel))

    def upload_fine(self, ilevel):
        _lib.check(self.L.rgpu_upload_fine(ilevel))

    def make_virtual_fine(self, ilevel):
        _lib.check(self.L.rgpu_make_virtual_fine(ilevel))

    def make_virtual_reverse(self, ilevel):
        _lib.check(self.L.rgpu_make_virtual_reverse(ilevel))

    def level_steps(self, ilevel, nstep):
        """nstep fused level steps (courant -> set_unew -> godunov_fine -> set_uold -> ghosts -> boundaries)."""
        dts = np.zeros(nstep)
        sums = (C.c_double * 4)()
        _lib.check(self.L.rgpu_level_steps(ilevel, nstep, _dp(dts), sums))
        return dts, list(sums)

    def amr_steps(self, levelmin, nsubcycle, ncoarse_steps):
        """ncoarse_steps x amr_step(levelmin, 1) with device-resident time steps (rgpu_amr_steps); returns dtnew(levelmin) per step.
        nsubcycle: list indexed by LEVEL (element 0 unused), like amr_step below; the C-ABI takes the Fortran array
        nsubcycle(1:nlevelmax), i.e. the same list without its element 0."""
        ns = np.ascontiguousarray((list(nsubcycle) + [2] * 64)[1: self.a.nlevelmax + 1], dtype=np.int32)
        dts = np.zeros(ncoarse_steps)
        _lib.check(self.L.rgpu_amr_steps(levelmin, _ip(ns), ncoarse_steps, _dp(dts)))
        return dts

    def hydro_flag(self, ilevel, flag1, err_grad, floor=(1e-10, 1e-10, 1e-10)):
        """hydro_flag(ilevel) (hydro/hydro_flag.f90): ORs the gradient criteria into the host array flag1(1:ncell) (int32);
        err_grad = (err_grad_d, err_grad_u, err_grad_p), floor = (floor_d, floor_u, floor_p) of &REFINE_PARAMS."""
        assert flag1.dtype == np.int32 and flag1.flags["C_CONTIGUOUS"]
        e = (C.c_double * 3)(*err_grad)
        f = (C.c_double * 3)(*floor)
        _lib.check(self.L.rgpu_hydro_flag(ilevel, e, f, _ip(flag1)))

    def set_boundary_var(self, ibound, var):
        """boundary_var(ibound, 1:nvar) of an imposed boundary region (bound_type=3); ibound is 1-based."""
        v = np.ascontiguousarray(var, dtype=np.float64)
        assert v.size >= self.a.nvar
        _lib.check(self.L.rgpu_set_boundary_var(int(ibound), _dp(v)))

    def upload_force(self, f):
        """poisson_commons' f(1:ncell,1:ndim) (numpy [ndim][ncell], C order = the Fortran column-major array) -> device."""
        assert f.dtype == np.float64 and f.flags["C_CONTIGUOUS"] and f.shape == (self.a.ndim, self.a.ncell)
        _lib.check(self.L.rgpu_upload_force(_dp(f)))

    def download_pressure_fix(self):
        """divu(1:ncell), enew(1:ncell) of hydro_commons from the device (pressure_fix)."""
        divu, enew = np.zeros(self.a.ncell), np.zeros(self.a.ncell)
        _lib.check(self.L.rgpu_download_pressure_fix(_dp(divu), _dp(enew)))
        return divu, enew

    def level_totals(self):
        """numbtot(1,1:nlevelmax): octs per level over all ranks (NCCL sum in AMR mode); stored in a.numbtot (dict by level)."""
        n = self.a.nlevelmax
        out = (C.c_int * n)()
        _lib.check(self.L.rgpu_level_totals(n, out))
        self.a.numbtot = {l: int(out[l - 1]) for l in range(1, n + 1)}
        self.a.numbtot[n + 1] = 0
        return self.a.numbtot

    def host_register(self, arr):
        _lib.check(self.L.rgpu_host_register(arr.ctypes.data, arr.nbytes))

    def host_unregister(self, arr):
        _lib.check(self.L.rgpu_host_unregister(arr.ctypes.data))

    def set_timing(self, on):
        _lib.check(self.L.rgpu_set_timing(int(on)))

    def set_pipeline(self, on):
        """Level-0 call: allow (default) / forbid the three-stream slab pipeline (rgpu_set_pipeline)."""
        _lib.check(self.L.rgpu_set_pipeline(int(on)))

    def synchronize(self):
        _lib.check(self.L.rgpu_device_synchronize())

    def finalize(self):
        _lib.check(self.L.rgpu_finalize())


def amr_step(h, ilevel, icount, levelmin, nsubcycle, dtnew, dtold, multi_rank=False):
    """amr_step(ilevel, icount) of amr/amr_step.f90 for the hydro solver on a frozen mesh (no flag/refine pass): the
    recursion and the sub-cycling stay on the host exactly like in the Fortran driver, every per-level routine is the
    `HydroGPU` call of the same name.  dtnew/dtold: dicts indexed by level (amr_commons dtnew/dtold); nsubcycle: list
    indexed by level (amr_parameters.f90:nsubcycle, 1 or 2).  Line numbers refer to amr/amr_step.f90."""
    a = h.a
    # numbtot(1,ilevel): the GLOBAL oct count gates the step and the recursion (:33, :345) -- a rank without octs at a level
    # still takes part in the level's all-reduce and exchanges.  a.numbtot (HydroGPU.level_totals) when set, else local counts
    nt = getattr(a, "numbtot", None)
    ntot = (lambda l: nt.get(l, 0)) if nt else (lambda l: len(a.active.get(l, [])))
    if ntot(ilevel) == 0:
        return
    dtold[ilevel] = dtnew[ilevel]
    a.dtnew[ilevel] = a.boxlen / a.smallc                        # newdt_fine :326 (pm/newdt_fine.f90:47-51)
    dtnew[ilevel] = h.courant_fine(ilevel)
    if ilevel > levelmin:
        dtnew[ilevel] = min(dtnew[ilevel - 1] / float(nsubcycle[ilevel - 1]), dtnew[ilevel])
    a.dtnew[ilevel] = dtnew[ilevel]
    h.set_unew(ilevel)                                           # :333
    if ilevel < a.nlevelmax and ntot(ilevel + 1) > 0:                      # recursive call :345-361
        for ic in ((1, 2) if nsubcycle[ilevel] == 2 else (1,)):
            amr_step(h, ilevel + 1, ic, levelmin, nsubcycle, dtnew, dtold, multi_rank)
    elif ilevel < a.nlevelmax:
        dtold[ilevel + 1] = dtnew[ilevel] / float(nsubcycle[ilevel])
        dtnew[ilevel + 1] = dtnew[ilevel] / float(nsubcycle[ilevel])
    a.dtnew[ilevel] = dtnew[ilevel]
    h.godunov_fine_dev(ilevel)                                   # :388
    if multi_rank:
        h.make_virtual_reverse(ilevel)                           # :397
    h.set_uold(ilevel)                                           # :423
    h.upload_fine(ilevel)                                        # :441
    if multi_rank:
        h.make_virtual_fine(ilevel)                              # :505
    h.make_boundary_hydro(ilevel)                                # :514
    if ilevel > levelmin:                                        # :567-577
        if nsubcycle[ilevel - 1] == 1:
            dtnew[ilevel - 1] = dtnew[ilevel]
        if icount == 2:
            dtnew[ilevel - 1] = dtold[ilevel] + dtnew[ilevel]
