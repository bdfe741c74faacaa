"""Shared test scaffolding: fabricate a RAMSES oct tree + state the way the Fortran caller would own it,
and run the CPU oracle beside the GPU library on the same arrays."""
import ctypes as C
import numpy as np

from oracle import orc
from ramses_b200.hydro import AmrCommons

SEDOV3D_REGIONS = [  # namelist/sedov3d.nml:19-34
    dict(type="square", x_center=0.5, y_center=0.5, z_center=0.5, length_x=10.0, length_y=10.0, length_z=10.0,
         exp_region=10.0, d=1.0, p=1e-5),
    dict(type="point", x_center=0.0, y_center=0.0, z_center=0.0, length_x=1.0, length_y=1.0, length_z=1.0,
         exp_region=10.0, d=0.0, p=0.4)]
SEDOV1D_REGIONS = [  # namelist/sedov1d.nml:18-27
    dict(type="square", x_center=0.5, length_x=1.0, d=1.0, p=1e-5),
    dict(type="point", x_center=0.0, length_x=1.0, d=0.0, p=0.4)]
SOD_REGIONS = [      # namelist/tube1d.nml
    dict(type="square", x_center=0.25, length_x=0.5, d=1.0, p=1.0),
    dict(type="square", x_center=0.75, length_x=0.5, d=0.125, p=0.1)]


def smooth_state(ndim, n, gamma=1.4):
    """SURVEY 8d M2b: smooth, everywhere non-trivial state; returns conservative dense array [nvar][nz][ny][nx]."""
    L = 1.0
    ax = (np.arange(n) + 0.5) / n
    shp = [n if d < ndim else 1 for d in range(3)]
    x = ax[None, None, :] * np.ones((shp[2], shp[1], 1))
    y = (ax[None, :, None] if ndim > 1 else np.zeros((1, 1, 1))) * np.ones((shp[2], 1, shp[0]))
    z = (ax[:, None, None] if ndim > 2 else np.zeros((1, 1, 1))) * np.ones((1, shp[1], shp[0]))
    tw = 2 * np.pi / L
    rho = 1 + 0.2 * np.sin(tw * x) * np.cos(tw * y)
    vel = [0.3 * np.sin(tw * y), 0.3 * np.sin(tw * z), 0.3 * np.sin(tw * x)][:ndim]
    if ndim == 1:
        vel = [0.3 * np.sin(tw * x)]
    p = 1 + 0.1 * np.cos(tw * (x + y + z))
    u = np.zeros((ndim + 2,) + rho.shape)
    u[0] = rho
    e = p / (gamma - 1)
    for d in range(ndim):
        u[1 + d] = rho * vel[d]
        e = e + 0.5 * rho * vel[d] ** 2
    u[ndim + 1] = e
    return u


class Case:
    """One run set-up: oracle mesh + params + the Fortran-side arrays (AmrCommons)."""

    def __init__(self, ndim, level, riemann="hllc", slope_type=1, bound=(0,) * 6, order=0, seed=1, boxlen=1.0,
                 gamma=1.4, courant_factor=0.8, niter_riemann=10, slope_theta=1.5, nvector=32, nvar=None, coarse=(1, 1, 1)):
        """coarse = (nx, ny, nz) domain coarse cells; dx = boxlen / nx / 2^level"""
        self.ndim, self.level, self.nvar = ndim, level, (nvar or ndim + 2)      # nvar > ndim+2: passive scalars
        self.mesh = orc.Mesh(ndim, level, bound, order, seed, coarse=coarse)
        self.p = orc.make_params(ndim=ndim, nvar=self.nvar, riemann=riemann, slope_type=slope_type, boxlen=boxlen, gamma=gamma,
                                 courant_factor=courant_factor, niter_riemann=niter_riemann, slope_theta=slope_theta,
                                 nvector=nvector)
        self.riemann, self.slope_type = riemann, slope_type
        self.u = self.mesh.new_state(self.nvar)

    # ---- initial conditions ---------------------------------------------------------------------------
    def init_regions(self, regions):
        orc.condinit_regions(self.p, self.mesh, self.level, self.u, regions)
        orc.lib().orc_make_boundary_hydro(C.byref(self.p), self.mesh.ptr, self.level, orc.dptr(self.u))

    def init_dense(self, dense):
        self.mesh.dense_to_level(dense, self.u, self.level, self.nvar)
        orc.lib().orc_make_boundary_hydro(C.byref(self.p), self.mesh.ptr, self.level, orc.dptr(self.u))

    def dense(self, u=None):
        return self.mesh.level_to_dense(self.u if u is None else u, self.level, self.nvar)

    # ---- oracle drivers ----------------------------------------------------------------------------------
    def oracle_courant(self, u=None, dt_in=None):
        u = self.u if u is None else u
        sums = np.zeros(3)
        dt_in = self.p.boxlen / self.p.smallc if dt_in is None else dt_in
        dt = orc.lib().orc_courant_fine(C.byref(self.p), self.mesh.ptr, self.level, dt_in, orc.dptr(u), orc.dptr(sums))
        return dt, sums

    def oracle_godunov(self, dt, u=None, nthreads=4):
        """set_unew + godunov_fine on a copy; returns unew."""
        u = self.u if u is None else u
        unew = np.zeros_like(u)
        L = orc.lib()
        L.orc_set_unew(C.byref(self.p), self.mesh.ptr, self.level, orc.dptr(u), orc.dptr(unew))
        L.orc_godunov_fine(C.byref(self.p), self.mesh.ptr, self.level, dt, orc.dptr(u), orc.dptr(unew), nthreads)
        return unew

    def oracle_steps(self, nstep, u=None, nthreads=4):
        u = (self.u if u is None else u).copy()
        dts, t = orc.run_uniform(self.p, self.mesh, self.level, nstep, u, nthreads=nthreads)
        return u, dts

    # ---- the Fortran caller's view --------------------------------------------------------------------------
    def amr_commons(self, u=None):
        m, s = self.mesh, self.mesh.s
        a = AmrCommons(self.ndim, self.nvar, s.ncoarse, s.ngridmax, s.nx, s.ny, s.nz,
                       (s.icoarse_min, s.icoarse_max), (s.jcoarse_min, s.jcoarse_max), (s.kcoarse_min, s.kcoarse_max),
                       nlevelmax=self.level, boxlen=self.p.boxlen)
        a.son[:] = m.son()[1:]
        a.father[:] = m.father()[1:]
        a.nbor[:, :] = m.nbor()[:, 1:]
        a.uold[:, :] = (self.u if u is None else u).reshape(self.nvar, s.ncell)
        a.unew[:, :] = 0.0
        for l in range(1, self.level + 1):
            a.active[l] = m.active(l).copy()
            a.boundary[l] = [m.bound(b, l).copy() for b in range(s.nboundary)]
        a.boundary_type = m.boundary_types()
        a.gamma, a.courant_factor = self.p.gamma, self.p.courant_factor
        a.smallr, a.smallc = self.p.smallr, self.p.smallc
        a.slope_type, a.slope_theta = self.p.slope_type, self.p.slope_theta
        a.niter_riemann = self.p.niter_riemann
        a.riemann = self.riemann
        return a

    def active_cells(self):
        """0-based cell indices (into the ncell axis) of the active cells of the level."""
        s = self.mesh.s
        ig = self.mesh.active(self.level).astype(np.int64)
        return np.concatenate([s.ncoarse + ind * s.ngridmax + ig - 1 for ind in range(1 << self.ndim)])


def max_rel_err(a, b):
    """max |a-b| / max|b| per variable (relative on the conserved state vector, BASELINE north_star)."""
    a = np.asarray(a); b = np.asarray(b)
    out = 0.0
    for v in range(a.shape[0]):
        scale = np.abs(b[v]).max()
        if scale == 0:
            scale = 1.0
        out = max(out, np.abs(a[v] - b[v]).max() / scale)
    return out


# ------------------------------------------------------------------------------------------------------------
# ideal MHD (NDIM=3, nvar=8 stored as 11)
def mhd_smooth_state(n, gamma=5.0 / 3.0, b0=(0.5, 0.3, 0.2), amp=0.1, periodic=(True, True, True)):
    """Smooth periodic MHD state with a divergence-free staggered field built from an edge-centred vector potential.
    Face values shared by two cells (incl. the periodic wrap) are the same number on both sides.
    Returns the dense conservative array [11][n][n][n]."""
    h = 1.0 / n
    xc = (np.arange(n) + 0.5) * h
    xe = np.arange(n) * h                       # low edges / faces; the high one wraps onto index 0
    tw = 2 * np.pi
    Z, Y, X = np.meshgrid(xc, xc, xc, indexing="ij")
    d = 1 + 0.2 * np.sin(tw * X) * np.cos(tw * Y)
    vel = [0.3 * np.sin(tw * Y), 0.2 * np.cos(tw * Z), 0.1 * np.sin(tw * X)]
    P = 1 + 0.1 * np.cos(tw * Z) * np.sin(tw * (X + Y))
    # vector potential on the low edges of every cell
    ze, ye, x_ = np.meshgrid(xe, xe, xc, indexing="ij"); Ax = amp * np.sin(tw * ye) * np.cos(tw * ze)
    ze, y_, xe_ = np.meshgrid(xe, xc, xe, indexing="ij"); Ay = amp * np.sin(tw * ze + 1.0) * np.cos(tw * xe_)
    z_, ye, xe_ = np.meshgrid(xc, xe, xe, indexing="ij"); Az = amp * np.cos(tw * xe_) * np.sin(tw * ye + 0.3)
    up = lambda a, ax: np.roll(a, -1, axis=ax)
    # left-face fields of every cell (curl of A), axis order (z,y,x)
    bx = (up(Az, 1) - Az) / h - (up(Ay, 0) - Ay) / h + b0[0]
    by = (up(Ax, 0) - Ax) / h - (up(Az, 2) - Az) / h + b0[1]
    bz = (up(Ay, 2) - Ay) / h - (up(Ax, 1) - Ax) / h + b0[2]
    u = np.zeros((11, n, n, n))
    u[0] = d
    for c in range(3):
        u[1 + c] = d * vel[c]
    u[5], u[6], u[7] = bx, by, bz
    u[8], u[9], u[10] = up(bx, 2), up(by, 1), up(bz, 0)
    ekin = 0.5 * d * (vel[0] ** 2 + vel[1] ** 2 + vel[2] ** 2)
    emag = 0.125 * ((u[5] + u[8]) ** 2 + (u[6] + u[9]) ** 2 + (u[7] + u[10]) ** 2)
    u[4] = P / (gamma - 1.0) + ekin + emag
    return u


def mhd_box_state(ext, gamma=5.0 / 3.0, b0=(0.5, 0.3, 0.2), amp=0.1):
    """mhd_smooth_state on a box of ext = (nx, ny, nz) cells of size h = 1/nx: one wave across the box per axis (different
    periods per axis), divergence-free staggered field from an edge-centred vector potential that is periodic on the box.
    Returns the dense conservative array [11][nz][ny][nx]."""
    nx, ny, nz = ext
    h = 1.0 / nx
    k = [2 * np.pi / (e * h) for e in ext]
    xc = [(np.arange(e) + 0.5) * h for e in ext]
    xe = [np.arange(e) * h for e in ext]
    Z, Y, X = np.meshgrid(xc[2], xc[1], xc[0], indexing="ij")
    d = 1 + 0.2 * np.sin(k[0] * X) * np.cos(k[1] * Y) + 0.1 * np.sin(k[2] * Z + 0.7)
    vel = [0.3 * np.sin(k[1] * Y), 0.2 * np.cos(k[2] * Z), 0.1 * np.sin(k[0] * X)]
    P = 1 + 0.1 * np.cos(k[2] * Z) * np.sin(k[0] * X + k[1] * Y)
    ze, ye, _ = np.meshgrid(xe[2], xe[1], xc[0], indexing="ij"); Ax = amp * np.sin(k[1] * ye) * np.cos(k[2] * ze)
    ze, _, xe_ = np.meshgrid(xe[2], xc[1], xe[0], indexing="ij"); Ay = amp * np.sin(k[2] * ze + 1.0) * np.cos(k[0] * xe_)
    _, ye, xe_ = np.meshgrid(xc[2], xe[1], xe[0], indexing="ij"); Az = amp * np.cos(k[0] * xe_) * np.sin(k[1] * ye + 0.3)
    up = lambda a, ax: np.roll(a, -1, axis=ax)
    bx = (up(Az, 1) - Az) / h - (up(Ay, 0) - Ay) / h + b0[0]
    by = (up(Ax, 0) - Ax) / h - (up(Az, 2) - Az) / h + b0[1]
    bz = (up(Ay, 2) - Ay) / h - (up(Ax, 1) - Ax) / h + b0[2]
    u = np.zeros((11, nz, ny, nx))
    u[0] = d
    for c in range(3):
        u[1 + c] = d * vel[c]
    u[5], u[6], u[7] = bx, by, bz
    u[8], u[9], u[10] = up(bx, 2), up(by, 1), up(bz, 0)
    ekin = 0.5 * d * (vel[0] ** 2 + vel[1] ** 2 + vel[2] ** 2)
    emag = 0.125 * ((u[5] + u[8]) ** 2 + (u[6] + u[9]) ** 2 + (u[7] + u[10]) ** 2)
    u[4] = P / (gamma - 1.0) + ekin + emag
    return u


def box_state(ndim, ext, seed=3, gamma=1.4):
    """a hydro state on a box of ext = (nx, ny, nz) cells (1 beyond ndim) of size h = 1/nx with no symmetry that could hide a
    swapped axis: one wave across the box per axis, an off-centre Gaussian blob and seeded density jumps.  Periodic on the box
    (the blob is small enough).  Returns the dense conservative array [ndim+2][nz][ny][nx]."""
    h = 1.0 / ext[0]
    L = [e * h for e in ext]
    xs = [(np.arange(e) + 0.5) * h for e in ext]
    Z, Y, X = np.meshgrid(xs[2], xs[1], xs[0], indexing="ij")
    tw = 2 * np.pi
    sx, sy, sz = tw * X / L[0], tw * Y / L[1], tw * Z / L[2]
    r2 = ((X - 0.3 * L[0]) / (0.15 * L[0])) ** 2
    if ndim > 1:
        r2 = r2 + ((Y - 0.6 * L[1]) / (0.2 * L[1])) ** 2
    if ndim > 2:
        r2 = r2 + ((Z - 0.45 * L[2]) / (0.25 * L[2])) ** 2
    blob = np.exp(-r2)
    rho = 1 + 0.2 * np.sin(sx) * np.cos(sy) + 0.1 * np.sin(sz + 0.3) + 0.5 * blob
    rho *= 1 + 0.3 * (np.random.default_rng(seed).standard_normal(rho.shape) > 1.3)
    vel = [0.3 * np.sin(sy + 0.2) + 0.1 * np.cos(sz) + 0.1 * np.sin(sx), 0.25 * np.sin(sz) - 0.1 * np.sin(sx), 0.2 * np.sin(sx + 0.5)]
    p = 1 + 0.1 * np.cos(sx + sy + sz) + 2.0 * blob
    u = np.zeros((ndim + 2,) + rho.shape)
    u[0] = rho
    e = p / (gamma - 1)
    for d in range(ndim):
        u[1 + d] = rho * vel[d]
        e = e + 0.5 * rho * vel[d] ** 2
    u[ndim + 1] = e
    return u


def level_slots(mesh, l, u, nvar):
    """The octs of level l of an oracle mesh (active and boundary octs) in the dense-box slot layout of the device (plan_level:
    lattice order of the oct positions over the box spanned by them): returns uin [nvar][2^ndim][nslot] and the (igrid, slot)
    of the active octs."""
    nd = mesh.ndim
    act = mesh.active(l).astype(np.int64)
    ig = np.concatenate([act] + [mesh.bound(b, l).astype(np.int64) for b in range(mesh.s.nboundary)])
    pos = mesh._pos_fast(l, ig)
    lo = pos.min(axis=0)
    no = pos.max(axis=0) - lo + 1
    q = pos - lo
    slot = q[:, 0] + no[0] * (q[:, 1] + no[1] * q[:, 2])
    T = 1 << nd
    U = u.reshape(nvar, mesh.s.ncell)
    uin = np.zeros((nvar, T, int(no.prod())))
    for ind in range(T):
        uin[:, ind, slot] = U[:, mesh.s.ncoarse + ind * mesh.s.ngridmax + ig - 1]
    return uin, act, slot[:len(act)]


def mhd_tube_state(n, left, right, x0, boxlen, gamma):
    """Shock tube along x (mhd/condinit.f90 with two 'square' regions spanning y,z): left/right = (d,u,v,w,P,A,B,C)."""
    xc = (np.arange(n) + 0.5) * boxlen / n
    u = np.zeros((11, n, n, n))
    for sel, s in ((xc < x0, left), (xc >= x0, right)):
        d, vx, vy, vz, P, A, B, C = s
        u[0][:, :, sel] = d
        u[1][:, :, sel] = d * vx; u[2][:, :, sel] = d * vy; u[3][:, :, sel] = d * vz
        u[5][:, :, sel] = A; u[8][:, :, sel] = A
        u[6][:, :, sel] = B; u[9][:, :, sel] = B
        u[7][:, :, sel] = C; u[10][:, :, sel] = C
        u[4][:, :, sel] = P / (gamma - 1.0) + 0.5 * d * (vx * vx + vy * vy + vz * vz) + 0.5 * (A * A + B * B + C * C)
    return u


def mhd_divb(u, n_per_len):
    """cell-wise div(B) of a dense [11][nz][ny][nx] state from the two face copies"""
    return ((u[8] - u[5]) + (u[9] - u[6]) + (u[10] - u[7])) * n_per_len


class MhdCase:
    """MHD run set-up: oracle mesh + MHD params + the Fortran-side arrays (AmrCommons of an MHD build)."""

    def __init__(self, level, riemann="hlld", riemann2d="llf", slope_type=1, slope_mag_type=-1, bound=(0,) * 6, order=0, seed=1,
                 boxlen=1.0, gamma=5.0 / 3.0, courant_factor=0.8, slope_theta=1.5, coarse=(1, 1, 1)):
        self.ndim, self.level, self.nvar, self.nvs = 3, level, 8, 11
        self.mesh = orc.Mesh(3, level, bound, order, seed, coarse=coarse)
        self.p = orc.make_mhd_params(slope_type=slope_type, slope_mag_type=slope_mag_type, riemann=riemann, riemann2d=riemann2d,
                                     gamma=gamma, courant_factor=courant_factor, boxlen=boxlen, slope_theta=slope_theta)
        self.riemann, self.riemann2d, self.slope_type, self.slope_mag_type = riemann, riemann2d, slope_type, slope_mag_type
        self.u = self.mesh.new_state(11)

    def init_dense(self, dense):
        self.mesh.dense_to_level(dense, self.u, self.level, 11)
        orc.lib().orc_mhd_make_boundary_hydro(C.byref(self.p), self.mesh.ptr, self.level, orc.dptr(self.u))

    def dense(self, u=None):
        return self.mesh.level_to_dense(self.u if u is None else u, self.level, 11)

    def oracle_courant(self, u=None, dt_in=None):
        u = self.u if u is None else u
        sums = np.zeros(4)
        dt_in = self.p.boxlen / self.p.smallc if dt_in is None else dt_in
        dt = orc.lib().orc_mhd_courant_fine(C.byref(self.p), self.mesh.ptr, self.level, dt_in, orc.dptr(u), orc.dptr(sums))
        return dt, sums

    def oracle_godunov(self, dt, u=None, nthreads=4):
        u = self.u if u is None else u
        unew = np.zeros_like(u)
        L = orc.lib()
        L.orc_mhd_set_unew(self.mesh.ptr, self.level, orc.dptr(u), orc.dptr(unew))
        L.orc_mhd_godunov_fine(C.byref(self.p), self.mesh.ptr, self.level, dt, orc.dptr(u), orc.dptr(unew), nthreads)
        return unew

    def oracle_steps(self, nstep, u=None, nthreads=4):
        u = (self.u if u is None else u).copy()
        dts, t = orc.mhd_run_uniform(self.p, self.mesh, self.level, nstep, u, nthreads=nthreads)
        return u, dts

    def amr_commons(self, u=None):
        m, s = self.mesh, self.mesh.s
        a = AmrCommons(3, 8, s.ncoarse, s.ngridmax, s.nx, s.ny, s.nz,
                       (s.icoarse_min, s.icoarse_max), (s.jcoarse_min, s.jcoarse_max), (s.kcoarse_min, s.kcoarse_max),
                       nlevelmax=self.level, boxlen=self.p.boxlen, mhd=True)
        a.son[:] = m.son()[1:]
        a.father[:] = m.father()[1:]
        a.nbor[:, :] = m.nbor()[:, 1:]
        a.uold[:, :] = (self.u if u is None else u).reshape(11, s.ncell)
        a.unew[:, :] = 0.0
        for l in range(1, self.level + 1):
            a.active[l] = m.active(l).copy()
            a.boundary[l] = [m.bound(b, l).copy() for b in range(s.nboundary)]
        a.boundary_type = m.boundary_types()
        a.gamma, a.courant_factor = self.p.gamma, self.p.courant_factor
        a.smallr, a.smallc = self.p.smallr, self.p.smallc
        a.slope_type, a.slope_theta = self.p.slope_type, self.p.slope_theta
        a.riemann, a.riemann2d, a.slope_mag_type = self.riemann, self.riemann2d, self.slope_mag_type
        return a

    def active_cells(self):
        s = self.mesh.s
        ig = self.mesh.active(self.level).astype(np.int64)
        return np.concatenate([s.ncoarse + ind * s.ngridmax + ig - 1 for ind in range(8)])
