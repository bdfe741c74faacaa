"""Fabricate the oct-tree arrays a RAMSES rank owns for a fully refined (levelmin=levelmax) periodic run.

This is host plumbing for benchmarks and multi-GPU tests: it produces exactly the arrays the Fortran side
hands to the C-ABI (amr/amr_commons.f90:68-79,108-119,170-180): son, father, nbor, active(l)%igrid and, for
ncpu>1, reception(icpu,l)%igrid / emission(icpu,l)%igrid.  The domain is the reference's coarse grid
(nx,ny,nz) (amr/amr_parameters.f90) with every coarse cell refined down to `levelmax`; with ncpu ranks, rank r
owns the subtree of coarse cell r (the Hilbert partition of a full cube at 2/4/8 ranks gives each rank one
such sub-cube, amr/load_balance.f90:657-688) and holds, like a RAMSES rank, only its own octs, one layer of
ghost octs (nexpand_bound=1) and their ancestors, in a rank-local igrid numbering.
"""
import numpy as np

from .hydro import AmrCommons


def _bits(ind, ndim):
    return np.stack([(ind >> d) & 1 for d in range(3)], axis=-1) * (np.arange(3) < ndim)


def coarse_dims_for_ranks(ndim, ncpu):
    """(nx,ny,nz): one coarse cell per rank, split x first, then y, then z."""
    dims = [1, 1, 1]
    d, n = 0, ncpu
    while n > 1:
        if n % 2:
            raise ValueError("ncpu must be a power of two")
        dims[d % ndim] *= 2
        n //= 2
        d += 1
    return tuple(dims)


def build_uniform_tree(ndim, levelmax, nvar=None, coarse=(1, 1, 1), myid=1, ncpu=1, order="creation", seed=1,
                       boxlen=1.0, mhd=False, xbound=None):
    """Returns an AmrCommons with the tree of rank `myid` (1-based).  order: 'creation' (the order in which the
    reference's refine pass creates octs: cell position outermost, amr/refine_utils.f90), 'lattice' or 'random'.
    xbound=(bound_type_min, bound_type_max) (single rank only; 1 reflexive, 2 zero gradient): the run has
    &BOUNDARY_PARAMS ibound_min=-1,+1 like namelist/tube_mhd.nml:17-22, i.e. a 3x1x1 coarse grid whose outer
    cells are boundary cells (icoarse_min=icoarse_max=1) carrying one layer of boundary octs per level."""
    nvar = nvar or (8 if mhd else ndim + 2)
    nx, ny, nz = coarse
    if xbound is not None:
        if ncpu != 1 or tuple(coarse) != (1, 1, 1):
            raise ValueError("xbound needs a single rank and a single domain coarse cell")
        nx = 3
    nc = np.array([nx, ny, nz], dtype=np.int64)
    if ncpu > 1 and nx * ny * nz != ncpu:
        raise ValueError("one coarse cell per rank is required")
    ncoarse = nx * ny * nz
    T = 1 << ndim
    r0 = myid - 1
    my_c = np.array([r0 % nx, (r0 // nx) % ny, r0 // (nx * ny)], dtype=np.int64)

    def key(pos, l):
        ext = nc << (l - 1)
        return pos[:, 0] + ext[0] * (pos[:, 1] + ext[1] * pos[:, 2])

    def unkey(k, l):
        ext = nc << (l - 1)
        return np.stack([k % ext[0], (k // ext[0]) % ext[1], k // (ext[0] * ext[1])], axis=1)

    # ---- which octs exist on this rank, level by level (finest first) ----------------------------------------
    L = levelmax
    ext = nc << (L - 1)
    n1 = 1 << (L - 1)
    if ncpu == 1:
        rng = [np.arange(ext[d]) for d in range(3)]
        if xbound is not None:
            rng[0] = np.arange(n1 - 1, 2 * n1 + 1)       # the domain [n1, 2 n1) plus one boundary oct on each side
    else:
        rng = []
        for d in range(3):
            if d < ndim:
                lo, hi = my_c[d] * n1 - 1, (my_c[d] + 1) * n1 + 1
                if nc[d] == 1:          # periodic onto itself: no ghost layer in that direction
                    lo, hi = 0, n1
                rng.append(np.unique(np.arange(lo, hi) % ext[d]))
            else:
                rng.append(np.arange(1))
    gz, gy, gx = np.meshgrid(rng[2], rng[1], rng[0], indexing="ij")
    pos = {L: np.stack([gx.ravel(), gy.ravel(), gz.ravel()], axis=1).astype(np.int64)}
    for l in range(L - 1, 0, -1):
        k = np.unique(key(pos[l + 1] >> 1, l))
        pos[l] = unkey(k, l)
    # ---- numbering ---------------------------------------------------------------------------------------------
    rs = np.random.RandomState(seed)
    keys, igrid0 = {}, {}
    nxt = 1
    for l in range(1, L + 1):
        p = pos[l]
        if order == "lattice":
            perm = np.argsort(key(p, l), kind="stable")
        elif order == "random":
            perm = rs.permutation(len(p))
        else:   # creation order: children of all parents for cell position 1, then position 2, ... recursively
            # digits: finest-level position most significant, coarse cell least significant
            rev = np.zeros(len(p), dtype=np.int64)
            q = p.copy()
            mult = 8 ** max(l - 2, 0)
            for k in range(l - 1):
                ind = (q[:, 0] & 1) + 2 * (q[:, 1] & 1) + 4 * (q[:, 2] & 1)
                rev += ind * mult
                mult //= 8
                q >>= 1
            rev = rev * ncoarse + (q[:, 0] + nx * (q[:, 1] + ny * q[:, 2]))
            perm = np.argsort(rev, kind="stable")
        pos[l] = p[perm]
        kk = key(pos[l], l)
        srt = np.argsort(kk, kind="stable")
        keys[l] = (kk[srt], srt)            # sorted keys and the local index of each
        igrid0[l] = nxt
        nxt += len(p)
    ngridmax = nxt - 1 + 8

    def lookup(l, p):
        """igrid (1-based) of the octs at positions p (periodic), 0 where absent."""
        e = nc << (l - 1)
        k = key(np.mod(p, e[None, :]), l)
        ks, srt = keys[l]
        i = np.searchsorted(ks, k)
        i = np.minimum(i, len(ks) - 1)
        ok = ks[i] == k
        return np.where(ok, igrid0[l] + srt[i], 0)

    a = AmrCommons(ndim, nvar, ncoarse, ngridmax, nx, ny, nz, (1, 1) if xbound is not None else (0, nx - 1), (0, ny - 1),
                   (0, nz - 1), nlevelmax=L, boxlen=boxlen, myid=myid, ncpu=ncpu, mhd=mhd)
    if xbound is not None:
        a.boundary_type = [(0 if t == 1 else 10) + k + 1 for k, t in enumerate(xbound)]    # hydro/read_hydro_params.f90:316-420
    # icoarse_min/max: the reference keeps nx_loc = icoarse_max-icoarse_min+1 = 1 for boxlen scaling unless the
    # user box spans several coarse cells; here the physical box spans the whole coarse grid in x
    for l in range(1, L + 1):
        p = pos[l]
        n = len(p)
        ig = igrid0[l] + np.arange(n)
        if l == 1:
            fcell = 1 + p[:, 0] + nx * (p[:, 1] + ny * p[:, 2])
        else:
            par = lookup(l - 1, p >> 1)
            ind = (p[:, 0] & 1) + 2 * (p[:, 1] & 1) + 4 * (p[:, 2] & 1)
            fcell = ncoarse + ind * ngridmax + par
        a.father[ig - 1] = fcell
        a.son[fcell - 1] = ig
        # nbor(igrid, 2d-1 / 2d): neighbouring father cell (level l-1 cell) in -d / +d
        for d in range(ndim):
            for s, sh in ((0, -1), (1, +1)):
                if l == 1:
                    q = p.copy()
                    q[:, d] = np.mod(q[:, d] + sh, nc[d])
                    nb = 1 + q[:, 0] + nx * (q[:, 1] + ny * q[:, 2])
                else:
                    q = p.copy()
                    q[:, d] += sh                       # neighbouring oct position = neighbouring father cell position
                    e = nc << (l - 1)
                    q[:, d] = np.mod(q[:, d], e[d])
                    par = lookup(l - 1, q >> 1)
                    ind = (q[:, 0] & 1) + 2 * (q[:, 1] & 1) + 4 * (q[:, 2] & 1)
                    nb = np.where(par > 0, ncoarse + ind * ngridmax + par, 0)
                a.nbor[2 * d + s, ig - 1] = nb
    # ---- ownership and communicator lists at every level ---------------------------------------------------------
    for l in range(1, L + 1):
        p = pos[l]
        ig = (igrid0[l] + np.arange(len(p))).astype(np.int32)
        cc = p >> (l - 1)                                # coarse cell containing the oct
        owner = cc[:, 0] + nx * (cc[:, 1] + ny * cc[:, 2])
        mine = owner == r0 if ncpu > 1 else np.ones(len(p), dtype=bool)
        a.boundary[l] = []
        if xbound is not None:
            mine = cc[:, 0] == 1
            a.boundary[l] = [ig[cc[:, 0] == 0], ig[cc[:, 0] == 2]]
        a.active[l] = ig[mine]
        if ncpu > 1:
            kk = key(p, l)
            rec, emi = [], []
            e = nc << (l - 1)
            n1l = 1 << (l - 1)
            for c in range(ncpu):
                if c == r0:
                    rec.append(np.zeros(0, np.int32)); emi.append(np.zeros(0, np.int32))
                    continue
                sel = np.nonzero(owner == c)[0]
                rec.append(ig[sel[np.argsort(kk[sel], kind="stable")]])        # ghost octs owned by c, by global key
                # my octs within one oct of rank c's cube (periodic)
                cpos = np.array([c % nx, (c // nx) % ny, c // (nx * ny)], dtype=np.int64)
                near = mine.copy()
                for d in range(ndim):
                    lo, hi = cpos[d] * n1l - 1, (cpos[d] + 1) * n1l
                    x = p[:, d]
                    inside = np.zeros(len(p), dtype=bool)
                    for shift in (-e[d], 0, e[d]):
                        inside |= (x + shift >= lo) & (x + shift <= hi)
                    near &= inside
                sel = np.nonzero(near)[0]
                emi.append(ig[sel[np.argsort(kk[sel], kind="stable")]])
            a.reception[l], a.emission[l] = rec, emi
    a._pos = pos
    a._igrid0 = igrid0
    return a


def cell_centers(a, ilevel):
    """(igrid array, ind, x[ncell_level, 3]) cell centres of the active cells in units of the full coarse grid
    length along x (periodic box [0, nx)x[0, ny)x[0, nz) coarse cells -> scaled so that x in [0, 1) * n_d/nx)."""
    pos = a._pos[ilevel]
    ig0 = a._igrid0[ilevel]
    ig = a.active[ilevel].astype(np.int64)
    p = pos[ig - ig0]
    out = []
    for ind in range(a.twotondim):
        b = np.array([(ind >> d) & 1 for d in range(3)])
        c = (2 * p + b[None, :] + 0.5) / (2 ** ilevel)        # coarse-cell units
        out.append(c)
    return ig, np.stack(out, axis=0)     # [ind][oct][3]


def fill_state(a, ilevel, fn):
    """uold(active cells of ilevel) = fn(x, y, z) -> conservative [nvar, n]; x in coarse-cell units."""
    ig, cc = cell_centers(a, ilevel)
    for ind in range(a.twotondim):
        u = fn(cc[ind][:, 0], cc[ind][:, 1], cc[ind][:, 2])
        a.uold[:, a.ncoarse + ind * a.ngridmax + ig - 1] = u


def build_nested_tree(levelmin, levelmax, half_width=8, boxlen=1.0, nvar=None, mhd=False):
    """A statically refined 3-D periodic tree (single rank): levels 1..levelmin cover the box, every level
    levelmin < l <= levelmax refines the centred cube of (2*half_width)^3 cells of level l-1 (so each fine level holds
    (2*half_width)^3 octs); half_width = (hx, hy, hz) refines a centred box of 2hx x 2hy x 2hz cells instead.  With
    every half width >= 2 every refined cell keeps its 3^3 neighbours at its own level, the rule the reference enforces
    through smooth_fine / nexpand (amr/flag_utils.f90:117-188), and a fine oct's six neighbouring father cells always
    exist.  Produces the arrays of amr/amr_commons.f90:68-79 like build_uniform_tree; oct numbering is lattice order
    level by level."""
    ndim, nx, ny, nz = 3, 1, 1, 1
    nvar = nvar or (8 if mhd else 5)
    hw = np.array(half_width if hasattr(half_width, "__len__") else (half_width,) * 3, dtype=np.int64)
    if hw.shape != (3,) or hw.min() < 2:
        raise ValueError("half_width must be >= 2")
    pos = {}
    for l in range(1, levelmax + 1):
        n = 1 << (l - 1)                                  # octs per dimension if the level were full
        if l <= levelmin:
            r = [np.arange(n)] * 3
        else:
            c = n // 2                                    # father cells at level l-1: n per dimension
            if (2 * hw > n).any():
                raise ValueError("refined box larger than the box")
            r = [np.arange(c - hw[d], c + hw[d]) for d in range(3)]
        gz, gy, gx = np.meshgrid(r[2], r[1], r[0], indexing="ij")
        pos[l] = np.stack([gx.ravel(), gy.ravel(), gz.ravel()], axis=1).astype(np.int64)
    igrid0, nxt = {}, 1
    for l in range(1, levelmax + 1):
        igrid0[l] = nxt
        nxt += len(pos[l])
    ngridmax = nxt - 1 + 8
    ncoarse = 1

    def lookup(l, p):
        n = 1 << (l - 1)
        p = np.mod(p, n)
        if l <= levelmin:
            return igrid0[l] + p[:, 0] + n * (p[:, 1] + n * p[:, 2])
        c = n // 2
        q = p - (c - hw)[None, :]
        ok = np.all((q >= 0) & (q < 2 * hw[None, :]), axis=1)
        return np.where(ok, igrid0[l] + q[:, 0] + 2 * hw[0] * (q[:, 1] + 2 * hw[1] * q[:, 2]), 0)

    a = AmrCommons(ndim, nvar, ncoarse, ngridmax, nx, ny, nz, (0, 0), (0, 0), (0, 0), nlevelmax=levelmax, boxlen=boxlen, mhd=mhd)
    for l in range(1, levelmax + 1):
        p = pos[l]
        ig = igrid0[l] + np.arange(len(p))
        if l == 1:
            fcell = np.ones(len(p), dtype=np.int64)
        else:
            par = lookup(l - 1, p >> 1)
            ind = (p[:, 0] & 1) + 2 * (p[:, 1] & 1) + 4 * (p[:, 2] & 1)
            fcell = ncoarse + ind * ngridmax + par
        a.father[ig - 1] = fcell
        a.son[fcell - 1] = ig
        for d in range(3):
            for s, sh in ((0, -1), (1, +1)):
                if l == 1:
                    nb = np.ones(len(p), dtype=np.int64)
                else:
                    q = p.copy()
                    q[:, d] += sh
                    par = lookup(l - 1, np.mod(q, 1 << (l - 1)) >> 1)
                    if (par <= 0).any():
                        raise RuntimeError("nested tree violates the 2:1 rule")
                    q = np.mod(q, 1 << (l - 1))
                    ind = (q[:, 0] & 1) + 2 * (q[:, 1] & 1) + 4 * (q[:, 2] & 1)
                    nb = ncoarse + ind * ngridmax + par
                a.nbor[2 * d + s, ig - 1] = nb
        a.active[l] = ig.astype(np.int32)
        a.boundary[l] = []
    a._pos = pos
    a._igrid0 = igrid0
    a.levelmin = levelmin
    return a


def leaf_cells(a, ilevel):
    """0-based indices (into the ncell axis) of the leaf cells of a level (son == 0)."""
    ig = a.active[ilevel].astype(np.int64)
    c = np.concatenate([a.ncoarse + ind * a.ngridmax + ig - 1 for ind in range(a.twotondim)])
    return c[a.son[c] == 0]
