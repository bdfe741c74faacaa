"""The MHD AMR kernels (ramses_b200/csrc/mhd_amr.cuh) away from the suite's one option set -- slope_mag_type apart from slope_type,
the prolongation limiters interpol_type / interpol_mag_type, reflexive walls in 1-D -- executed on the CPU by the emulated launch
(tests/host_numerics) and compared with the oracle bit for bit.  Every option value is first shown to change the oracle's result
on the same mesh and state, so that a setting dropped on its way to the kernels cannot pass unnoticed; the 1-D invariances are
asserted the other way round on purpose.  The reflexive-wall branch of the oracle is tied to a mirror property of the equations."""
import ctypes as C

import numpy as np
import pytest

from test_device_numerics_host import dev, _mhd_amr_compare_levels, _mhd3_static_run, MHD_R1D, MHD_R2D  # noqa: F401


@pytest.fixture(autouse=True)
def _default_interpol(orc):
    """orc_mhd_set_interpol sets process globals of the oracle: every test leaves them at the default (2, -1)"""
    L = orc.lib()
    L.orc_mhd_set_interpol.argtypes = [C.c_int, C.c_int]
    try:
        yield
    finally:
        L.orc_mhd_set_interpol(2, -1)


# ---- meshes ------------------------------------------------------------------------------------------------------------------
# the imhd-tube regions (tests/mhd/imhd-tube) with the two states moving, so that a wall sees flow into and out of it
IMHD_MOVING = [dict(type="square", x_center=0.75, length_x=1.5, d=1.0, u=0.6, v=0.1, w=0.0, p=1.0, A=1.0, B=1.0, C=0.0),
               dict(type="square", x_center=2.5, length_x=2.0, d=0.2, u=-0.5, v=0.0, w=0.2, p=0.2, A=1.0, B=-0.989992, C=0.141120)]


def tube_run(bound=(2, 2), riemann="hlld", slope_type=1, interpol_type=2, regions=None, max_coarse=10, **kw):
    """the refined imhd-tube mesh (NDIM=1, levelmin 5, gradient criteria) after max_coarse coarse steps; bound = (x-, x+) types"""
    from oracle.amr_mhd import MhdAmrRun
    from test_oracle_golden import IMHD
    r = MhdAmrRun(5, 9, tuple(bound) + (0, 0, 0, 0), 3.5, nsubcycle=[1, 1, 1, 1], riemann=riemann, slope_type=slope_type,
                  gamma=1.6666667, courant_factor=0.8, err_grad_d=0.01, err_grad_u=0.05, err_grad_p=0.05, interpol_type=interpol_type,
                  regions=IMHD if regions is None else regions, tout=[1e9], ngridmax=10000, **kw)
    r.run(max_coarse=max_coarse)
    return r


def ot_run(r1="hlld", r2="hlld", slope_type=2, **kw):
    """the adaptively refined Orszag-Tang vortex (NDIM=2, levels 4..6) after 6 coarse steps"""
    from oracle.amr_mhd import MhdAmrRun2D
    r = MhdAmrRun2D(4, 6, 1.0, nsubcycle=[1], riemann=r1, riemann2d=r2, slope_type=slope_type, gamma=1.6666667, courant_factor=0.8,
                    err_grad_p=0.1, tout=[1e9], nexpand=1, ngridmax=20000, **kw)
    r.run(max_coarse=6)
    return r


def _finest_godunov(orc, r, pm=None, interpol=None):
    """the oracle's godunov_fine of the finest populated level of r on r's state (whole unew: own and refluxed cells), with the
    parameters pm (default r.pm) and the prolongation limiters interpol = (interpol_type, interpol_mag_type) (default r's)"""
    L = orc.lib()
    fn = {1: L.orc_mhd1_godunov_fine, 2: L.orc_mhd2_godunov_fine, 3: L.orc_mhd3_godunov_fine}[r.ndim]
    l = max(k for k in range(1, r.nlevelmax + 1) if len(r.active[k]))
    assert l > r.levelmin
    unew = np.zeros_like(r.uold)
    L.orc_mhdn_set_unew(r.mp, l - 1, orc.dptr(r.uold), orc.dptr(unew))
    L.orc_mhdn_set_unew(r.mp, l, orc.dptr(r.uold), orc.dptr(unew))
    it, mt = interpol if interpol is not None else (r.interpol_type, r.interpol_mag_type)
    L.orc_mhd_set_interpol(it, mt)
    dt = 0.25 * r.dtnew[r.levelmin] / 2 ** (l - r.levelmin)
    fn(C.byref(pm if pm is not None else r.pm), r.mp, l, r.levelmin, r.nvector, dt, orc.dptr(r.uold), orc.dptr(unew))
    return unew


def _with_slope_mag(orc, pm, smt):
    p = orc.make_mhd_params(slope_type=pm.slope_type, slope_mag_type=smt, riemann=pm.riemann, riemann2d=pm.riemann2d, gamma=pm.gamma,
                            smallr=pm.smallr, smallc=pm.smallc, slope_theta=pm.slope_theta, courant_factor=pm.courant_factor,
                            boxlen=pm.boxlen)
    return p


# ---- slope_mag_type apart from slope_type ----------------------------------------------------------------------------------
SLOPE_PAIRS = [(0, 1), (0, 2), (1, 0), (1, 2), (2, 0), (2, 1)]


@pytest.mark.parametrize("slope_type,slope_mag_type", SLOPE_PAIRS)
@pytest.mark.parametrize("r1,r2", [("hlld", "hlld"), ("roe", "llf"), ("llf", "roe")])
def test_mhd_amr_2d_slope_mag_type_emulated_equals_oracle(orc, dev, r1, r2, slope_type, slope_mag_type):
    """NDIM=2 Orszag-Tang with a face-field limiter (slope_mag_type, mhd/umuscl.f90:2333) other than the cell one: the face
    slopes of mhd_amr2_godfine_kernel (mhd_amr.cuh, the P.slope_mag_type branch) equal mhd2_godfine1 of the oracle on every level
    -- unew incl. the refluxed coarse cells, upload_fine, cmpdt.  The oracle itself gives a different unew with slope_mag_type =
    slope_type on the same mesh and state."""
    r = ot_run(r1, r2, slope_type, slope_mag_type=slope_mag_type)
    assert r.pm.slope_mag_type == slope_mag_type
    same = _finest_godunov(orc, r, _with_slope_mag(orc, r.pm, slope_type))
    assert not np.array_equal(_finest_godunov(orc, r), same)
    L = orc.lib()
    nlev, nrefl, moved = _mhd_amr_compare_levels(orc, dev, r, 2, r1, r2, slope_type, 2, L.orc_mhd2_godunov_fine, L.orc_mhdn_upload_fine,
                                                 L.orc_mhdn_courant_fine, slope_mag_type=slope_mag_type)
    assert nlev >= 3 and nrefl > 0 and moved > 1e-6


@pytest.mark.parametrize("slope_type,slope_mag_type,r1,r2", [(0, 1, "hlld", "hlld"), (0, 2, "roe", "llf"), (1, 0, "llf", "roe"),
                                                             (1, 2, "hlld", "hlld"), (2, 0, "hll", "hlla"), (2, 1, "roe", "llf")])
def test_mhd_amr_3d_slope_mag_type_emulated_equals_oracle(orc, dev, slope_type, slope_mag_type, r1, r2):
    """NDIM=3 nested mesh (64 octs per level, fully 3-D divergence-free field): the face slopes of mhd_amr3_godfine_kernel with
    slope_mag_type != slope_type equal mhd3_godfine1 on every level; the oracle differs from slope_mag_type = slope_type."""
    r = _mhd3_static_run(r1, r2, slope_type)
    r.pm = _with_slope_mag(orc, r.pm, slope_mag_type)
    same = _finest_godunov(orc, r, _with_slope_mag(orc, r.pm, slope_type))
    assert not np.array_equal(_finest_godunov(orc, r), same)
    L = orc.lib()
    nlev, nrefl, moved = _mhd_amr_compare_levels(orc, dev, r, 3, r1, r2, slope_type, 2, L.orc_mhd3_godunov_fine, L.orc_mhdn_upload_fine,
                                                 L.orc_mhdn_courant_fine, slope_mag_type=slope_mag_type)
    assert nlev == 3 and nrefl > 0 and moved > 1e-6


@pytest.mark.parametrize("slope_type", [0, 1, 2])
def test_mhd_amr_1d_slope_mag_type_makes_no_difference(orc, dev, slope_type):
    """NDIM=1: the reference's uslope (mhd/umuscl.f90:2226-2252, the NDIM==1 branch) limits the cell-centred variables with
    slope_type and never reads slope_mag_type -- B_x is one constant in 1-D and has no transverse slope.  The oracle and the
    emulated mhd_amr1_godfine_kernel both give the same bits for every slope_mag_type, and equal each other."""
    r = tube_run(slope_type=slope_type, max_coarse=8)
    ref = _finest_godunov(orc, r)
    L = orc.lib()
    for smt in (0, 1, 2):
        assert np.array_equal(_finest_godunov(orc, r, _with_slope_mag(orc, r.pm, smt)), ref)
        nlev, nrefl, moved = _mhd_amr_compare_levels(orc, dev, r, 1, "hlld", "llf", slope_type, 2, L.orc_mhd1_godunov_fine,
                                                     L.orc_mhd1_upload_fine, L.orc_mhd1_courant_fine, slope_mag_type=smt)
        assert nlev >= 3 and moved > 1e-6


# ---- the prolongation limiters: each value changes the oracle's result on the meshes the GPU tests run ------------------------
@pytest.fixture(scope="module")
def option_meshes(orc):
    return {1: tube_run(), 2: ot_run(interpol_type=2), 3: _mhd3_static_run("hlld", "hlld", 2)}


# (ndim, interpol_type, interpol_mag_type) of tests/test_gpu_mhd_amr_options.py
INTERPOL_CASES = [(2, 0, -1), (2, 1, -1), (2, 3, -1), (2, 2, 0), (2, 2, 1), (2, 2, 3), (2, 0, 3), (2, 1, 2), (2, 3, 0),
                  (3, 0, -1), (3, 1, -1), (3, 3, -1), (3, 2, 0), (3, 2, 1), (3, 2, 3), (3, 1, 2), (3, 3, 1)]


@pytest.mark.parametrize("ndim,itype,mtype", INTERPOL_CASES)
def test_mhd_amr_prolongation_limiter_changes_the_oracle(orc, option_meshes, ndim, itype, mtype):
    """interpol_type / interpol_mag_type reach the ghost-oct prolongation of the oracle's godfine1: on the imhd-tube, Orszag-Tang
    and nested 3-D meshes (the GPU tests run these problems at other solver pairs and step counts, and repeat the check on their
    own states), the finest level's unew differs from the one with the default limiters (2, -1)"""
    r = option_meshes[ndim]
    assert not np.array_equal(_finest_godunov(orc, r, interpol=(itype, mtype)), _finest_godunov(orc, r, interpol=(2, -1)))


@pytest.mark.parametrize("itype", [0, 1, 3])
def test_mhd_amr_1d_interpol_type_changes_the_oracle_and_interpol_mag_type_does_not(orc, option_meshes, itype):
    """NDIM=1: the ghost cells come from interpol_hydro alone (mhd1_interpol_cell reads interpol_type only); interpol_type changes
    the oracle's unew, interpol_mag_type does not"""
    r = option_meshes[1]
    got = _finest_godunov(orc, r, interpol=(itype, -1))
    assert not np.array_equal(got, _finest_godunov(orc, r, interpol=(2, -1)))
    for mt in (0, 1, 2, 3):
        assert np.array_equal(_finest_godunov(orc, r, interpol=(itype, mt)), got)


# ---- reflexive walls in 1-D ---------------------------------------------------------------------------------------------------
def _cell_x(r, l):
    """(cells, x): 1-based cell indices of the active cells of level l and their centres in box coordinates"""
    dx = 0.5 ** l
    scale = r.p.boxlen / (r.m.icoarse_max - r.m.icoarse_min + 1)
    ig = np.asarray(r.active[l], dtype=np.int64)
    cells = np.concatenate([r.ncoarse + ind * r.ngridmax + ig for ind in range(2)])
    x = np.concatenate([(r.xg[0, ig] + (ind - 0.5) * dx - r.m.icoarse_min) * scale for ind in range(2)])
    return cells, x


def _mirror_state(s, Lh, gamma, bx=0.0):
    """conservative MHD state at positions s: v_x odd, every other primitive even about s = 0 and s = Lh (period 2 Lh)"""
    k = np.pi * s / Lh
    d = 1.0 + 0.3 * np.cos(k) + 0.1 * np.cos(2 * k)
    vx, vy, vz = 0.5 * np.sin(k) + 0.2 * np.sin(2 * k), 0.2 * np.cos(k), 0.1 + 0.05 * np.cos(3 * k)
    P = 1.0 + 0.2 * np.cos(2 * k) + 0.1 * np.cos(k)
    By, Bz = 0.8 + 0.3 * np.cos(k), 0.2 * np.cos(2 * k)
    u = np.zeros((11, len(s)))
    u[0] = d
    u[1], u[2], u[3] = d * vx, d * vy, d * vz
    u[4] = 0.5 * d * (vx ** 2 + vy ** 2 + vz ** 2) + P / (gamma - 1.0) + 0.5 * (bx ** 2 + By ** 2 + Bz ** 2)
    u[5], u[6], u[7] = bx, By, Bz
    u[8], u[9], u[10] = bx, By, Bz
    return u


def _mirror_run(bound, levelmin, levelmax, boxlen, shift, widths, bx=0.0, nsubcycle=(2, 2, 2)):
    """MhdAmrRun with the statically nested mesh |x - shift| < widths[level - levelmin] and the state _mirror_state(x - shift)"""
    from oracle.amr_mhd import MhdAmrRun
    Lh = 1.0

    class Run(MhdAmrRun):
        def smooth_fine(self, l):
            pass

        def hydro_flag(self, l):
            if l == self.nlevelmax or self.numbtot(l) == 0:
                return
            cells, x = _cell_x(self, l)
            w = widths[l - self.levelmin] if l - self.levelmin < len(widths) else 0.0
            self.flag1[cells[np.abs(x - shift) < w]] = 1

        def init_flow_fine(self, l):
            if self.numbtot(l) == 0:
                return
            cells, x = _cell_x(self, l)
            self.uold.reshape(11, self.ncell)[:, cells - 1] = _mirror_state(x - shift, Lh, self.p.gamma, bx)

    r = Run(levelmin, levelmax, tuple(bound) + (0, 0, 0, 0), boxlen, nsubcycle=list(nsubcycle), riemann="hlld", slope_type=2,
            gamma=1.6666667, courant_factor=0.8, err_grad_d=0.01, interpol_type=2, tout=[1e9], ngridmax=4000)
    r.flag_coarse(); r.init_refine(); r.init_refine_2()
    r.static = True
    return r


def _level_states(r, shift):
    """{(level, round(x / dx)): state column} of every active cell, x measured from `shift`"""
    U = r.uold.reshape(11, r.ncell)
    out = {}
    for l in range(1, r.nlevelmax + 1):
        if len(r.active[l]) == 0:
            continue
        cells, x = _cell_x(r, l)
        dx = r.p.boxlen / (r.m.icoarse_max - r.m.icoarse_min + 1) * 0.5 ** l
        for c, xx in zip(cells, x):
            out[(l, int(np.floor((xx - shift) / dx)))] = U[:, c - 1]
    return out


@pytest.mark.parametrize("nested", [False, True])
def test_mhd_amr_1d_reflexive_walls_mirror_property(orc, nested):
    """The oracle's reflexive branch of make_boundary_hydro (NDIM=1, mhd/hydro_boundary.f90: v_x flipped, the other variables
    mirrored, B_x = 2 B_wall - B_mirror) against the symmetry of the equations: a run on [0, 1] between two reflexive walls equals
    the [0, 1] half of a periodic run on [-1, 1] whose state is the mirrored one (v_x odd, every other primitive even about 0 and
    1; B_x = 0), on a uniform level and on a static nested mesh refined next to the wall at x = 0, over 3 coarse steps, to
    round-off.  The same run between outflow boundaries does not have the property."""
    lmin, lmax = (5, 7) if nested else (6, 6)
    widths = (0.3, 0.15)                              # refined bands next to x = 0 (oct-aligned at levels 5 and 6)
    wall = _mirror_run((1, 1), lmin, lmax, 1.0, 0.0, widths)
    per = _mirror_run((0, 0), lmin + 1, lmax + 1, 2.0, 1.0, widths)
    out = _mirror_run((2, 2), lmin, lmax, 1.0, 0.0, widths)
    assert [len(wall.active[l]) for l in range(1, lmax + 1)] == [len(out.active[l]) for l in range(1, lmax + 1)]
    for r in (wall, per, out):
        for _ in range(3):
            r.amr_step(r.levelmin, 1)
            r.nstep_coarse += 1
    sw, so = _level_states(wall, 0.0), _level_states(out, 0.0)
    sp = {(l - 1, i): v for (l, i), v in _level_states(per, 1.0).items()}
    assert sorted(sw) == sorted(so)
    assert all(k in sp for k in sw)
    if nested:
        assert len({l for l, _ in sw if l >= wall.levelmin}) == 3
    got = np.array([sw[k] for k in sorted(sw)]).T
    exp = np.array([sp[k] for k in sorted(sw)]).T
    flow = np.array([so[k] for k in sorted(sw)]).T
    scale = np.abs(exp).max(axis=1, keepdims=True) + 1e-300
    assert np.abs(exp[1]).max() > 0.1
    assert (np.abs(got - exp) <= 1e-13 * scale).all(), float((np.abs(got - exp) / scale).max())
    assert (np.abs(flow - exp) / scale).max() > 1e-3
    assert np.isclose(wall.t, per.t, rtol=1e-13, atol=0) and wall.t > 0


def _scramble_and_perturb(r, seed):
    """boundary octs of every level set to 9, B_x of every interior face perturbed (B_x varying, so that the reflexive
    B_x = 2 B_wall - B_mirror lines are distinguishable from a copy)"""
    U = r.uold.reshape(11, r.ncell)
    rng = np.random.default_rng(seed)
    for l in range(1, r.nlevelmax + 1):
        if len(r.active[l]):
            cells, _ = _cell_x(r, l)
            U[5, cells - 1] += 0.01 * rng.standard_normal(len(cells))
            U[8, cells - 1] += 0.01 * rng.standard_normal(len(cells))
        for b in range(r.m.nboundary):
            for ig in r.bound[b][l]:
                for ind in range(2):
                    U[:, r.cell(ind, ig) - 1] = 9.0


@pytest.mark.parametrize("bound", [(1, 1), (1, 2), (2, 1)])
def test_mhd_amr_1d_reflexive_boundary_kernel_emulated_equals_oracle(orc, dev, bound):
    """NDIM=1 reflexive walls (bound = (x-, x+) types, 1 reflexive, 2 outflow: both dir tables of mhd_amr1_boundary_kernel) on the
    refined imhd-tube mesh with moving states and B_x = 1: every level's godunov_fine, upload_fine, cmpdt and make_boundary_hydro of the
    emulated kernels equal the oracle's bit for bit; then the boundary pass alone on a state whose B_x varies from face to face,
    boundary octs scrambled first, and the result differs from the outflow pass on the same state."""
    r = tube_run(bound=bound, regions=IMHD_MOVING, max_coarse=8)
    assert any(len(r.bound[b][l]) for b in range(r.m.nboundary) for l in range(r.levelmin + 1, r.nlevelmax + 1))
    L = orc.lib()
    nlev, nrefl, moved = _mhd_amr_compare_levels(orc, dev, r, 1, "hlld", "llf", 1, 2, L.orc_mhd1_godunov_fine, L.orc_mhd1_upload_fine,
                                                 L.orc_mhd1_courant_fine, boundary=L.orc_mhd1_make_boundary_hydro)
    assert nlev >= 3 and moved > 1e-6
    son = np.ascontiguousarray(r.son[1:], dtype=np.int32)
    father = np.ascontiguousarray(r.father[1:], dtype=np.int32)
    nbor = np.ascontiguousarray(r.nbor[:, 1:], dtype=np.int32)
    m = r.m
    tree = (1, r.ncoarse, r.ngridmax, m.nx, m.ny, m.nz, orc.iptr(son), orc.iptr(father), orc.iptr(nbor))
    _scramble_and_perturb(r, 7)
    nb = 0
    for l in range(r.levelmin, r.nlevelmax + 1):
        u_o, u_k = r.uold.copy(), r.uold.copy()
        L.orc_mhd1_make_boundary_hydro(C.byref(r.pm), r.mp, l, orc.dptr(u_o))
        for b in range(m.nboundary):
            lst = np.ascontiguousarray(r.bound[b][l], dtype=np.int32)
            if len(lst) == 0:
                continue
            bt = m.boundary_type[b]
            dev.devnum_mhd_amr_pass(1, *tree, orc.iptr(lst), len(lst), orc.dptr(u_k), r.pm.gamma, r.pm.smallr, r.pm.smallc,
                                    r.pm.courant_factor, 0.5 ** l, bt % 10, bt // 10, None)
            if bt // 10 == 0:
                nb += len(lst)
                u_f = u_o.copy()
                dev.devnum_mhd_amr_pass(1, *tree, orc.iptr(lst), len(lst), orc.dptr(u_f), r.pm.gamma, r.pm.smallr, r.pm.smallc,
                                        r.pm.courant_factor, 0.5 ** l, bt % 10, 1, None)
                assert not np.array_equal(u_f, u_o), (l, b)      # outflow on the same octs gives other values
        assert np.array_equal(u_k, u_o), (l, np.abs(u_k - u_o).max())
    assert nb > 0
