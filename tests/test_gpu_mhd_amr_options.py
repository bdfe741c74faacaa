"""The MHD AMR kernels on the GPU through the C-ABI away from the suite's one option set: the prolongation limiters
(rgpu_set_amr interpol_type, rgpu_set_interpol_mag), slope_mag_type apart from slope_type, reflexive walls in 1-D -- host-driven
amr_step order and the device-resident stepper (rgpu_amr_steps), bit for bit against the oracle's amr_step.  Before stepping,
each case shows on the oracle, on the same mesh and state, that its option changes the result (tests/test_mhd_amr_options_host.py
holds the same checks on the CPU)."""
import ctypes as C

import numpy as np
import pytest

from ramses_b200.hydro import HydroGPU, amr_step
from test_gpu_mhd import _mhd_commons_from_run
from test_mhd_amr_options_host import IMHD_MOVING, _finest_godunov, _with_slope_mag, ot_run, tube_run
from test_device_numerics_host import _mhd3_static_run

pytestmark = pytest.mark.gpu

RGPU_EINVAL, RGPU_EUNSUPPORTED = -1, -3        # include/ramses_gpu.h


@pytest.fixture(autouse=True)
def _default_interpol(orc):
    """the oracle's prolongation limiters are process globals: every test leaves them at the default (2, -1)"""
    L = orc.lib()
    L.orc_mhd_set_interpol.argtypes = [C.c_int, C.c_int]
    try:
        yield
    finally:
        L.orc_mhd_set_interpol(2, -1)


def _freeze(r, regrid=True):
    """regrid once more like the head of amr_step, then keep the mesh (test_gpu_mhd._mhd_amr_gpu_vs_oracle)"""
    for i in range(r.levelmin, r.nlevelmax + 1 if regrid else r.levelmin):
        if i > r.levelmin:
            r.make_boundary_hydro(i)
        r.refine_fine(i)
    r.static = True


def _gpu_steps(r, ndim, riemann, riemann2d, slope_type, ncoarse, resident, interpol, mag_after=None):
    """ncoarse coarse steps of the frozen mesh of r on the device (r is only read); interpol = (interpol_type, interpol_mag_type).
    mag_after: resident only -- one rgpu_amr_steps call of 2 coarse steps (the first runs eagerly, the second is captured as a
    graph), then rgpu_set_interpol_mag(mag_after) and one call with the remaining steps (its second step replays the graph)."""
    levelmax, levelmin = r.nlevelmax, r.levelmin
    a = _mhd_commons_from_run(r, ndim, riemann, riemann2d, slope_type)
    h = HydroGPU(a, amr_mode=True, interpol_type=interpol[0], interpol_mag_type=interpol[1])
    for l in range(1, levelmax + 1):
        if len(a.active[l]):
            h.bind_level(l)
    h.upload_state(0)
    for l in range(1, levelmax + 1):
        if len(a.active[l]):
            h.make_boundary_hydro(l)
    nsub = [0] + [r.nsubcycle[l] for l in range(1, levelmax + 1)] + [2] * 8
    if resident:
        a.numbtot = {l: len(a.active[l]) for l in range(1, levelmax + 1)}
        if mag_after is None:
            dts = list(h.amr_steps(levelmin, nsub, ncoarse))
        else:
            assert ncoarse >= 4
            dts = list(h.amr_steps(levelmin, nsub, 2))
            h.set_interpol_mag(mag_after)
            dts += list(h.amr_steps(levelmin, nsub, ncoarse - 2))
    else:
        dtnew = {l: r.dtnew[l] for l in range(0, levelmax + 2)}
        dtold = {l: r.dtold[l] for l in range(0, levelmax + 2)}
        dts = []
        for _ in range(ncoarse):
            amr_step(h, levelmin, 1, levelmin, nsub, dtnew, dtold)
            dts.append(dtnew[levelmin])
    h.download_state(0)
    h.finalize()
    return a.uold.copy(), np.array(dts)


def _oracle_steps(r, ncoarse, mag_after=None):
    for l in range(1, r.nlevelmax + 1):
        r.make_boundary_hydro(l)
    dts = []
    for k in range(ncoarse):
        if k == 2 and mag_after is not None:
            r.interpol_mag_type = mag_after
        r.amr_step(r.levelmin, 1)
        dts.append(r.dtnew[r.levelmin])
    return r.uold.reshape(11, -1).copy(), np.array(dts)


def _active_cells(r):
    return np.concatenate([[r.cell(ind, ig) - 1 for ig in r.active[l] for ind in range(r.T)]
                           for l in range(1, r.nlevelmax + 1) if r.active[l]]).astype(np.int64)


def _assert_equal(r, got, dts, ref, dts_ref, whole=False):
    cells = _active_cells(r)
    assert np.array_equal(dts, dts_ref), (dts, dts_ref)
    assert np.isfinite(got[:, cells]).all()
    assert np.array_equal(got[:, cells], ref[:, cells]), float(np.abs(got[:, cells] - ref[:, cells]).max())
    if whole:
        assert np.array_equal(got, ref)


def _mesh(ndim, r1, r2, slope_type, **kw):
    """the meshes of tests/test_gpu_mhd.py: imhd-tube (1-D), Orszag-Tang (2-D), the nested 3-D cube; returns (run, regrid)"""
    if ndim == 1:
        return tube_run(riemann=r1, slope_type=slope_type, max_coarse=12, **kw), True
    if ndim == 2:
        return ot_run(r1, r2, slope_type, **kw), True
    r = _mhd3_static_run(r1, r2, slope_type)
    return r, False


# ---- prolongation limiters through the C-ABI ----------------------------------------------------------------------------------
@pytest.mark.parametrize("resident", [False, True])
@pytest.mark.parametrize("ndim,itype,mtype", [(2, 0, -1), (2, 1, -1), (2, 3, -1), (2, 2, 0), (2, 2, 1), (2, 2, 3), (2, 0, 3), (2, 1, 2),
                                              (2, 3, 0), (3, 0, -1), (3, 1, -1), (3, 3, -1), (3, 2, 0), (3, 2, 3), (3, 1, 2), (3, 3, 1)])
def test_mhd_amr_prolongation_limiters_bitwise(orc, ndim, itype, mtype, resident):
    """interpol_type (rgpu_set_amr) and interpol_mag_type (rgpu_set_interpol_mag; -1 = interpol_type) reach the ghost-oct
    prolongation of mhd_amr{2,3}_godfine_kernel: 2 coarse steps of the Orszag-Tang / nested 3-D mesh == the oracle with the same
    limiters, bit for bit.  The oracle differs from the default limiters (2, -1) on the same mesh and state."""
    r1, r2, st = ("hlld", "hlld", 2) if ndim == 2 else ("roe", "llf", 1)
    r, regrid = _mesh(ndim, r1, r2, st)
    _freeze(r, regrid)
    r.interpol_type, r.interpol_mag_type = itype, mtype
    assert not np.array_equal(_finest_godunov(orc, r), _finest_godunov(orc, r, interpol=(2, -1)))
    got, dts = _gpu_steps(r, ndim, r1, r2, st, 2, resident, (itype, mtype))
    ref, dts_ref = _oracle_steps(r, 2)
    _assert_equal(r, got, dts, ref, dts_ref)


@pytest.mark.parametrize("resident", [False, True])
@pytest.mark.parametrize("itype", [0, 1, 3])
def test_mhd_amr_1d_prolongation_interpol_mag_type_invariant(orc, itype, resident):
    """NDIM=1: mhd1_interpol_cell reads interpol_type only, so the device state is the same bits for every interpol_mag_type
    (-1, 0..3), and equals the oracle's; interpol_type itself changes the oracle's result on the same mesh"""
    r, _ = _mesh(1, "hlld", "llf", 1, interpol_type=itype)
    _freeze(r)
    assert not np.array_equal(_finest_godunov(orc, r), _finest_godunov(orc, r, interpol=(2, -1)))
    runs = [_gpu_steps(r, 1, "hlld", "llf", 1, 3, resident, (itype, mt)) for mt in (-1, 0, 1, 2, 3)]
    for got, dts in runs[1:]:
        assert np.array_equal(got, runs[0][0]) and np.array_equal(dts, runs[0][1])
    ref, dts_ref = _oracle_steps(r, 3)
    _assert_equal(r, runs[0][0], runs[0][1], ref, dts_ref)


@pytest.mark.parametrize("ndim,m0,m1", [(2, 0, 3), (3, 3, 1)])
def test_mhd_amr_set_interpol_mag_drops_the_captured_graph(orc, ndim, m0, m1):
    """rgpu_amr_steps runs the first coarse step of a call eagerly, captures the second as a CUDA graph and replays it for the
    rest, also in later calls.  A first call of 2 steps captures the graph with the limiter m0; rgpu_set_interpol_mag(m1) must drop
    it, so that the second call of 2 steps -- whose second step would replay a graph still held -- runs with m1 throughout:
    4 coarse steps == the oracle switching from m0 to m1 after two steps"""
    r1, r2, st = ("hlld", "hlld", 2) if ndim == 2 else ("roe", "llf", 1)
    r, regrid = _mesh(ndim, r1, r2, st)
    _freeze(r, regrid)
    r.interpol_mag_type = m0
    for m in (m0, m1):
        assert not np.array_equal(_finest_godunov(orc, r, interpol=(2, m)), _finest_godunov(orc, r, interpol=(2, -1)))
    got, dts = _gpu_steps(r, ndim, r1, r2, st, 4, True, (2, m0), mag_after=m1)
    ref, dts_ref = _oracle_steps(r, 4, mag_after=m1)
    _assert_equal(r, got, dts, ref, dts_ref)


def test_mhd_amr_prolongation_limiter_rejections(orc):
    """rgpu_set_interpol_mag accepts -1..3 only.  rgpu_set_amr refuses interpol_type 4 with interpol_var 0 in any build (the type
    is designed for interpol_var 2); in the MHD build interpol_var 0 is the only value accepted, so interpol_type 4 cannot be set"""
    from ramses_b200 import lib as _l
    r = ot_run()
    a = _mhd_commons_from_run(r, 2, "hlld", "hlld", 2)
    h = HydroGPU(a, amr_mode=True, interpol_type=2)
    try:
        for bad in (4, -2):
            with pytest.raises(_l.RgpuError) as e:
                h.set_interpol_mag(bad)
            assert e.value.code == RGPU_EINVAL and f"interpol_mag_type={bad}" in str(e.value)
        for ok in (-1, 0, 3):
            h.set_interpol_mag(ok)
        rc = h.L.rgpu_set_amr(1, 4, 0)
        assert rc == RGPU_EINVAL and "interpol_type=4" in h.L.rgpu_last_error().decode()
    finally:
        h.finalize()


# ---- slope_mag_type apart from slope_type -----------------------------------------------------------------------------------
@pytest.mark.parametrize("resident", [False, True])
@pytest.mark.parametrize("ndim,slope_type,slope_mag_type,r1,r2", [
    (2, 0, 1, "hlld", "hlld"), (2, 0, 2, "roe", "llf"), (2, 1, 0, "llf", "roe"), (2, 1, 2, "hlld", "hlld"), (2, 2, 0, "hll", "hlla"),
    (2, 2, 1, "roe", "llf"), (3, 0, 1, "hlld", "hlld"), (3, 0, 2, "roe", "llf"), (3, 1, 0, "llf", "roe"), (3, 1, 2, "hlld", "hlld"),
    (3, 2, 0, "hll", "hlla"), (3, 2, 1, "roe", "llf")])
def test_mhd_amr_slope_mag_type_bitwise(orc, ndim, slope_type, slope_mag_type, r1, r2, resident):
    """slope_mag_type (rgpu_params) other than slope_type reaches the face slopes of mhd_amr{2,3}_godfine_kernel: 2 coarse steps
    == the oracle with the same pair, bit for bit; the oracle differs from slope_mag_type = slope_type on the same mesh and state"""
    r, regrid = _mesh(ndim, r1, r2, slope_type)
    _freeze(r, regrid)
    r.pm = _with_slope_mag(orc, r.pm, slope_mag_type)
    assert not np.array_equal(_finest_godunov(orc, r), _finest_godunov(orc, r, _with_slope_mag(orc, r.pm, slope_type)))
    got, dts = _gpu_steps(r, ndim, r1, r2, slope_type, 2, resident, (2, -1))
    ref, dts_ref = _oracle_steps(r, 2)
    _assert_equal(r, got, dts, ref, dts_ref)


@pytest.mark.parametrize("resident", [False, True])
def test_mhd_amr_1d_slope_mag_type_invariant(orc, resident):
    """NDIM=1: uslope (mhd/umuscl.f90:2226-2252) never reads slope_mag_type; the device state is the same bits for 0, 1, 2 and
    equals the oracle's"""
    r, _ = _mesh(1, "hlld", "llf", 1)
    _freeze(r)
    runs = []
    for smt in (0, 1, 2):
        pm = r.pm
        r.pm = _with_slope_mag(orc, pm, smt)
        runs.append(_gpu_steps(r, 1, "hlld", "llf", 1, 3, resident, (2, -1)))
        r.pm = pm
    for got, dts in runs[1:]:
        assert np.array_equal(got, runs[0][0]) and np.array_equal(dts, runs[0][1])
    ref, dts_ref = _oracle_steps(r, 3)
    _assert_equal(r, runs[0][0], runs[0][1], ref, dts_ref)


# ---- reflexive walls in 1-D -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("resident", [False, True])
@pytest.mark.parametrize("bound", [(1, 1), (1, 2), (2, 1)])
def test_mhd_amr_1d_reflexive_walls_bitwise(orc, bound, resident):
    """NDIM=1 reflexive walls (mhd_amr1_boundary_kernel; bound = (x-, x+) types, 1 reflexive, 2 outflow) on the refined imhd-tube mesh with moving
    states and B_x = 1: 3 coarse steps == the oracle, every cell of uold (boundary octs included) bit for bit; the same mesh
    and state, from a fresh run, between outflow boundaries gives another state in the oracle"""
    r = tube_run(bound=bound, regions=IMHD_MOVING, max_coarse=12)
    _freeze(r)
    assert any(len(r.bound[b][l]) for b in range(r.m.nboundary) for l in range(r.levelmin + 1, r.nlevelmax + 1))
    u0, t0, son0 = r.uold.copy(), r.t, r.son.copy()
    got, dts = _gpu_steps(r, 1, "hlld", "llf", 1, 3, resident, (2, -1))
    ref, dts_ref = _oracle_steps(r, 3)
    _assert_equal(r, got, dts, ref, dts_ref, whole=True)
    f = tube_run(bound=bound, regions=IMHD_MOVING, max_coarse=12)        # the same mesh, state, time and dt history
    _freeze(f)
    assert np.array_equal(f.son, son0) and np.array_equal(f.uold, u0) and f.t == t0
    for b in range(f.m.nboundary):
        f.m.boundary_type[b] = 10 + f.m.boundary_type[b] % 10     # the same faces as outflow (bound_type 2)
    out, _ = _oracle_steps(f, 3)
    assert not np.array_equal(out[:, _active_cells(r)], ref[:, _active_cells(r)])


# ---- several coarse cells, non-cubic patches, more octs per level than SMs ------------------------------------------------------
def _potential_state(a, l, ndim, period, gamma=1.6666667):
    """conservative state of the active cells of level l (coordinates in coarse-cell units = box units): smooth, periodic with
    `period` per axis, and the face fields B = B0 + curl A as face averages (Stokes: the flux through a face is the circulation of
    A = (A_x(y, z), 0, A_z(x, y)) round its edges), so that the discrete div B vanishes to round-off on every level"""
    from ramses_b200.tree import cell_centers
    ig, cc = cell_centers(a, l)
    h = 0.5 ** l
    kx, ky, kz = (2 * np.pi / p for p in period)
    Az = lambda x, y: 0.3 * np.sin(kx * x) * np.sin(ky * y) + 0.2 * np.cos(kx * x + ky * y)
    Ax = (lambda y, z: 0.25 * np.cos(ky * y) * np.sin(kz * z)) if ndim == 3 else (lambda y, z: 0.0 * y)
    for ind in range(1 << ndim):
        x, y, z = cc[ind][:, 0], cc[ind][:, 1], cc[ind][:, 2] if ndim == 3 else 0.0 * cc[ind][:, 0]
        bx = [(Az(xf, y + h / 2) - Az(xf, y - h / 2)) / h + 0.4 for xf in (x - h / 2, x + h / 2)]
        by = [(Ax(yf, z + h / 2) - Ax(yf, z - h / 2)) / h - (Az(x + h / 2, yf) - Az(x - h / 2, yf)) / h - 0.3
              for yf in (y - h / 2, y + h / 2)]
        bz = [-(Ax(y + h / 2, zf) - Ax(y - h / 2, zf)) / h + 0.2 for zf in (z - h / 2, z + h / 2)]
        if ndim == 1:
            bx = [np.full_like(x, 0.7)] * 2
            by = [0.5 * np.cos(kx * x)] * 2
            bz = [0.2 + 0.3 * np.sin(kx * x)] * 2
        d = 1.0 + 0.2 * np.sin(kx * x) * np.cos(ky * y) + 0.1 * np.sin(kz * z)
        v = (0.3 * np.sin(ky * y) + 0.1 * np.cos(kx * x), -0.2 * np.cos(kx * x), 0.1 * np.sin(kx * x + kz * z))
        P = 1.0 + 0.1 * np.cos(kx * x) + 0.05 * np.sin(ky * y)
        u = np.zeros((11, len(x)))
        u[0] = d
        for k in range(3):
            u[1 + k] = d * v[k]
        u[5], u[6], u[7], u[8], u[9], u[10] = bx[0], by[0], bz[0], bx[1], by[1], bz[1]
        u[4] = P / (gamma - 1.0) + 0.5 * d * sum(vk * vk for vk in v) + 0.125 * sum((u[5 + k] + u[8 + k]) ** 2 for k in range(3))
        a.uold[:, a.ncoarse + ind * a.ngridmax + ig - 1] = u


def _oracle_on_tree(a, ndim, levelmin, levelmax, boxlen, coarse, nsubcycle, r1, r2, slope_type):
    """the oracle's MHD AMR driver on the tree and state of `a` (frozen mesh)"""
    from oracle.amr_mhd import MhdAmrRun, MhdAmrRun2D, MhdAmrRun3D
    kw = dict(riemann=r1, slope_type=slope_type, gamma=1.6666667, courant_factor=0.8, tout=[1e9], ngridmax=a.ngridmax, coarse=coarse)
    if ndim == 1:
        r = MhdAmrRun(levelmin, levelmax, (0,) * 6, boxlen, nsubcycle, **kw)
    else:
        r = (MhdAmrRun2D if ndim == 2 else MhdAmrRun3D)(levelmin, levelmax, boxlen, nsubcycle, riemann2d=r2, nexpand=1, **kw)
    assert r.ncell == a.ncell
    r.son[1:] = a.son; r.father[1:] = a.father; r.nbor[:, 1:] = a.nbor
    for l in range(1, levelmax + 1):
        r.active[l] = [int(g) for g in a.active[l]]
    r.push_all()
    r.uold[:] = a.uold.ravel()
    r.static = True
    return r


def _divb(u, cells, ndim):
    return np.abs(sum(u[8 + k, cells] - u[5 + k, cells] for k in range(ndim))).max()


@pytest.mark.parametrize("ndim,coarse,level,r1,r2,slope_type", [
    (1, (3, 1, 1), 1, "hlld", "llf", 1), (2, (3, 2, 1), 1, "hlld", "hlld", 2), (2, (3, 2, 1), 1, "llf", "roe", 1),
    (3, (3, 2, 1), 1, "hlld", "hlld", 2), (3, (3, 2, 1), 2, "roe", "llf", 1), (3, (3, 2, 1), 2, "llf", "roe", 2)])
def test_mhd_amr_mode_uniform_box_of_several_coarse_cells(orc, ndim, coarse, level, r1, r2, slope_type):
    """AMR mode on a uniform periodic domain of several coarse cells per axis refined to `level`: the neighbour and father walks
    of the MHD oct kernels decode coarse cells through nx, ny, nz at levels 1 and 2 (ramses_b200.tree.build_uniform_tree
    fabricates 1-D and 2-D domains of several coarse cells at level 1 only).  3 level steps in amr_step order (host-driven
    and rgpu_amr_steps) == the oracle's mhd{1,2,3}_godunov_fine on the same arrays, bit for bit; the field is the face average of
    a vector potential and div B stays at round-off on the device state"""
    from ramses_b200.tree import build_uniform_tree
    nx = coarse[0]
    a = build_uniform_tree(ndim, level, coarse=coarse, boxlen=float(nx), mhd=True)
    _potential_state(a, level, ndim, coarse)
    for resident in (False, True):
        r = _oracle_on_tree(a, ndim, level, level, float(nx), coarse, [1], r1, r2, slope_type)
        cells = _active_cells(r)
        assert _divb(r.uold.reshape(11, -1), cells, ndim) < 1e-13
        got, dts = _gpu_steps(r, ndim, r1, r2, slope_type, 3, resident, (2, -1))
        ref, dts_ref = _oracle_steps(r, 3)
        _assert_equal(r, got, dts, ref, dts_ref)
        assert np.abs(got[:, cells] - a.uold[:, cells]).max() > 1e-4        # the state moved
        assert _divb(got, cells, ndim) < 1e-12


@pytest.mark.parametrize("r1,r2,slope_type,resident", [("hlld", "hlld", 2, False), ("roe", "llf", 1, True)])
def test_mhd_amr_3d_non_cubic_patch_more_octs_than_sms(orc, r1, r2, slope_type, resident):
    """3-D nested tree whose refined levels are 12 x 6 x 8-oct boxes (576 octs at levels 5 and 6, 512 at level 4): every launch of
    mhd_amr3_godfine_kernel (one oct per CTA) has more CTAs than the H100 has SMs (132).  2 sub-cycled coarse steps == the oracle's
    amr_step on the same arrays, bit for bit, with div B at round-off on the device state"""
    from ramses_b200.tree import build_nested_tree
    levelmin, levelmax = 4, 6
    a = build_nested_tree(levelmin, levelmax, half_width=(6, 3, 4), mhd=True)
    assert [len(a.active[l]) for l in (4, 5, 6)] == [512, 576, 576]
    for l in range(1, levelmax + 1):
        _potential_state(a, l, 3, (1.0, 1.0, 1.0))
    r = _oracle_on_tree(a, 3, levelmin, levelmax, 1.0, (1, 1, 1), [1, 2, 2], r1, r2, slope_type)
    cells = _active_cells(r)
    assert _divb(r.uold.reshape(11, -1), cells, 3) < 1e-13
    got, dts = _gpu_steps(r, 3, r1, r2, slope_type, 2, resident, (2, -1))
    ref, dts_ref = _oracle_steps(r, 2)
    _assert_equal(r, got, dts, ref, dts_ref)
    assert _divb(got, cells, 3) < 1e-12


# ---- Level-0 drop-in with non-default limiters ---------------------------------------------------------------------------------
def test_mhd_amr_2d_level0_dropin_with_prolongation_limiters(orc):
    """the oracle's AMR driver (regridding every coarse step) with godunov_fine on the GPU through rgpu_godunov_fine, Orszag-Tang
    with interpol_type 1 and interpol_mag_type 3: 6 coarse steps == the all-oracle run with the same limiters, bit for bit (mesh,
    state, time); the default limiters give another state"""
    from oracle.amr_mhd import MhdAmrRun2D
    from test_gpu_zz_golden import attach_gpu_godunov
    kw = dict(nsubcycle=[1], riemann="hlld", riemann2d="hlld", slope_type=2, gamma=1.6666667, courant_factor=0.8, err_grad_p=0.1,
              tout=[1e9], nexpand=1, ngridmax=20000)
    runs = {}
    for name, (it, mt) in (("ref", (1, 3)), ("default", (2, -1))):
        runs[name] = MhdAmrRun2D(4, 6, 1.0, interpol_type=it, interpol_mag_type=mt, **kw)
        runs[name].run(max_coarse=6)
    r = MhdAmrRun2D(4, 6, 1.0, interpol_type=1, interpol_mag_type=3, **kw)
    h, st = attach_gpu_godunov(r, mhd=True, riemann="hlld", riemann2d="hlld", slope_type=2, interpol_type=1)
    h.set_interpol_mag(3)
    try:
        r.run(max_coarse=6)
    finally:
        h.finalize()
    ref = runs["ref"]
    assert st["calls"] > 6 and st["syncs"] > 1
    assert r.t == ref.t and np.array_equal(r.son, ref.son)
    assert np.array_equal(r.uold, ref.uold)
    assert not np.array_equal(runs["default"].uold, ref.uold)
