"""AMR levels on the GPU (oct-batch kernels: godfine1 with interpol_hydro ghost prolongation, flux masking, coarse
refluxing; upload_fine; boundaries; leaf-cell Courant scan) against the pinned oracle on meshes produced by the oracle's
AMR driver (oracle/amr.py).  One coarse step in amr_step order with sub-cycling, mesh kept static on both sides."""
import numpy as np
import pytest

from ramses_b200.hydro import AmrCommons

pytestmark = pytest.mark.gpu

SOD = [dict(type="square", x_center=0.25, length_x=0.5, d=1.0, p=1.0),
       dict(type="square", x_center=0.75, length_x=0.5, d=0.125, p=0.1)]


def commons_from_run(r, riemann, slope_type):
    m = r.m
    a = AmrCommons(r.ndim, r.nvar, m.ncoarse, m.ngridmax, m.nx, m.ny, m.nz, (m.icoarse_min, m.icoarse_max),
                   (m.jcoarse_min, m.jcoarse_max), (m.kcoarse_min, m.kcoarse_max), nlevelmax=r.nlevelmax, boxlen=r.p.boxlen)
    a.son[:] = r.son[1:]
    a.father[:] = r.father[1:]
    a.nbor[:, :] = r.nbor[:, 1:]
    a.uold[:, :] = r.uold.reshape(r.nvar, m.ncell)
    for l in range(1, r.nlevelmax + 1):
        a.active[l] = np.array(r.active[l], dtype=np.int32)
        a.boundary[l] = [np.array(r.bound[b][l], dtype=np.int32) for b in range(m.nboundary)]
    a.boundary_type = [m.boundary_type[b] for b in range(m.nboundary)]
    a.gamma, a.courant_factor = r.p.gamma, r.p.courant_factor
    a.slope_type, a.riemann, a.nvector = slope_type, riemann, r.nvector
    a.difmag = r.p.difmag
    a.smallr, a.smallc = r.p.smallr, r.p.smallc
    return a


def gpu_amr_step(h, a, r, l, icount, dtnew, dtold):
    """amr/amr_step.f90 on a static mesh, every pass through the C-ABI"""
    if len(a.active[l]) == 0:
        return
    dtold[l] = dtnew[l]
    a.dtnew[l] = a.boxlen / a.smallc               # pm/newdt_fine.f90:51
    dtnew[l] = h.courant_fine(l)
    if l > r.levelmin:
        dtnew[l] = min(dtnew[l - 1] / float(r.nsubcycle[l - 1]), dtnew[l])
    a.dtnew[l] = dtnew[l]
    h.set_unew(l)
    if l < r.nlevelmax and len(a.active.get(l + 1, [])) > 0:
        if r.nsubcycle[l] == 2:
            gpu_amr_step(h, a, r, l + 1, 1, dtnew, dtold)
            gpu_amr_step(h, a, r, l + 1, 2, dtnew, dtold)
        else:
            gpu_amr_step(h, a, r, l + 1, 1, dtnew, dtold)
    elif l < r.nlevelmax:
        dtold[l + 1] = dtnew[l] / float(r.nsubcycle[l])
        dtnew[l + 1] = dtnew[l] / float(r.nsubcycle[l])
    a.dtnew[l] = dtnew[l]
    h.godunov_fine_dev(l)
    h.set_uold(l)
    h.upload_fine(l)
    h.make_boundary_hydro(l)
    if l > r.levelmin:
        if r.nsubcycle[l - 1] == 1:
            dtnew[l - 1] = dtnew[l]
        if icount == 2:
            dtnew[l - 1] = dtold[l] + dtnew[l]


# 2-D box with reflexive x walls and outflow y faces: BOUNDARY_PARAMS whose y regions include the corner cells, like the
# reference's own namelists (tests/hydro/implosion/implosion.nml:17-24) -- every oct of the box then has all its neighbour
# father cells (a region per face only would leave the diagonal father cell of a corner oct undefined: son(0))
BOUND_2D_WALLS_X_OUTFLOW_Y = [(1, (0, 0), (1, 1), (0, 0)), (2, (2, 2), (1, 1), (0, 0)), (13, (0, 2), (0, 0), (0, 0)), (14, (0, 2), (2, 2), (0, 0))]


def run_case(ndim, levelmin, levelmax, bound, regions, riemann, slope_type, ncoarse_dev, interpol_type, nsub, boxlen=1.0,
             err=0.05, nexpand=1, difmag=0.0, bound_regions=None, interpol_var=0, gravity=False, pressure_fix=False, beta_fix=0.5,
             device_resident=False, floors=None):
    """one coarse step of an adaptively refined mesh, developed by the oracle's regridding driver and then frozen, on the GPU
    (host-driven amr_step order, or rgpu_amr_steps) and on the oracle; floors: every cell then holds a floor_state cell under
    helpers.FLOORS[floors] (helpers.fill_floor_state) for the compared step"""
    from oracle.amr import AmrRun
    from ramses_b200.hydro import HydroGPU
    r = AmrRun(ndim, levelmin, levelmax, bound, boxlen, nsubcycle=nsub, nexpand=nexpand, ngridmax=20000, riemann=riemann,
               slope_type=slope_type, err_grad_d=err, err_grad_u=err, err_grad_p=err, interpol_type=interpol_type,
               interpol_var=interpol_var, regions=regions, tout=[1e9], bound_regions=bound_regions)
    r.p.difmag = difmag                            # hydro_parameters.f90:81 (cmpdivu + consup in unsplit)
    r.flag_coarse(); r.init_refine(); r.init_refine_2()
    for _ in range(ncoarse_dev):                   # develop the flow with the full (regridding) driver
        r.refine_coarse(); r.push_lists(1)
        for l in range(1, levelmin + 1):
            r.make_boundary_hydro(l)
            if l < levelmin:
                r.refine_fine(l)
        r.amr_step(levelmin, 1)
        for l in range(levelmin - 1, 0, -1):
            r.upload_fine(l); r.make_boundary_hydro(l)
        for l in range(levelmin - 1, 0, -1):
            r.flag_fine(l, 2)
        r.flag_coarse()
        r.nstep_coarse += 1
    # regrid once more like the head of amr_step, then freeze the mesh
    for i in range(levelmin, levelmax + 1):
        if i > levelmin:
            r.make_boundary_hydro(i)
        r.refine_fine(i)
    nlev = [len(r.active[l]) for l in range(1, levelmax + 1)]
    assert sum(1 for n in nlev[levelmin:] if n > 0) >= 1, nlev      # a genuinely refined mesh
    if floors:
        from helpers import fill_floor_state
        r.p.smallr, r.p.smallc = fill_floor_state(r.uold, ndim, r.nvar, m_ncell(r), floors, 60 + ndim)
    a = commons_from_run(r, riemann, slope_type)
    # source terms are switched on for the compared coarse step only (the mesh was developed without them): poisson with an
    # arbitrary acceleration field f (an INPUT of the path) and pressure_fix (divu / enew, reset by set_unew of every level)
    a.poisson, a.pressure_fix, a.beta_fix = bool(gravity), bool(pressure_fix), beta_fix
    force = None
    if gravity:
        rng = np.random.default_rng(17 + ndim)
        force = np.ascontiguousarray((np.array([0.7, -0.4, 0.3])[:ndim, None] + 0.3 * rng.standard_normal((ndim, m_ncell(r)))) * 5.0)
    h = HydroGPU(a, amr_mode=True, interpol_type=interpol_type, interpol_var=interpol_var)
    for l in range(1, levelmax + 1):
        if len(a.active[l]):
            h.bind_level(l)
    h.upload_state(0)
    if gravity:
        h.upload_force(force)
    for l in range(1, levelmax + 1):
        if len(a.active[l]):
            h.make_boundary_hydro(l)
    dtnew = {l: r.dtnew[l] for l in range(0, levelmax + 2)}
    dtold = {l: r.dtold[l] for l in range(0, levelmax + 2)}
    if device_resident:      # rgpu_amr_steps: dtnew / dtold stay on the device, the source passes read dt from there
        a.numbtot = {l: len(a.active[l]) for l in range(1, levelmax + 1)}
        dts = h.amr_steps(levelmin, [0] + [r.nsubcycle[l] for l in range(1, levelmax + 1)], 1)
        dtnew[levelmin] = dts[0]
    else:
        gpu_amr_step(h, a, r, levelmin, 1, dtnew, dtold)
    h.download_state(0)
    extra = h.download_pressure_fix() if pressure_fix else None
    h.finalize()
    # oracle: the same coarse step on the frozen mesh
    r.static = True
    for l in range(1, levelmax + 1):
        r.make_boundary_hydro(l)
    import ctypes as C
    from oracle import orc
    L = orc.lib()
    L.orc_set_pressure_fix.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_double]
    L.orc_set_gravity.argtypes = [C.POINTER(C.c_double)]
    divu_o, enew_o = np.zeros(m_ncell(r)), np.zeros(m_ncell(r))
    try:
        if pressure_fix:
            L.orc_set_pressure_fix(orc.dptr(divu_o), orc.dptr(enew_o), beta_fix)
        if gravity:
            L.orc_set_gravity(orc.dptr(force))
        r.amr_step(levelmin, 1)
    finally:
        L.orc_set_pressure_fix(None, None, 0.0)
        L.orc_set_gravity(None)
    ref = r.uold.reshape(r.nvar, -1)
    cells = np.concatenate([[r.cell(ind, ig) - 1 for ig in r.active[l] for ind in range(r.T)] for l in range(1, levelmax + 1) if r.active[l]]).astype(np.int64)
    if pressure_fix:
        r.pfix_cmp = (extra[0][cells], divu_o[cells], extra[1][cells], enew_o[cells])
    return a.uold[:, cells], ref[:, cells], dtnew, r, nlev


def m_ncell(r):
    return r.m.ncell


@pytest.mark.parametrize("ndim,gravity,pfix,resident", [(1, True, True, False), (2, True, True, False), (3, True, True, False),
                                                        (3, True, False, True), (3, False, True, True), (2, True, True, True)])
def test_amr_gravity_and_pressure_fix_bitwise(ndim, gravity, pfix, resident):
    """poisson (gloc gather, gravity predictor, add_gravity_source_terms, gravity-limited Courant step) and pressure_fix (divu /
    enew through the sweep, the coarse refluxes and set_uold's pdV source and energy switch) over one sub-cycled coarse step of
    a refined mesh: state, divu, enew and dtnew equal the oracle's, host-driven and with the device-resident stepper."""
    kw = dict(gravity=gravity, pressure_fix=pfix, device_resident=resident)
    if ndim == 1:
        got, ref, dtnew, r, nlev = run_case(1, 3, 8, (1, 1, 0, 0, 0, 0), SOD, "hllc", 2, 6, 2, [1, 1, 1, 2], **kw)
    elif ndim == 2:
        regs = [dict(type="square", x_center=0.5, y_center=0.5, length_x=10, length_y=10, exp_region=10, d=1.0, p=0.1),
                dict(type="square", x_center=0.3, y_center=0.4, length_x=0.3, length_y=0.25, exp_region=2, d=2.0, u=0.3, v=-0.2, p=1.0)]
        got, ref, dtnew, r, nlev = run_case(2, 3, 5, (1, 1, 2, 2, 0, 0), regs, "hllc", 2, 2, 2, [1, 2], bound_regions=BOUND_2D_WALLS_X_OUTFLOW_Y, **kw)
    else:
        regs = [dict(type="square", x_center=0.5, y_center=0.5, z_center=0.5, length_x=10, length_y=10, length_z=10, exp_region=10, d=1.0, p=1e-5),
                dict(type="square", x_center=0.4, y_center=0.45, z_center=0.55, length_x=0.3, length_y=0.3, length_z=0.3, exp_region=2, d=1.5, p=2.0)]
        got, ref, dtnew, r, nlev = run_case(3, 3, 4, (0,) * 6, regs, "hllc", 1, 1, 1, [2, 2], **kw)
    lm = r.levelmin
    assert dtnew[lm] == r.dtnew[lm]
    assert np.array_equal(got, ref), (np.abs(got - ref).max(), nlev)
    if pfix:
        dk, do, ek, eo = r.pfix_cmp
        assert np.array_equal(dk, do) and np.array_equal(ek, eo)
        assert np.abs(do).max() > 0


@pytest.mark.parametrize("riemann,slope_type,interpol_type", [("hllc", 2, 2), ("llf", 1, 1), ("hll", 7, 3), ("acoustic", 8, 0)])
def test_amr_1d_sod_bitwise(riemann, slope_type, interpol_type):
    got, ref, dtnew, r, nlev = run_case(1, 3, 8, (1, 1, 0, 0, 0, 0), SOD, riemann, slope_type, 6, interpol_type, [1, 1, 1, 2])
    assert dtnew[3] == r.dtnew[3]
    assert np.array_equal(got, ref), (np.abs(got - ref).max(), nlev)


def test_amr_2d_bitwise():
    regs = [dict(type="square", x_center=0.5, y_center=0.5, length_x=10, length_y=10, exp_region=10, d=1.0, p=0.1),
            dict(type="square", x_center=0.3, y_center=0.4, length_x=0.3, length_y=0.25, exp_region=2, d=2.0, u=0.3, v=-0.2, p=1.0)]
    got, ref, dtnew, r, nlev = run_case(2, 3, 5, (1, 1, 2, 2, 0, 0), regs, "hllc", 2, 2, 2, [1, 2], bound_regions=BOUND_2D_WALLS_X_OUTFLOW_Y)
    assert dtnew[3] == r.dtnew[3]
    assert np.array_equal(got, ref), (np.abs(got - ref).max(), nlev)


@pytest.mark.parametrize("riemann", ["hllc", "exact"])
def test_amr_3d_sedov_like(riemann):
    regs = [dict(type="square", x_center=0.5, y_center=0.5, z_center=0.5, length_x=10, length_y=10, length_z=10, exp_region=10, d=1.0, p=0.1),
            dict(type="square", x_center=0.4, y_center=0.45, z_center=0.55, length_x=0.3, length_y=0.3, length_z=0.3, exp_region=2, d=1.5, p=2.0)]
    got, ref, dtnew, r, nlev = run_case(3, 3, 4, (0,) * 6, regs, riemann, 1, 1, 1, [2, 2])
    if riemann == "exact":
        scale = np.abs(ref).max(axis=1, keepdims=True)
        assert (np.abs(got - ref) / scale).max() <= 1e-12
    else:
        assert np.array_equal(got, ref), (np.abs(got - ref).max(), nlev)


@pytest.mark.parametrize("ndim,itype,ivar", [(3, 2, 1), (3, 4, 2), (3, 1, 2), (2, 2, 2), (2, 4, 2), (1, 2, 1)])
def test_amr_interpol_var_bitwise(ndim, itype, ivar):
    """interpol_var 1, 2 and interpol_type 4 (hydro/interpol_hydro.f90:318-440) on adaptively refined meshes: the oct-batch
    kernel's ghost prolongation and upload_fine's internal-energy averaging equal the oracle bit for bit."""
    if ndim == 1:
        got, ref, dtnew, r, nlev = run_case(1, 3, 8, (1, 1, 0, 0, 0, 0), SOD, "hllc", 2, 6, itype, [1, 1, 1, 2], interpol_var=ivar)
    elif ndim == 2:
        regs = [dict(type="square", x_center=0.5, y_center=0.5, length_x=10, length_y=10, exp_region=10, d=1.0, p=0.1),
                dict(type="square", x_center=0.3, y_center=0.4, length_x=0.3, length_y=0.25, exp_region=2, d=2.0, u=0.3, v=-0.2, p=1.0)]
        got, ref, dtnew, r, nlev = run_case(2, 3, 5, (1, 1, 2, 2, 0, 0), regs, "hllc", 2, 2, itype, [1, 2], interpol_var=ivar,
                                            bound_regions=BOUND_2D_WALLS_X_OUTFLOW_Y)
    else:
        regs = [dict(type="square", x_center=0.5, y_center=0.5, z_center=0.5, length_x=10, length_y=10, length_z=10, exp_region=10, d=1.0, p=0.1),
                dict(type="square", x_center=0.4, y_center=0.45, z_center=0.55, length_x=0.3, length_y=0.3, length_z=0.3, exp_region=2, d=1.5, u=0.2, p=2.0)]
        got, ref, dtnew, r, nlev = run_case(3, 3, 4, (0,) * 6, regs, "hllc", 1, 1, itype, [2, 2], interpol_var=ivar)
    assert dtnew[3] == r.dtnew[3]
    assert np.array_equal(got, ref), (np.abs(got - ref).max(), nlev)


@pytest.mark.parametrize("ndim", [1, 2, 3])
def test_amr_difmag_bitwise(ndim):
    """difmag>0: cmpdivu + consup (hydro/uplmde.f90:702,769) inside the oct-batch kernel, refined meshes in 1-D/2-D/3-D."""
    if ndim == 1:
        got, ref, dtnew, r, nlev = run_case(1, 3, 8, (1, 1, 0, 0, 0, 0), SOD, "hllc", 2, 6, 2, [1, 1, 1, 2], difmag=0.3)
    elif ndim == 2:
        regs = [dict(type="square", x_center=0.5, y_center=0.5, length_x=10, length_y=10, exp_region=10, d=1.0, p=0.1),
                dict(type="square", x_center=0.3, y_center=0.4, length_x=0.3, length_y=0.25, exp_region=2, d=2.0, u=0.3, v=-0.2, p=1.0)]
        got, ref, dtnew, r, nlev = run_case(2, 3, 5, (1, 1, 2, 2, 0, 0), regs, "hllc", 2, 2, 2, [1, 2], difmag=0.2, bound_regions=BOUND_2D_WALLS_X_OUTFLOW_Y)
    else:
        regs = [dict(type="square", x_center=0.5, y_center=0.5, z_center=0.5, length_x=10, length_y=10, length_z=10, exp_region=10, d=1.0, p=0.1),
                dict(type="square", x_center=0.4, y_center=0.45, z_center=0.55, length_x=0.3, length_y=0.3, length_z=0.3, exp_region=2, d=1.5, p=2.0)]
        got, ref, dtnew, r, nlev = run_case(3, 3, 4, (0,) * 6, regs, "llf", 1, 1, 1, [2, 2], difmag=0.25)
    assert dtnew[3] == r.dtnew[3]
    assert np.array_equal(got, ref), (np.abs(got - ref).max(), nlev)


def test_difmag_uniform_grid_through_amr_mode_and_dense_path_rejects():
    """levelmin=levelmax run with difmag>0: the dense fast path refuses, the oct-batch kernel (AMR mode) runs it bit-exactly."""
    from helpers import Case, smooth_state
    from ramses_b200 import lib as _l
    from ramses_b200.hydro import HydroGPU
    c = Case(3, 3, riemann="hllc", slope_type=1)
    c.p.difmag = 0.4
    u0 = smooth_state(3, 8)
    u0[1] += u0[0] * 0.8 * np.sin(2 * np.pi * (np.arange(8) + 0.5) / 8)[None, None, :]   # compression around x = 0.5: min(0, div u) is active
    c.init_dense(u0)
    dt, _ = c.oracle_courant()
    exp = c.oracle_godunov(dt).reshape(5, -1)
    c0 = Case(3, 3, riemann="hllc", slope_type=1)
    c0.init_dense(u0)
    assert not np.array_equal(c0.oracle_godunov(dt).reshape(5, -1), exp)      # the term is active
    a = c.amr_commons()
    a.difmag = 0.4
    h = HydroGPU(a)
    with pytest.raises(_l.RgpuError):
        h.bind_level(3)
    h.finalize()
    a = c.amr_commons()
    a.difmag = 0.4
    a.unew[:, :] = a.uold
    a.dtnew[3] = dt
    h = HydroGPU(a, amr_mode=True)
    for l in (1, 2, 3):
        h.bind_level(l)
    h.godunov_fine(3)
    h.finalize()
    act = c.active_cells()
    assert np.array_equal(a.unew[:, act], exp[:, act])


def _nested_case(levelmin, levelmax, half_width, riemann="hllc", slope_type=1):
    from ramses_b200.tree import build_nested_tree, cell_centers
    a = build_nested_tree(levelmin, levelmax, half_width=half_width, boxlen=1.0)
    a.gamma, a.courant_factor, a.slope_type, a.riemann = 1.4, 0.8, slope_type, riemann

    def ic(x, y, z):          # smooth blast at the box centre, resolved by the refined cube
        r2 = (x - 0.5) ** 2 + (y - 0.5) ** 2 + (z - 0.5) ** 2
        u = np.zeros((5, len(x)))
        u[0] = 1.0 + 0.5 * np.exp(-r2 / 0.01)
        u[1] = 0.1 * u[0] * np.sin(2 * np.pi * y)
        u[4] = (0.1 + 2.0 * np.exp(-r2 / 0.005)) / 0.4 + 0.5 * u[1] ** 2 / u[0]
        return u
    for l in range(levelmin, levelmax + 1):
        ig, cc = cell_centers(a, l)
        for ind in range(8):
            a.uold[:, a.ncoarse + ind * a.ngridmax + ig - 1] = ic(cc[ind][:, 0], cc[ind][:, 1], cc[ind][:, 2])
    return a


def _run_nested_gpu(a, levelmin, levelmax, ncoarse_steps=1, interpol_type=1, interpol_var=0):
    from ramses_b200.hydro import HydroGPU, amr_step
    h = HydroGPU(a, amr_mode=True, interpol_type=interpol_type, interpol_var=interpol_var)
    for l in range(1, levelmax + 1):
        h.bind_level(l)
    h.upload_state(0)
    for l in range(levelmax - 1, 0, -1):
        h.upload_fine(l)                      # restriction: split cells <- mean of their sons (init_refine does the same)
    nsub = [1] * (levelmin + 1) + [2] * 64   # nsubcycle(levelmin)=... 2 above levelmin-1
    nsub[levelmin - 1] = 1
    dtnew = {l: 0.0 for l in range(0, levelmax + 2)}
    dtold = {l: 0.0 for l in range(0, levelmax + 2)}
    h.download_state(0)
    u0 = a.uold.copy()
    for _ in range(ncoarse_steps):
        amr_step(h, levelmin, 1, levelmin, nsub, dtnew, dtold)
    h.download_state(0)
    launches = sum(h.level_info(l).kernel_launches for l in range(1, levelmax + 1))
    h.finalize()
    return u0, dtnew, nsub, launches


@pytest.mark.parametrize("itype,ivar", [(1, 0), (2, 1), (4, 2), (1, 2)])
def test_nested_tree_gpu_matches_oracle_bitwise(itype, ivar):
    """(interpol_type, interpol_var) incl. the coupled prolongations (internal energy / velocities, type 4) in the oct-batch
    kernel, the patch-mode shell fill and upload_fine.
    Product-side tree fabricator (ramses_b200.tree.build_nested_tree: 3 refined levels, 2:1 nesting) driven by the host
    mirror of amr_step (ramses_b200.hydro.amr_step, sub-cycling 1,2,2) == the oracle's amr_step on the same arrays."""
    from oracle.amr import AmrRun
    levelmin, levelmax, hw = 4, 6, 3
    a = _nested_case(levelmin, levelmax, hw)
    r = AmrRun(3, levelmin, levelmax, (0,) * 6, 1.0, nsubcycle=[1, 2, 2], ngridmax=a.ngridmax, riemann="hllc", slope_type=1,
               interpol_type=itype, interpol_var=ivar, tout=[1e9])
    assert r.ncell == a.ncell
    r.son[1:] = a.son; r.father[1:] = a.father; r.nbor[:, 1:] = a.nbor
    for l in range(1, levelmax + 1):
        r.active[l] = [int(g) for g in a.active[l]]
    r.push_all()
    u0, dtnew, nsub, launches = _run_nested_gpu(a, levelmin, levelmax, interpol_type=itype, interpol_var=ivar)
    r.uold[:] = u0.ravel()
    r.static = True
    r.amr_step(levelmin, 1)
    ref = r.uold.reshape(5, -1)
    assert dtnew[levelmin] == r.dtnew[levelmin]
    cells = np.concatenate([[a.ncoarse + ind * a.ngridmax + int(g) - 1 for g in a.active[l] for ind in range(8)] for l in range(1, levelmax + 1)])
    assert np.array_equal(a.uold[:, cells], ref[:, cells]), float(np.abs(a.uold[:, cells] - ref[:, cells]).max())


def test_amr_full_size_conservation_levelmin7_levelmax10():
    """BASELINE config 4 size (levelmin=7, levelmax=10: 2.1 M base cells + three refined levels of 32^3 octs) through a
    size-independent property: with refluxing and restriction the coarse step conserves mass, momentum and energy summed
    over the leaf cells to round-off (periodic box)."""
    from ramses_b200.tree import leaf_cells
    levelmin, levelmax = 7, 10
    a = _nested_case(levelmin, levelmax, 16)
    u0, dtnew, nsub, launches = _run_nested_gpu(a, levelmin, levelmax)

    def totals(u):
        t = np.zeros(5)
        for l in range(levelmin, levelmax + 1):
            c = leaf_cells(a, l)
            t += u[:, c].sum(axis=1) * (0.5 ** l) ** 3
        return t
    t0, t1 = totals(u0), totals(a.uold)
    assert dtnew[levelmin] > 0 and np.isfinite(a.uold).all()
    for iv in (0, 4):
        assert abs(t1[iv] - t0[iv]) <= 2e-13 * abs(t0[iv]), (iv, t0, t1)
    for iv in (1, 2, 3):
        assert abs(t1[iv] - t0[iv]) < 1e-13, (iv, t0, t1)
    # the solution moved
    assert np.abs(a.uold - u0).max() > 1e-3


@pytest.mark.parametrize("riemann", ["llf", "hll", "hllc", "acoustic"])
def test_passive_scalars_uniform_grid_bitwise(riemann):
    """NVAR = 7 (two passive scalars) on a levelmin=levelmax run through the oct-batch kernel: three level steps in amr_step
    order (courant, set_unew, godunov_fine, set_uold incl. the floor fix, boundaries) == the oracle."""
    from helpers import Case, smooth_state
    from ramses_b200.hydro import HydroGPU
    n = 8
    u7 = np.zeros((7, n, n, n))
    u7[:5] = smooth_state(3, n)
    u7[5] = 0.3 * u7[0]
    u7[6] = u7[0] * (0.5 + 0.4 * np.sin(2 * np.pi * (np.arange(n) + 0.5) / n))[None, :, None]
    c = Case(3, 3, riemann=riemann, slope_type=2, nvar=7, bound=(1, 1, 2, 2, 0, 0))
    c.init_dense(u7)
    ref, dts_ref = c.oracle_steps(3)
    a = c.amr_commons()
    h = HydroGPU(a, amr_mode=True)
    for l in (1, 2, 3):
        h.bind_level(l)
    h.upload_state(0)
    h.make_boundary_hydro(3)
    dts = []
    for _ in range(3):
        a.dtnew[3] = a.boxlen / a.smallc
        dts.append(h.courant_fine(3))
        h.set_unew(3); h.godunov_fine_dev(3); h.set_uold(3); h.make_boundary_hydro(3)
    h.download_state(0)
    h.finalize()
    act = c.active_cells()
    assert np.array_equal(np.array(dts), dts_ref)
    assert np.array_equal(a.uold[:, act], ref.reshape(7, -1)[:, act])


def test_passive_scalars_refined_mesh_bitwise():
    """Two passive scalars on the 3-level nested tree (prolongation, refluxing and restriction of all 7 variables)."""
    from oracle.amr import AmrRun
    from ramses_b200.tree import build_nested_tree, cell_centers
    from ramses_b200.hydro import HydroGPU, amr_step
    levelmin, levelmax = 4, 6
    a = build_nested_tree(levelmin, levelmax, half_width=3, boxlen=1.0, nvar=7)
    a.gamma, a.courant_factor, a.slope_type, a.riemann = 1.4, 0.8, 1, "hllc"
    for l in range(levelmin, levelmax + 1):
        ig, cc = cell_centers(a, l)
        for ind in range(8):
            x, y, z = cc[ind][:, 0], cc[ind][:, 1], cc[ind][:, 2]
            r2 = (x - 0.5) ** 2 + (y - 0.5) ** 2 + (z - 0.5) ** 2
            u = np.zeros((7, len(x)))
            u[0] = 1.0 + 0.5 * np.exp(-r2 / 0.01)
            u[1] = 0.1 * u[0] * np.sin(2 * np.pi * y)
            u[4] = (0.1 + 2.0 * np.exp(-r2 / 0.005)) / 0.4 + 0.5 * u[1] ** 2 / u[0]
            u[5] = u[0] * (0.2 + 0.1 * np.cos(2 * np.pi * x))
            u[6] = u[0] * np.exp(-r2 / 0.02)
            a.uold[:, a.ncoarse + ind * a.ngridmax + ig - 1] = u
    h = HydroGPU(a, amr_mode=True, interpol_type=1)
    for l in range(1, levelmax + 1):
        h.bind_level(l)
    h.upload_state(0)
    for l in range(levelmax - 1, 0, -1):
        h.upload_fine(l)
    h.download_state(0)
    u0 = a.uold.copy()
    nsub = [1] * (levelmin + 1) + [2] * 64
    dtnew = {l: 0.0 for l in range(0, levelmax + 2)}
    dtold = {l: 0.0 for l in range(0, levelmax + 2)}
    amr_step(h, levelmin, 1, levelmin, nsub, dtnew, dtold)
    h.download_state(0)
    h.finalize()
    r = AmrRun(3, levelmin, levelmax, (0,) * 6, 1.0, nsubcycle=[1, 2, 2], ngridmax=a.ngridmax, riemann="hllc", slope_type=1,
               interpol_type=1, tout=[1e9], nvar=7)
    r.uold[:] = u0.ravel()
    r.son[1:] = a.son; r.father[1:] = a.father; r.nbor[:, 1:] = a.nbor
    for l in range(1, levelmax + 1):
        r.active[l] = [int(g) for g in a.active[l]]
    r.push_all()
    r.static = True
    r.amr_step(levelmin, 1)
    ref = r.uold.reshape(7, -1)
    assert dtnew[levelmin] == r.dtnew[levelmin]
    cells = np.concatenate([[a.ncoarse + ind * a.ngridmax + int(g) - 1 for g in a.active[l] for ind in range(8)] for l in range(1, levelmax + 1)])
    assert np.array_equal(a.uold[:, cells], ref[:, cells]), float(np.abs(a.uold[:, cells] - ref[:, cells]).max())
    assert np.abs(a.uold[5:, cells] - u0[5:, cells]).max() > 1e-4


def test_passive_scalars_rejected_where_not_built():
    from helpers import Case
    from ramses_b200 import lib as _l
    from ramses_b200.hydro import HydroGPU
    c = Case(3, 2, nvar=7)
    a = c.amr_commons()
    h = HydroGPU(a)                      # fused dense path: refuses at bind time, pointing to rgpu_set_amr
    with pytest.raises(_l.RgpuError):
        h.bind_level(2)
    h.finalize()
    c = Case(3, 2, nvar=9)
    with pytest.raises(_l.RgpuError):
        HydroGPU(c.amr_commons(), amr_mode=True)
    c = Case(2, 2, nvar=5)
    with pytest.raises(_l.RgpuError):
        HydroGPU(c.amr_commons(), amr_mode=True)


def test_amr_steps_device_resident_dt_equals_host_driven():
    """rgpu_amr_steps (recursion on the host, every time step on the device, no round trip) == the host-driven amr_step
    sequence: same state, same dtnew(levelmin), over 3 coarse steps of the nested tree (oct-batch, dense-base and patch paths)."""
    levelmin, levelmax = 4, 6
    from ramses_b200.hydro import HydroGPU, amr_step
    res = []
    for mode in ("host", "device"):
        a = _nested_case(levelmin, levelmax, 3)
        h = HydroGPU(a, amr_mode=True, interpol_type=1)
        for l in range(1, levelmax + 1):
            h.bind_level(l)
        h.upload_state(0)
        for l in range(levelmax - 1, 0, -1):
            h.upload_fine(l)
        nsub = [1] * (levelmin + 1) + [2] * 64
        if mode == "host":
            dtnew = {l: 0.0 for l in range(0, levelmax + 2)}
            dtold = {l: 0.0 for l in range(0, levelmax + 2)}
            dts = []
            for _ in range(3):
                amr_step(h, levelmin, 1, levelmin, nsub, dtnew, dtold)
                dts.append(dtnew[levelmin])
        else:
            dts = list(h.amr_steps(levelmin, nsub, 3))
        h.download_state(0)
        h.finalize()
        res.append((np.array(dts), a.uold.copy()))
    assert np.array_equal(res[0][0], res[1][0]), (res[0][0], res[1][0])
    assert np.array_equal(res[0][1], res[1][1])
    assert (res[0][0] > 0).all()


@pytest.mark.parametrize("ndim", [2, 3])
def test_hydro_flag_on_device_equals_oracle(ndim):
    """rgpu_hydro_flag (hydro/hydro_flag.f90 + hydro_refine on the device-resident state; only the 4-byte flags of the level travel)
    == the oracle's hydro_flag on an adaptively refined mesh: flag1 of every active cell of every level below levelmax."""
    from oracle.amr import AmrRun
    from ramses_b200.hydro import HydroGPU
    if ndim == 2:
        regs = [dict(type="square", x_center=0.5, y_center=0.5, length_x=10, length_y=10, exp_region=10, d=1.0, p=0.1),
                dict(type="square", x_center=0.3, y_center=0.4, length_x=0.3, length_y=0.25, exp_region=2, d=2.0, u=0.3, v=-0.2, p=1.0)]
        r = AmrRun(2, 3, 5, (1, 1, 2, 2, 0, 0), 1.0, nsubcycle=[1, 2], ngridmax=20000, riemann="hllc", slope_type=2, err_grad_d=0.05,
                   err_grad_u=0.05, err_grad_p=0.05, interpol_type=2, regions=regs, tout=[1e9], bound_regions=BOUND_2D_WALLS_X_OUTFLOW_Y)
    else:
        regs = [dict(type="square", x_center=0.5, y_center=0.5, z_center=0.5, length_x=10, length_y=10, length_z=10, exp_region=10, d=1.0, p=0.1),
                dict(type="square", x_center=0.4, y_center=0.45, z_center=0.55, length_x=0.3, length_y=0.3, length_z=0.3, exp_region=2, d=1.5, u=0.2, p=2.0)]
        r = AmrRun(3, 3, 4, (0,) * 6, 1.0, nsubcycle=[2, 2], ngridmax=20000, riemann="hllc", slope_type=1, err_grad_d=0.05,
                   err_grad_u=0.05, err_grad_p=0.05, interpol_type=1, regions=regs, tout=[1e9])
    r.flag_coarse(); r.init_refine(); r.init_refine_2()
    for i in range(r.levelmin, r.nlevelmax + 1):
        if i > r.levelmin:
            r.make_boundary_hydro(i)
        r.refine_fine(i)
    for l in range(1, r.nlevelmax + 1):
        r.make_boundary_hydro(l)
    a = commons_from_run(r, "hllc", r.p.slope_type)
    h = HydroGPU(a, amr_mode=True, interpol_type=1)
    for l in range(1, r.nlevelmax + 1):
        if len(a.active[l]):
            h.bind_level(l)
    h.upload_state(0)
    nflag = 0
    for l in range(r.levelmin, r.nlevelmax):
        if not len(a.active[l]):
            continue
        flag1 = np.zeros(a.ncell, dtype=np.int32)
        h.hydro_flag(l, flag1, (r.err_grad_d, r.err_grad_u, r.err_grad_p), (r.floor_d, r.floor_u, r.floor_p))
        r.flag1[:] = 0
        r.hydro_flag(l)
        assert np.array_equal(flag1, np.asarray(r.flag1[1:], dtype=np.int32)), l
        nflag += int(flag1.sum())
    h.finalize()
    assert nflag > 10
