"""CPU pins of the oracle on domains of several coarse cells (nx, ny, nz of AMR_PARAMS): the builder agrees with the product's
tree fabricator, a state that repeats with the period of one coarse cell evolves exactly like the single-cell run (which the
golden files pin), and the x<->y transposed problem gives the transposed answer.  The GPU tests on non-cubic boxes
(test_gpu_box_shapes.py) and the emulated launches on non-cubic boxes (test_device_numerics_host.py) compare with this."""
import numpy as np
import pytest

from helpers import Case, MhdCase, box_state, mhd_smooth_state

LEVEL = 4


def _split(c, ngm, nco):
    """cell index -> (position in its oct or -1 for a coarse cell, igrid or coarse index): comparable across ngridmax"""
    c = np.asarray(c, dtype=np.int64)
    ind = np.where(c > nco, (c - nco - 1) // ngm, -1)
    g = np.where(c > nco, (c - nco - 1) % ngm + 1, c)
    return ind, g


@pytest.mark.parametrize("coarse", [(3, 2, 1), (1, 2, 3)])
@pytest.mark.parametrize("order", ["creation", "lattice"])
def test_tree_builder_matches_oracle_builder_on_box(orc, coarse, order):
    """ramses_b200.tree.build_uniform_tree(coarse=...) and the oracle's orc_mesh_build_box fabricate the same tree: father,
    son, nbor and the active list of every level, in the reference's creation order and in lattice order."""
    from ramses_b200.tree import build_uniform_tree
    lev = 3
    a = build_uniform_tree(3, lev, coarse=coarse, order=order)
    m = orc.Mesh(3, lev, order={"creation": 0, "lattice": 1}[order], coarse=coarse)
    n = m.s.ngrid_used
    assert (m.s.nx, m.s.ny, m.s.nz) == coarse and m.s.ncoarse == a.ncoarse == coarse[0] * coarse[1] * coarse[2]
    assert m.coarse() == coarse and (a.icoarse_min, a.icoarse_max) == (m.s.icoarse_min, m.s.icoarse_max)
    assert n == sum(len(a.active[l]) for l in range(1, lev + 1))
    fa, fm = _split(a.father[:n], a.ngridmax, a.ncoarse), _split(m.father()[1:n + 1], m.ngridmax, m.ncoarse)
    assert np.array_equal(fa[0], fm[0]) and np.array_equal(fa[1], fm[1])
    for j in range(6):
        na, nm = _split(a.nbor[j, :n], a.ngridmax, a.ncoarse), _split(m.nbor()[j, 1:n + 1], m.ngridmax, m.ncoarse)
        assert np.array_equal(na[0], nm[0]) and np.array_equal(na[1], nm[1])
    for l in range(1, lev + 1):
        assert np.array_equal(a.active[l], m.active(l))
    son_m = m.son()[1:]
    assert np.array_equal(a.son[:a.ncoarse], son_m[:m.ncoarse])
    for ind in range(8):
        assert np.array_equal(a.son[a.ncoarse + ind * a.ngridmax:a.ncoarse + ind * a.ngridmax + n],
                              son_m[m.ncoarse + ind * m.ngridmax:m.ncoarse + ind * m.ngridmax + n])


def _cell_state(n, seed):
    """a smooth periodic state on one coarse cell of n^3 cells with different wave numbers per axis and seeded density jumps"""
    ax = (np.arange(n) + 0.5) / n
    Z, Y, X = np.meshgrid(ax, ax, ax, indexing="ij")
    tw = 2 * np.pi
    rho = 1 + 0.2 * np.sin(tw * X) * np.cos(2 * tw * Y) + 0.1 * np.sin(3 * tw * Z + 0.4)
    rho *= 1 + 0.3 * (np.random.default_rng(seed).standard_normal(rho.shape) > 1.2)
    vel = [0.3 * np.sin(2 * tw * Y + 0.1), 0.25 * np.sin(tw * Z), 0.2 * np.cos(3 * tw * X)]
    p = 1 + 0.1 * np.cos(tw * (X + 2 * Y + 3 * Z))
    u = np.zeros((5, n, n, n))
    u[0] = rho
    for d in range(3):
        u[1 + d] = rho * vel[d]
    u[4] = p / 0.4 + 0.5 * rho * (vel[0] ** 2 + vel[1] ** 2 + vel[2] ** 2)
    return u


def _blocks(d, coarse, n):
    """the coarse-cell blocks of a dense [nvar][nz][ny][nx] array"""
    return [d[:, k * n:(k + 1) * n, j * n:(j + 1) * n, i * n:(i + 1) * n]
            for k in range(coarse[2]) for j in range(coarse[1]) for i in range(coarse[0])]


@pytest.mark.parametrize("riemann", ["llf", "exact", "acoustic", "hllc", "hll"])
@pytest.mark.parametrize("slope_type", [1, 2, 8])
def test_tiled_box_equals_single_cell_run_bitwise(orc, riemann, slope_type):
    """A state with the period of one coarse cell on a 3x2x1 domain (boxlen 3, so dx is that of the 1x1x1 domain with boxlen 1):
    after 6 level steps every coarse-cell block and the dt history equal the single-cell run, bit for bit."""
    n = 1 << LEVEL
    u1 = _cell_state(n, 5)
    one = Case(3, LEVEL, riemann=riemann, slope_type=slope_type, boxlen=1.0)
    box = Case(3, LEVEL, riemann=riemann, slope_type=slope_type, boxlen=3.0, coarse=(3, 2, 1), order=1)
    assert orc.lib().orc_dx(orc.C.byref(one.p), one.mesh.ptr, LEVEL) == orc.lib().orc_dx(orc.C.byref(box.p), box.mesh.ptr, LEVEL)
    one.init_dense(u1)
    box.init_dense(np.tile(u1, (1, 1, 2, 3)))
    r1, dts1 = one.oracle_steps(6)
    rb, dtsb = box.oracle_steps(6)
    d1 = one.dense(r1)
    assert np.abs(d1 - u1).max() > 1e-3
    assert np.array_equal(dtsb, dts1)
    blocks = _blocks(box.dense(rb), (3, 2, 1), n)
    assert len(blocks) == 6
    for b in blocks:
        assert np.array_equal(b, d1)


def test_tiled_box_equals_single_cell_run_bitwise_mhd(orc):
    """The same for the MHD solver (hlld / hlld, constrained transport) on a 3x2x1 domain."""
    n = 1 << LEVEL
    u1 = mhd_smooth_state(n)
    u1[0] *= 1 + 0.2 * (np.random.default_rng(8).standard_normal(u1[0].shape) > 1.2)
    one = MhdCase(LEVEL, riemann="hlld", riemann2d="hlld", slope_type=2, boxlen=1.0)
    box = MhdCase(LEVEL, riemann="hlld", riemann2d="hlld", slope_type=2, boxlen=3.0, coarse=(3, 2, 1), order=1)
    one.init_dense(u1)
    box.init_dense(np.tile(u1, (1, 1, 2, 3)))
    r1, dts1 = one.oracle_steps(6)
    rb, dtsb = box.oracle_steps(6)
    d1 = one.dense(r1)
    assert np.abs(d1 - u1).max() > 1e-3
    assert np.array_equal(dtsb, dts1)
    for b in _blocks(box.dense(rb), (3, 2, 1), n):
        assert np.array_equal(b, d1)


@pytest.mark.parametrize("riemann", ["hllc", "llf", "exact"])
def test_axis_permutation_on_box(orc, riemann):
    """A non-repeating state on a 3x2x1 domain and the x<->y transposed state (momenta swapped) on a 2x3x1 domain, same dx:
    after 6 level steps the second run is the transpose of the first to the tolerance of the corner-blast permutation test."""
    n = 1 << LEVEL
    a = Case(3, LEVEL, riemann=riemann, slope_type=2, boxlen=3.0, coarse=(3, 2, 1), order=2, seed=4)
    b = Case(3, LEVEL, riemann=riemann, slope_type=2, boxlen=2.0, coarse=(2, 3, 1), order=1)
    ua = box_state(3, (3 * n, 2 * n, n))
    ub = ua.transpose(0, 1, 3, 2)[[0, 2, 1, 3, 4]].copy()
    a.init_dense(ua)
    b.init_dense(ub)
    ra, dta = a.oracle_steps(6)
    rb, dtb = b.oracle_steps(6)
    da, db = a.dense(ra), b.dense(rb)
    assert np.abs(da - ua).max() > 1e-3
    assert np.allclose(dta, dtb, rtol=1e-13, atol=0)
    back = db.transpose(0, 1, 3, 2)[[0, 2, 1, 3, 4]]
    assert np.abs(back[0] - da[0]).max() < 1e-13 * np.abs(da[0]).max()
    for v in (1, 2, 3, 4):
        assert np.abs(back[v] - da[v]).max() < 1e-11 * np.abs(da[v]).max()


def test_amr_driver_on_a_box_tree_equals_uniform_run(orc):
    """oracle.amr.AmrRun(coarse=(3, 2, 1)) holding the arrays of a fully refined 3x2x1 tree (the way fabricated trees are loaded
    for the AMR comparisons): two static coarse steps of its amr_step equal two level steps of the uniform driver"""
    from oracle.amr import AmrRun
    lev, coarse = 3, (3, 2, 1)
    c = Case(3, lev, riemann="hllc", slope_type=2, boxlen=3.0, coarse=coarse, order=2, seed=6)
    c.init_dense(box_state(3, c.mesh.extent(lev)))
    ref, dts = c.oracle_steps(2, nthreads=1)
    m = c.mesh
    r = AmrRun(3, lev, lev, (0,) * 6, 3.0, nsubcycle=[1], ngridmax=m.ngridmax, riemann="hllc", slope_type=2, tout=[1e9],
               coarse=coarse)
    assert (r.m.nx, r.m.ny, r.m.nz, r.m.icoarse_max, r.m.jcoarse_max, r.ncell) == (3, 2, 1, 2, 1, m.ncell)
    r.son[:] = m.son(); r.father[:] = m.father(); r.nbor[:, :] = m.nbor(); r.xg[:, :] = m.xg()
    for l in range(1, lev + 1):
        r.active[l] = [int(g) for g in m.active(l)]
    r.push_all()
    r.uold[:] = c.u
    r.static = True
    got = []
    for _ in range(2):
        r.amr_step(lev, 1)
        got.append(r.dtnew[lev])
    idx = c.active_cells()
    assert np.array_equal(np.array(got), dts)
    assert np.array_equal(r.uold.reshape(5, -1)[:, idx], ref.reshape(5, -1)[:, idx])
