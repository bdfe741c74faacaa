// The GRAV (poisson) instantiations of the dense sweep compiled for the host (RGPU_HOST_NUMERICS) and run by the emulated launch
// of devnum.cpp: C entry point used by tests/test_gravity_dense_host.py.  TEST HARNESS ONLY, built like devnum.cpp
// (g++ -O2 -ffp-contract=off) into a library of its own; it reuses devnum.cpp's emulated launch and geometry helpers.
#include "devnum.cpp"

#pragma GCC visibility push(default)
extern "C" {

// the GRAV instantiation of the dense sweep (poisson) as launch_sweep_dense_grav builds it: runtime slope switch, default tile
// height.  force = f in the level-store layout [ndim][2^ndim][nslot]; gsrc = 1: the fused add_gravity_source_terms and the
// gravity term of the Courant partials (rgpu_level_steps); refined != NULL: the 3-D AMR variant (uout holds unew on entry)
int devnum_sweep_dense_grav_box(int ndim, int solver, const int* n, const int* shell, int nblocks, const double* uin, double* uout,
                                const double* force, int gsrc, const unsigned char* refined, double dt, double dx, int slope_type,
                                double slope_theta, double courant_factor, double gamma, double smallr, double smallc, int niter,
                                double* part) {
  SweepArgs a;
  std::memset(&a, 0, sizeof a);
  a.g = box_geom(ndim, n, shell);
  const DenseGeom& g = a.g;
  a.uin = uin; a.uout = uout; a.force = force; a.gsrc = gsrc; a.refined = refined;
  a.P = make_phys(gamma, smallr, smallc, slope_theta, courant_factor, slope_type, niter);
  a.dt_dev = nullptr; a.dt_val = dt; a.dx = dx; a.inv_dx = 1.0 / dx;
  int ex;
  a.dx_pow2 = (std::frexp(dx, &ex) == 0.5) ? 1 : 0;
  const int by = tile_by_default(ndim, solver);
  const int txo = 30, tyo = ndim > 1 ? by - 2 : 1;
  a.ntx = (g.ox1 - g.ox0 + txo - 1) / txo;
  a.nty = ndim > 1 ? (g.oy1 - g.oy0 + tyo - 1) / tyo : 1;
  a.nwork = (long long)a.ntx * a.nty * (ndim > 2 ? (g.oz1 - g.oz0) : 1);
  if (nblocks > a.nwork) nblocks = (int)a.nwork;
  a.part = part;
#define SG(ND, RS, BY, AMRV) emulate_launch(sweep_dense_kernel<ND, RS, -1, 32, BY, AMRV, false, true>, a, nblocks, 32, BY, \
                                            SweepSmem<ND, 32, BY, true>::doubles)
#define SG_ND(ND, BY, AMRV)                                                                                          \
  do {                                                                                                               \
    if (solver == RIEMANN_LLF) SG(ND, RIEMANN_LLF, BY, AMRV); else if (solver == RIEMANN_EXACT) SG(ND, RIEMANN_EXACT, BY, AMRV); \
    else if (solver == RIEMANN_ACOUSTIC) SG(ND, RIEMANN_ACOUSTIC, BY, AMRV);                                         \
    else if (solver == RIEMANN_HLLC) SG(ND, RIEMANN_HLLC, BY, AMRV); else SG(ND, RIEMANN_HLL, BY, AMRV);             \
  } while (0)
  if (ndim == 1) SG_ND(1, 1, false);
  else if (ndim == 2) SG_ND(2, 8, false);
  else if (refined) SG_ND(3, 12, true);
  else SG_ND(3, 12, false);
#undef SG_ND
#undef SG
  return nblocks;
}

}  // extern "C"
#pragma GCC visibility pop
