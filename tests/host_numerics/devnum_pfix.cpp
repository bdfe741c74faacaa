// The PFIX (pressure_fix) instantiations of the dense sweep's 3-D AMR variant compiled for the host (RGPU_HOST_NUMERICS) and run
// by the emulated launch of devnum.cpp: C entry point used by tests/test_pfix_dense_host.py.  TEST HARNESS ONLY, built like
// devnum.cpp (g++ -O2 -ffp-contract=off) into a library of its own; it reuses devnum.cpp's emulated launch and geometry helpers.
#include "devnum.cpp"

#pragma GCC visibility push(default)
extern "C" {

// the PFIX instantiation as launch_sweep_dense_pfix builds it: 3-D AMR variant, runtime slope switch, 12-row tiles.  uout holds
// unew and pfix holds divu / enew ([2][8][nslot], the level-store layout) on entry, both updated in place for the owned cells;
// force != NULL: the GRAV+PFIX form with f in the level-store layout [3][8][nslot] (predictor only, as AMR mode runs it)
int devnum_sweep_dense_pfix_box(int solver, const int* n, const int* shell, int nblocks, const double* uin, double* uout, double* pfix,
                                const double* force, const unsigned char* refined, double dt, double dx, int slope_type,
                                double slope_theta, double courant_factor, double gamma, double smallr, double smallc, int niter) {
  SweepArgs a;
  std::memset(&a, 0, sizeof a);
  a.g = box_geom(3, n, shell);
  const DenseGeom& g = a.g;
  a.uin = uin; a.uout = uout; a.pfix = pfix; a.force = force; a.gsrc = 0; a.refined = refined;
  a.P = make_phys(gamma, smallr, smallc, slope_theta, courant_factor, slope_type, niter);
  a.dt_dev = nullptr; a.dt_val = dt; a.dx = dx; a.inv_dx = 1.0 / dx;
  int ex;
  a.dx_pow2 = (std::frexp(dx, &ex) == 0.5) ? 1 : 0;
  constexpr int BY = tile_by_default(3, 0);
  const int txo = 30, tyo = BY - 2;
  a.ntx = (g.ox1 - g.ox0 + txo - 1) / txo;
  a.nty = (g.oy1 - g.oy0 + tyo - 1) / tyo;
  a.nwork = (long long)a.ntx * a.nty * (g.oz1 - g.oz0);
  if (nblocks > a.nwork) nblocks = (int)a.nwork;
  a.part = nullptr;
#define SP(RS, GRAV) emulate_launch(sweep_dense_kernel<3, RS, -1, 32, BY, true, false, GRAV, true>, a, nblocks, 32, BY, \
                                    SweepSmem<3, 32, BY, GRAV, true>::doubles)
#define SP_G(GRAV)                                                                                                   \
  do {                                                                                                               \
    if (solver == RIEMANN_LLF) SP(RIEMANN_LLF, GRAV); else if (solver == RIEMANN_EXACT) SP(RIEMANN_EXACT, GRAV);     \
    else if (solver == RIEMANN_ACOUSTIC) SP(RIEMANN_ACOUSTIC, GRAV);                                                 \
    else if (solver == RIEMANN_HLLC) SP(RIEMANN_HLLC, GRAV); else SP(RIEMANN_HLL, GRAV);                             \
  } while (0)
  if (force) SP_G(true);
  else SP_G(false);
#undef SP_G
#undef SP
  return nblocks;
}

}  // extern "C"
#pragma GCC visibility pop
