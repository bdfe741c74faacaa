// pressure_fix on a levelmin=levelmax level, compiled for the host (RGPU_HOST_NUMERICS): the plain PFIX instantiations of the
// dense sweep run by the emulated launch of devnum.cpp, and the dense set_unew / set_uold passes (dense_pfix_init_kernel,
// dense_pdv_kernel, dense_pfix_switch_kernel of sweep_dense.cuh) run thread by thread.  C entry point used by
// tests/test_pfix_uniform_host.py.  TEST HARNESS ONLY, built like devnum.cpp (g++ -O2 -ffp-contract=off) into a library of its own.
#include "devnum.cpp"

namespace {
struct PfixPassArgs {
  int ndim, kind;                // kind 0: init, 1: pdV, 2: energy switch
  const double* uold;
  double* u;                     // kind 2: the new state, switched in place
  double* pfix;
  DenseGeom g;
  double gamma, smallr, beta_fix, dx, dt;
};
template <int ND>
void pfix_pass(const PfixPassArgs& p) {
  if (p.kind == 0) dense_pfix_init_kernel<ND>(p.uold, p.pfix, p.g, p.smallr);
  else if (p.kind == 1) dense_pdv_kernel<ND>(p.uold, p.pfix, p.g, p.gamma, p.smallr, p.dx, p.dt, nullptr);
  else dense_pfix_switch_kernel<ND>(p.u, p.pfix, p.g, p.smallr, p.beta_fix, p.dx, p.dt, nullptr);
}
void run_pass(PfixPassArgs p, int kind) {
  p.kind = kind;
  const long long n = (long long)(p.g.ox1 - p.g.ox0) * (p.g.oy1 - p.g.oy0) * (p.g.oz1 - p.g.oz0);
  const long long nb = (n + 127) / 128;
  if (p.ndim == 1) emulate_serial(pfix_pass<1>, p, nb, 128);
  else if (p.ndim == 2) emulate_serial(pfix_pass<2>, p, nb, 128);
  else emulate_serial(pfix_pass<3>, p, nb, 128);
}
}  // namespace

#pragma GCC visibility push(default)
extern "C" {

// one level step of rgpu_level_steps with pressure_fix on a box of n[0] x n[1] x n[2] owned cells (box_geom): set_unew's
// divu / enew from uold into pfix ([2][2^ndim][nslot]), the plain PFIX sweep (launch_sweep_dense_pfix_plain: runtime slope
// switch, default tile height; uin = uold -> uout), set_uold's pdV source from uold and the energy switch on uout.  uold must hold
// its ghost / boundary shell.  part != NULL receives the sweep's Courant partials [4][nblocks] (of the state before the switch).
int devnum_pfix_plain_step(int ndim, int solver, const int* n, const int* shell, int nblocks, const double* uold, double* uout,
                           double* pfix, double dt, double dx, int slope_type, double slope_theta, double courant_factor, double gamma,
                           double smallr, double smallc, int niter, double beta_fix, double* part) {
  SweepArgs a;
  std::memset(&a, 0, sizeof a);
  a.g = box_geom(ndim, n, shell);
  const DenseGeom& g = a.g;
  a.uin = uold; a.uout = uout; a.pfix = pfix;
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
  PfixPassArgs p{ndim, 0, uold, uout, pfix, g, gamma, smallr, beta_fix, dx, dt};
  run_pass(p, 0);
#define SP(ND, RS, BY) emulate_launch(sweep_dense_kernel<ND, RS, -1, 32, BY, false, false, false, true>, a, nblocks, 32, BY, \
                                      SweepSmem<ND, 32, BY, false, true>::doubles)
#define SP_ND(ND, BY)                                                                                                \
  do {                                                                                                               \
    if (solver == RIEMANN_LLF) SP(ND, RIEMANN_LLF, BY); else if (solver == RIEMANN_EXACT) SP(ND, RIEMANN_EXACT, BY); \
    else if (solver == RIEMANN_ACOUSTIC) SP(ND, RIEMANN_ACOUSTIC, BY);                                               \
    else if (solver == RIEMANN_HLLC) SP(ND, RIEMANN_HLLC, BY); else SP(ND, RIEMANN_HLL, BY);                         \
  } while (0)
  if (ndim == 1) SP_ND(1, 1);
  else if (ndim == 2) SP_ND(2, 8);
  else SP_ND(3, 12);
#undef SP_ND
#undef SP
  run_pass(p, 1);
  run_pass(p, 2);
  return nblocks;
}

}  // extern "C"
#pragma GCC visibility pop
