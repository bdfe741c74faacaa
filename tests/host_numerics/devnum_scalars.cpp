// Passive scalars (NVAR = NDIM+2+NPS, NDIM = 3, NPS <= 2) in the device code compiled for the host (RGPU_HOST_NUMERICS) and run by
// the emulated launch of devnum.cpp: C entry points used by tests/test_passive_scalars_host.py.  TEST HARNESS ONLY, built like
// devnum.cpp (g++ -O2 -ffp-contract=off) into a library of its own; it reuses devnum.cpp's emulated launch and helpers.
#include "devnum.cpp"

namespace {

template <int NX>
void riemann_nx_rows(int solver, int n, const double* ql, const double* qr, double* fg, double* fe, const Phys& P) {
  constexpr int NV = 5 + NX;
  for (int i = 0; i < n; i++) {
    const double *l = ql + i * NV, *r = qr + i * NV;
    double* f = fg + i * NV;
    switch (solver) {
      case RIEMANN_LLF: riemann<3, RIEMANN_LLF, NX>(l, r, f, P, fe + i); break;
      case RIEMANN_EXACT: riemann<3, RIEMANN_EXACT, NX>(l, r, f, P, fe + i); break;
      case RIEMANN_ACOUSTIC: riemann<3, RIEMANN_ACOUSTIC, NX>(l, r, f, P, fe + i); break;
      case RIEMANN_HLLC: riemann<3, RIEMANN_HLLC, NX>(l, r, f, P, fe + i); break;
      default: riemann<3, RIEMANN_HLL, NX>(l, r, f, P, fe + i); break;
    }
  }
}

template <int ND>
AmrGodfineKernel select_nd(int solver, const AmrSweepArgs& a) {
  switch (solver) {   // dispatch_amr_nd (rgpu_api.cu) -> launch_amr_godfine
    case RIEMANN_LLF: return amr_godfine_select<ND, RIEMANN_LLF>(a);
    case RIEMANN_EXACT: return amr_godfine_select<ND, RIEMANN_EXACT>(a);
    case RIEMANN_ACOUSTIC: return amr_godfine_select<ND, RIEMANN_ACOUSTIC>(a);
    case RIEMANN_HLLC: return amr_godfine_select<ND, RIEMANN_HLLC>(a);
    default: return amr_godfine_select<ND, RIEMANN_HLL>(a);
  }
}

AmrTree make_tree(int ndim, int ncoarse, int ngridmax, int nx, int ny, int nz, const int* son, const int* father, const int* nbor) {
  AmrTree t;
  std::memset(&t, 0, sizeof t);
  t.son = son - 1; t.father = father - 1; t.nbor = nbor; t.ncoarse = ncoarse; t.ngridmax = ngridmax; t.nx = nx; t.ny = ny; t.nz = nz;
  t.ncell = (long long)ncoarse + (long long)(1 << ndim) * ngridmax;
  return t;
}

}  // namespace

#pragma GCC visibility push(default)
extern "C" {

// n 3-D Riemann problems with nx = 1, 2 passive scalars: ql, qr [n][5+nx] in solver order (rho, u_n, P, u_t1, u_t2, Z...);
// fg [n][5+nx], fe [n] the internal-energy flux fgdnv(nvar+1)
int devnum_riemann_nx(int solver, int nx, int n, const double* ql, const double* qr, double* fg, double* fe, double gamma,
                      double smallr, double smallc, int niter) {
  const Phys P = make_phys(gamma, smallr, smallc, kNotRead, kNotRead, 1, niter);
  if (nx == 1) riemann_nx_rows<1>(solver, n, ql, qr, fg, fe, P);
  else if (nx == 2) riemann_nx_rows<2>(solver, n, ql, qr, fg, fe, P);
  else return -1;
  return 0;
}

// devnum_amr_godfine with nvar (NPS = nvar - ndim - 2 passive scalars) and interpol_var: the instantiation is the one
// launch_amr_godfine launches (amr_godfine_select); rflux [nact][2*ndim][2^(ndim-1)][nvar].  Returns -1 when none is built.
int devnum_amr_godfine_nps(int ndim, int solver, int ncoarse, int ngridmax, int nx, int ny, int nz, const int* son, const int* father,
                           const int* nbor, const int* active, int nact, int ilevel, const double* uold, double* unew, double* rflux,
                           double dt, double dx, int interpol_type, int interpol_var, int slope_type, double slope_theta, double gamma,
                           double smallr, double smallc, int niter, int nvar) {
  AmrSweepArgs a;
  std::memset(&a, 0, sizeof a);
  a.t = make_tree(ndim, ncoarse, ngridmax, nx, ny, nz, son, father, nbor);
  a.active = active; a.nact = nact; a.ilevel = ilevel; a.uold = uold; a.unew = unew; a.rflux = rflux;
  a.P = make_phys(gamma, smallr, smallc, slope_theta, kNotRead, slope_type, niter);
  a.dt = dt; a.dx = dx; a.inv_dx = 1.0 / dx;
  int ex;
  a.dx_pow2 = (std::frexp(dx, &ex) == 0.5) ? 1 : 0;
  a.interpol_type = interpol_type; a.interpol_var = interpol_var;
  a.nps = nvar - (ndim + 2);                        // amr_godunov (rgpu_api.cu)
  a.nvr = nvar;
  const AmrGodfineKernel k = ndim == 3 ? select_nd<3>(solver, a) : nullptr;   // scalars are built for NDIM = 3 only
  if (!k) return -1;
  emulate_launch(k, a, (nact + AMR_OPB - 1) / AMR_OPB, AMR_TPO * AMR_OPB);
  return 0;
}

// godunov_fine of one level: devnum_amr_godfine_nps + the coarse reflux pass of all nvar variables with the bind-time schedule
// (amr_schedules.h), as rgpu_godunov_fine does in AMR mode.  uold / unew [nvar][ncell].
int devnum_amr_godunov_nps(int ndim, int solver, int ncoarse, int ngridmax, int nx, int ny, int nz, const int* son, const int* father,
                           const int* nbor, const int* active, int nact, int ilevel, const double* uold, double* unew, double dt,
                           double dx, int interpol_type, int interpol_var, int slope_type, double slope_theta, double gamma,
                           double smallr, double smallc, int niter, int nvar, int nvector) {
  const int TW = 2 * ndim, NSF = 1 << (ndim - 1);
  // room for 7 columns whatever nvar is: a kernel of the wrong NPS then gives wrong numbers instead of writing past the buffer
  std::vector<double> rflux((size_t)std::max(1, nact) * TW * NSF * std::max(nvar, 7), 0.0);
  const int rc = devnum_amr_godfine_nps(ndim, solver, ncoarse, ngridmax, nx, ny, nz, son, father, nbor, active, nact, ilevel, uold, unew,
                                        rflux.data(), dt, dx, interpol_type, interpol_var, slope_type, slope_theta, gamma, smallr, smallc,
                                        niter, nvar);
  if (rc) return rc;
  std::vector<int> cells, start, srcs, src;
  build_reflux_schedule(ndim, nvector, nact, active, nbor, son, ngridmax, cells, start, srcs, src);
  if (!cells.empty()) {
    RefluxArgs r;
    std::memset(&r, 0, sizeof r);
    r.nent = (int)cells.size(); r.cell = cells.data(); r.start = start.data(); r.src = srcs.data(); r.rflux = rflux.data(); r.unew = unew;
    r.ncell = (long long)ncoarse + (long long)(1 << ndim) * ngridmax; r.nvar = nvar; r.nsides = TW; r.nsf = NSF;
    r.oneontwotondim = 1.0 / (double)(1 << ndim);
    emulate_serial(amr_reflux_kernel, r, (r.nent * nvar + 127) / 128, 128);
  }
  return 0;
}

// list passes of AMR mode over n octs igrid[] of a level, thread after thread, with the arguments rgpu_api.cu passes:
//   kind 0: amr_scalar_floor_kernel (set_uold: uold, unew)               -- u = uold, u2 = unew
//   kind 1: amr_upload_kernel (upload_fine; interpol_var)                 -- u = uold
//   kind 2: amr_boundary_kernel for boundary type bt (amr_boundaries)     -- u = uold, bvar[nvar] for imposed boundaries
int devnum_amr_list_pass(int kind, int ndim, int ncoarse, int ngridmax, int nx, int ny, int nz, const int* son, const int* father,
                         const int* nbor, const int* igrid, int n, int nvar, double* u, double* u2, double smallr, int interpol_var,
                         int bt, const double* bvar) {
  const AmrTree t = make_tree(ndim, ncoarse, ngridmax, nx, ny, nz, son, father, nbor);
  const int T = 1 << ndim;
  if (kind == 0) {
    struct S { const double* uo; double* un; const int* ig; int n, ncoarse, ngridmax; long long ncell; int T, nh, nvar; double smallr; };
    const S s{u, u2, igrid, n, ncoarse, ngridmax, t.ncell, T, ndim + 2, nvar, smallr};
    emulate_serial([](const S& x) { amr_scalar_floor_kernel(x.uo, x.un, x.ig, x.n, x.ncoarse, x.ngridmax, x.ncell, x.T, x.nh, x.nvar, x.smallr); },
                   s, (n * T + 127) / 128, 128);
  } else if (kind == 1) {
    struct S { double* u; const int* son1; const int* ig; int n, ncoarse, ngridmax; long long ncell; int T, nvar; double smallr; int iv, nd; };
    const S s{u, son - 1, igrid, n, ncoarse, ngridmax, t.ncell, T, nvar, smallr, interpol_var, ndim};
    emulate_serial([](const S& x) { amr_upload_kernel(x.u, x.son1, x.ig, x.n, x.ncoarse, x.ngridmax, x.ncell, x.T, x.nvar, x.smallr, x.iv, x.nd); },
                   s, (n * T + 127) / 128, 128);
  } else if (kind == 2) {
    static const int ref_x[8] = {2, 1, 4, 3, 6, 5, 8, 7}, ref_y[8] = {3, 4, 1, 2, 7, 8, 5, 6}, ref_z[8] = {5, 6, 7, 8, 1, 2, 3, 4};
    static const int fre[6][8] = {{1, 1, 3, 3, 5, 5, 7, 7}, {2, 2, 4, 4, 6, 6, 8, 8}, {1, 2, 1, 2, 5, 6, 5, 6},
                                  {3, 4, 3, 4, 7, 8, 7, 8}, {1, 2, 3, 4, 1, 2, 3, 4}, {5, 6, 7, 8, 5, 6, 7, 8}};
    static const int inb[7] = {0, 2, 1, 4, 3, 6, 5};
    const int dir = bt - 10 * (bt / 10), d = (dir - 1) / 2;
    AmrBoundArgs b;
    std::memset(&b, 0, sizeof b);
    b.n = n; b.igrid = igrid; b.inbor = inb[dir];
    const int* ir = (bt / 10 == 0) ? (d == 0 ? ref_x : d == 1 ? ref_y : ref_z) : fre[dir - 1];
    for (int i = 0; i < 8; i++) b.ind_ref[i] = ir[i];
    b.gs[0] = b.gs[1] = b.gs[2] = 1.0;
    if (bt >= 1 && bt <= 6) b.gs[d] = -1.0;
    b.kind = bt / 10; b.ndim = ndim; b.nvar = nvar; b.smallr = smallr;
    for (int iv = 0; iv < nvar && iv < 8; iv++) b.bvar[iv] = bvar ? bvar[iv] : 0.0;
    struct S { double* u; AmrTree t; AmrBoundArgs b; };
    const S s{u, t, b};
    emulate_serial([](const S& x) { amr_boundary_kernel(x.u, x.t, x.b); }, s, (n * T + 127) / 128, 128);
  } else return -1;
  return 0;
}

}  // extern "C"
#pragma GCC visibility pop
