// Device numerics of ramses_b200/csrc compiled for the host (RGPU_HOST_NUMERICS): C entry points used by
// tests/test_device_numerics_host.py to compare the formulas the kernels execute with the oracle, bit for bit, on the CPU.
// TEST HARNESS ONLY.  Built with  g++ -O2 -ffp-contract=off  (the device build uses -fmad=false for the same reason).
#define RGPU_HOST_NUMERICS 1
#define MHD_DEFINE_KERNELS 1
static double* rgpu_host_dyn_smem = nullptr;   // dynamic shared memory of an emulated launch (sweep_dense.cuh)
#include "mhd_dense.cuh"    // the six MHD passes; pulls sweep_dense.cuh, mhd_device.cuh, hydro_device.cuh, real64.cuh
#include "amr_kernels.cuh"  // the AMR oct-batch kernel and its __device__ tree-walk / prolongation helpers
#include "mhd_amr.cuh"      // ideal MHD in AMR mode, NDIM = 1, 2
#include "amr_schedules.h"  // host-side reflux schedules (shared with rgpu_api.cu)
#include "sweep_dense4.cuh" // one-barrier form (includes sweep_dense3.cuh)
#include "sweep_dense3.cuh" // round-2 form of the 3-D dense sweep + the lane-generic solvers (hydro_vec.cuh)

#include <limits>
#include <pthread.h>
#include <thread>
#include <vector>

using namespace rgpu;

// ---- emulated launch of a barrier-only kernel: one OS thread per CUDA thread of a block, blocks one after the other ----------
static pthread_barrier_t g_block_barrier;
static void block_barrier() { pthread_barrier_wait(&g_block_barrier); }

template <class Kernel, class Args>
static void emulate_launch(Kernel kernel, const Args& a, int nblocks, int bx, int by = 1, size_t dyn_smem_doubles = 0) {
  const int nthreads = bx * by, nwarps = (nthreads + 31) / 32;
  pthread_barrier_init(&g_block_barrier, nullptr, (unsigned)nthreads);
  rgpu_stub_sync_hook = block_barrier;
  const bool warps = (nthreads % 32 == 0);             // warp exchange needs full warps
  if (warps) for (int w = 0; w < nwarps; w++) pthread_barrier_init(&rgpu_stub_warp_bar[w], nullptr, 32);
  rgpu_stub_warp_on = warps;
  std::vector<double> dyn(dyn_smem_doubles + 1, 0.0);
  rgpu_host_dyn_smem = dyn.data();
  std::vector<std::thread> team;
  for (int t = 0; t < nthreads; t++)
    team.emplace_back([&, t] {
      for (int b = 0; b < nblocks; b++) {
        threadIdx = {(unsigned)(t % bx), (unsigned)(t / bx), 0}; blockIdx = {(unsigned)b, 0, 0};
        blockDim = {(unsigned)bx, (unsigned)by, 1}; gridDim = {(unsigned)nblocks, 1, 1};
        kernel(a);
        pthread_barrier_wait(&g_block_barrier);      // the next block reuses the __shared__ storage
      }
    });
  for (auto& th : team) th.join();
  rgpu_stub_sync_hook = nullptr;
  rgpu_stub_warp_on = false;
  rgpu_host_dyn_smem = nullptr;
  if (warps) for (int w = 0; w < nwarps; w++) pthread_barrier_destroy(&rgpu_stub_warp_bar[w]);
  pthread_barrier_destroy(&g_block_barrier);
}

// one thread after the other: good for kernels whose threads do not communicate (the per-cell MHD passes)
template <class Kernel, class Args>
static void emulate_serial(Kernel kernel, const Args& a, long long nblocks, int nthreads) {
  rgpu_stub_sync_hook = nullptr;
  for (long long b = 0; b < nblocks; b++)
    for (int t = 0; t < nthreads; t++) {
      threadIdx = {(unsigned)t, 0, 0}; blockIdx = {(unsigned)b, 0, 0};
      blockDim = {(unsigned)nthreads, 1, 1}; gridDim = {(unsigned)nblocks, 1, 1};
      kernel(a);
    }
}

// a parameter that the kernels behind an entry point do not read: NaN, so that a kernel which did read it gives NaN instead of
// the oracle's bits
static const double kNotRead = std::numeric_limits<double>::quiet_NaN();

static Phys make_phys(double gamma, double smallr, double smallc, double slope_theta, double courant_factor, int slope_type,
                      int niter) {   // mirrors rgpu_init (ramses_b200/csrc/rgpu_api.cu)
  Phys P;
  P.gamma = gamma; P.smallr = smallr; P.smallc = smallc; P.slope_theta = slope_theta; P.courant_factor = courant_factor;
  P.smalle = smallc * smallc / gamma / (gamma - 1.0);
  P.smallp = smallc * smallc / gamma;
  P.smallpp = smallr * P.smallp;
  P.entho = 1.0 / (gamma - 1.0);
  P.gamma6 = (gamma + 1.0) / (2.0 * gamma);
  P.smallc2 = smallc * smallc;
  P.inv_gamma = 1.0 / gamma;
  P.cfl_g = 0.0001;
  P.cfl_rg = 1.0 / P.cfl_g;
  P.cfl_k = std::sqrt(1.0 + 2.0 * courant_factor * P.cfl_g) - 1.0;
  P.slope_type = slope_type; P.niter_riemann = niter;
  return P;
}

template <int NDIM>
static void riemann_nd(int solver, const double* ql, const double* qr, double* fg, const Phys& P) {
  switch (solver) {
    case RIEMANN_LLF: riemann<NDIM, RIEMANN_LLF>(ql, qr, fg, P); break;
    case RIEMANN_EXACT: riemann<NDIM, RIEMANN_EXACT>(ql, qr, fg, P); break;
    case RIEMANN_ACOUSTIC: riemann<NDIM, RIEMANN_ACOUSTIC>(ql, qr, fg, P); break;
    case RIEMANN_HLLC: riemann<NDIM, RIEMANN_HLLC>(ql, qr, fg, P); break;
    default: riemann<NDIM, RIEMANN_HLL>(ql, qr, fg, P); break;
  }
}

// Built with -fvisibility=hidden -Wl,-Bsymbolic: the kernels compiled here have the same mangled names as the CUDA launch stubs
// of libramses_gpu.so (loaded RTLD_GLOBAL by the ABI tests in the same process) and must never be interposed by them.
// interpol_hydro for the whole state (interpol_var 0/1/2, interpol_type 0..4): u1 [n][2*ndim+1][ndim+2] -> u2 [n][2^ndim][ndim+2]
template <int ND>
static void interpol_full_nd(int itype, int ivar, int n, const double* u1, double* u2, double smallr) {
  constexpr int NVX = ND + 2, T = 1 << ND, NA = 2 * ND + 1;
  for (int i = 0; i < n; i++) {
    double a[7][NVX], b[T][NVX];
    for (int j = 0; j < NA; j++) for (int v = 0; v < NVX; v++) a[j][v] = u1[(i * NA + j) * NVX + v];
    amr_interpol_hydro<ND, NVX>(a, itype, ivar, smallr, b);
    for (int t = 0; t < T; t++) for (int v = 0; v < NVX; v++) u2[(i * T + t) * NVX + v] = b[t][v];
  }
}
// dense-box geometry of an owned box of n[d] cells per axis, set the way plan_level (rgpu_api.cu) sets it: an axis without a
// shell is periodic over the box, an axis with shell[d] != 0 carries one ghost oct (2 cells) on each side; n[d] = 1 beyond ndim
static DenseGeom box_geom(int ndim, const int n[3], const int shell[3]) {
  DenseGeom g;
  std::memset(&g, 0, sizeof g);
  int nc[3], o0[3], o1[3], wr[3];
  for (int d = 0; d < 3; d++) {
    const int sh = (d < ndim && shell[d]) ? 2 : 0;
    nc[d] = d < ndim ? n[d] + 2 * sh : 1;
    o0[d] = sh; o1[d] = d < ndim ? sh + n[d] : 1;
    wr[d] = d < ndim && !shell[d];
  }
  g.ncx = nc[0]; g.ncy = nc[1]; g.ncz = nc[2];
  g.nox = (nc[0] + 1) / 2; g.noy = (nc[1] + 1) / 2; g.noz = (nc[2] + 1) / 2;
  g.ox0 = o0[0]; g.ox1 = o1[0]; g.oy0 = o0[1]; g.oy1 = o1[1]; g.oz0 = o0[2]; g.oz1 = o1[2];
  g.wrapx = wr[0]; g.wrapy = wr[1]; g.wrapz = wr[2];
  g.nslot = (long long)g.nox * g.noy * g.noz;
  return g;
}
static const int k_no_shell[3] = {0, 0, 0};

#pragma GCC visibility push(default)
extern "C" {

// n Riemann problems: ql, qr [n][ndim+2] in solver order (rho, u_n, P, u_t1, u_t2), fg [n][ndim+2]
void devnum_riemann(int ndim, int solver, int n, const double* ql, const double* qr, double* fg, double gamma, double smallr,
                    double smallc, int niter) {
  const Phys P = make_phys(gamma, smallr, smallc, kNotRead, kNotRead, 1, niter);
  const int nv = ndim + 2;
  for (int i = 0; i < n; i++) {
    if (ndim == 1) riemann_nd<1>(solver, ql + i * nv, qr + i * nv, fg + i * nv, P);
    else if (ndim == 2) riemann_nd<2>(solver, ql + i * nv, qr + i * nv, fg + i * nv, P);
    else riemann_nd<3>(solver, ql + i * nv, qr + i * nv, fg + i * nv, P);
  }
}

// n cells: u [n][ndim+2] conservative -> q [n][ndim+3] (rho, v, P, 1/rho as the kernels keep it is NOT part of q here)
void devnum_ctoprim(int ndim, int n, const double* u, double* q, double gamma, double smallr, double smallc) {
  const Phys P = make_phys(gamma, smallr, smallc, kNotRead, kNotRead, 1, 10);
  const int nv = ndim + 2;
  for (int i = 0; i < n; i++) {
    if (ndim == 1) ctoprim<1>(u + i * nv, q + i * nv, P);
    else if (ndim == 2) ctoprim<2>(u + i * nv, q + i * nv, P);
    else ctoprim<3>(u + i * nv, q + i * nv, P);
  }
}

// n cells: dt = cmpdt_cell(u, dx)
void devnum_cmpdt(int ndim, int n, const double* u, double dx, double* dt, double gamma, double smallr, double smallc, double cfl) {
  const Phys P = make_phys(gamma, smallr, smallc, kNotRead, cfl, 1, 10);
  const int nv = ndim + 2;
  for (int i = 0; i < n; i++) {
    double ei;
    if (ndim == 1) dt[i] = cmpdt_cell<1>(u + i * nv, dx, P, ei);
    else if (ndim == 2) dt[i] = cmpdt_cell<2>(u + i * nv, dx, P, ei);
    else dt[i] = cmpdt_cell<3>(u + i * nv, dx, P, ei);
  }
}

// n limited slopes of (ql, qc, qr) for slope_type 1, 2, 7, 8 (the one-dimensional limiters)
void devnum_slope(int slope_type, int n, const double* ql, const double* qc, const double* qr, double* dq, double slope_theta) {
  const Phys P = make_phys(1.4, 1e-10, 1e-10, slope_theta, kNotRead, slope_type, 10);
  for (int i = 0; i < n; i++) dq[i] = slope_lcr<3, -1>(ql[i], qc[i], qr[i], P);
}

// unsplit (hydro/umuscl.f90:22) on ONE 6x6x6 patch assembled from the per-cell device functions in the order the sweep kernel
// uses them: ctoprim -> slope_lcr per direction -> trace_sources -> trace_faces -> riemann per face -> flux*dt/dx.
// uin and flux use the oracle's array layout with nvector=1: uin[ivar*216 + (i+1) + 6*((j+1) + 6*(k+1))], i,j,k = -1..4;
// flux[(ivar + 5*idim)*27 + (i-1) + 3*((j-1) + 3*(k-1))], faces 1..3.  slope_type 3 is not covered (27-point limiter).
void devnum_unsplit3d(int solver, int slope_type, double slope_theta, const double* uin, double dx, double dt, double* flux,
                      double gamma, double smallr, double smallc, int niter) {
  const Phys P = make_phys(gamma, smallr, smallc, slope_theta, kNotRead, slope_type, niter);
  static double q[6][6][6][5], rinv[6][6][6], qm[6][6][6][3][5], qp[6][6][6][3][5];
  for (int k = 0; k < 6; k++)
    for (int j = 0; j < 6; j++)
      for (int i = 0; i < 6; i++) {
        double u[5];
        for (int v = 0; v < 5; v++) u[v] = uin[v * 216 + i + 6 * (j + 6 * k)];
        ctoprim<3>(u, q[k][j][i], P);
        rinv[k][j][i] = rcp_rn(q[k][j][i][0]);
      }
  const double dtdx = dt / dx;
  for (int k = 1; k <= 4; k++)
    for (int j = 1; j <= 4; j++)
      for (int i = 1; i <= 4; i++) {
        double dq[3][5], s0[5];
        for (int v = 0; v < 5; v++) {
          dq[0][v] = slope_lcr<3, -1>(q[k][j][i - 1][v], q[k][j][i][v], q[k][j][i + 1][v], P);
          dq[1][v] = slope_lcr<3, -1>(q[k][j - 1][i][v], q[k][j][i][v], q[k][j + 1][i][v], P);
          dq[2][v] = slope_lcr<3, -1>(q[k - 1][j][i][v], q[k][j][i][v], q[k + 1][j][i][v], P);
        }
        trace_sources<3>(q[k][j][i], dq, rinv[k][j][i], s0, P);
        for (int d = 0; d < 3; d++) trace_faces<3>(q[k][j][i], dq[d], s0, dtdx, qm[k][j][i][d], qp[k][j][i][d], P);
      }
  static const int perm[3][5] = {{0, 1, 4, 2, 3}, {0, 2, 4, 1, 3}, {0, 3, 4, 1, 2}};   // (rho, u_n, P, u_t1, u_t2): cmpflxm :749-789
  for (int d = 0; d < 3; d++) {
    const int i0 = d == 0, j0 = d == 1, k0 = d == 2;
    for (int k3 = 1; k3 <= 2 + k0; k3++)
      for (int j3 = 1; j3 <= 2 + j0; j3++)
        for (int i3 = 1; i3 <= 2 + i0; i3++) {
          const double* m_ = qm[k3 + 1 - k0][j3 + 1 - j0][i3 + 1 - i0][d];   // Fortran cell (i3-1,...) -> C index +1
          const double* p_ = qp[k3 + 1][j3 + 1][i3 + 1][d];
          double ql[5], qr[5], fg[5];
          for (int v = 0; v < 5; v++) { ql[v] = m_[perm[d][v]]; qr[v] = p_[perm[d][v]]; }
          if (solver == RIEMANN_LLF) riemann<3, RIEMANN_LLF>(ql, qr, fg, P);
          else if (solver == RIEMANN_EXACT) riemann<3, RIEMANN_EXACT>(ql, qr, fg, P);
          else if (solver == RIEMANN_ACOUSTIC) riemann<3, RIEMANN_ACOUSTIC>(ql, qr, fg, P);
          else if (solver == RIEMANN_HLLC) riemann<3, RIEMANN_HLLC>(ql, qr, fg, P);
          else riemann<3, RIEMANN_HLL>(ql, qr, fg, P);
          for (int v = 0; v < 5; v++)
            flux[(perm[d][v] + 5 * d) * 27 + (i3 - 1) + 3 * ((j3 - 1) + 3 * (k3 - 1))] = fg[v] * dt / dx;
        }
  }
}

// tree walks of the AMR kernels on a host copy of the tree arrays (1-based Fortran arrays handed over as 0-based views)
void devnum_amr_get3cubefather(int ndim, int ncoarse, int ngridmax, int nx, int ny, int nz, const int* son, const int* father,
                               const int* nbor, int n, const int* igrid, int ilevel, int* nfc /*[n][3^ndim]*/) {
  AmrTree t;
  t.son = son - 1; t.father = father - 1; t.nbor = nbor; t.ncoarse = ncoarse; t.ngridmax = ngridmax; t.nx = nx; t.ny = ny; t.nz = nz;
  t.ncell = (long long)ncoarse + (long long)(1 << ndim) * ngridmax;
  const int n3 = ndim == 1 ? 3 : (ndim == 2 ? 9 : 27);
  for (int i = 0; i < n; i++) {
    int ng[8];
    if (ndim == 1) amr_get3cubefather<1>(t, igrid[i], ilevel, nfc + i * n3, ng);
    else if (ndim == 2) amr_get3cubefather<2>(t, igrid[i], ilevel, nfc + i * n3, ng);
    else amr_get3cubefather<3>(t, igrid[i], ilevel, nfc + i * n3, ng);
  }
}

void devnum_amr_getnborfather(int ndim, int ncoarse, int ngridmax, int nx, int ny, int nz, const int* son, const int* father,
                              const int* nbor, int n, const int* cells, int ilevel, int* fa /*[n][2*ndim+1]*/) {
  AmrTree t;
  t.son = son - 1; t.father = father - 1; t.nbor = nbor; t.ncoarse = ncoarse; t.ngridmax = ngridmax; t.nx = nx; t.ny = ny; t.nz = nz;
  t.ncell = (long long)ncoarse + (long long)(1 << ndim) * ngridmax;
  for (int i = 0; i < n; i++) {
    if (ndim == 1) amr_getnborfather<1>(t, cells[i], ilevel, fa + i * 3);
    else if (ndim == 2) amr_getnborfather<2>(t, cells[i], ilevel, fa + i * 5);
    else amr_getnborfather<3>(t, cells[i], ilevel, fa + i * 7);
  }
}

// amr_hydro_flag_kernel (hydro_flag + hydro_refine on the device) over the active octs of one level, thread by thread
void devnum_amr_hydro_flag(int ndim, int ncoarse, int ngridmax, int nx, int ny, int nz, const int* son, const int* father,
                           const int* nbor, const int* active, int nact, int ilevel, const double* uold, double gamma,
                           double smallr, const double* err, const double* flo, int* out /*[nact][2^ndim]*/) {
  AmrTree t;
  t.son = son - 1; t.father = father - 1; t.nbor = nbor; t.ncoarse = ncoarse; t.ngridmax = ngridmax; t.nx = nx; t.ny = ny; t.nz = nz;
  t.ncell = (long long)ncoarse + (long long)(1 << ndim) * ngridmax;
  const int n = nact * (1 << ndim), nb = (n + 127) / 128;
  rgpu_stub_sync_hook = nullptr;
  for (int b = 0; b < nb; b++)
    for (int th = 0; th < 128; th++) {
      threadIdx = {(unsigned)th, 0, 0}; blockIdx = {(unsigned)b, 0, 0}; blockDim = {128, 1, 1}; gridDim = {(unsigned)nb, 1, 1};
      if (ndim == 1) amr_hydro_flag_kernel<1>(t, uold, active, nact, ilevel, gamma, smallr, err[0], err[1], err[2], flo[0], flo[1], flo[2], out);
      else if (ndim == 2) amr_hydro_flag_kernel<2>(t, uold, active, nact, ilevel, gamma, smallr, err[0], err[1], err[2], flo[0], flo[1], flo[2], out);
      else amr_hydro_flag_kernel<3>(t, uold, active, nact, ilevel, gamma, smallr, err[0], err[1], err[2], flo[0], flo[1], flo[2], out);
    }
}

// interpol_hydro for one variable: a [n][2*ndim+1] -> u2 [n][2^ndim]
void devnum_amr_interpol(int ndim, int interpol_type, int n, const double* a, double* u2) {
  const int na = 2 * ndim + 1, T = 1 << ndim;
  for (int i = 0; i < n; i++) {
    if (ndim == 1) amr_interpol_var<1>(a + i * na, interpol_type, u2 + i * T);
    else if (ndim == 2) amr_interpol_var<2>(a + i * na, interpol_type, u2 + i * T);
    else amr_interpol_var<3>(a + i * na, interpol_type, u2 + i * T);
  }
}

void devnum_amr_interpol_full(int ndim, int interpol_type, int interpol_var, int n, const double* u1, double* u2, double smallr) {
  if (ndim == 1) interpol_full_nd<1>(interpol_type, interpol_var, n, u1, u2, smallr);
  else if (ndim == 2) interpol_full_nd<2>(interpol_type, interpol_var, n, u1, u2, smallr);
  else interpol_full_nd<3>(interpol_type, interpol_var, n, u1, u2, smallr);
}

// amr_godfine_kernel (the oct-batch kernel of AMR mode) run by the emulated launch on host copies of the arrays: updates unew of
// the level's own cells and writes the outer-face fluxes rflux [nact][2*ndim][2^(ndim-1)][nvar]
void devnum_amr_godfine(int ndim, int solver, int ncoarse, int ngridmax, int nx, int ny, int nz, const int* son, const int* father,
                        const int* nbor, const int* active, int nact, int ilevel, const double* uold, double* unew, double* rflux,
                        double dt, double dx, int interpol_type, int slope_type, double slope_theta, double gamma, double smallr,
                        double smallc, int niter, double difmag) {
  AmrSweepArgs a;
  std::memset(&a, 0, sizeof a);
  a.t.son = son - 1; a.t.father = father - 1; a.t.nbor = nbor; a.t.ncoarse = ncoarse; a.t.ngridmax = ngridmax;
  a.t.nx = nx; a.t.ny = ny; a.t.nz = nz; a.t.ncell = (long long)ncoarse + (long long)(1 << ndim) * ngridmax;
  a.active = active; a.nact = nact; a.ilevel = ilevel; a.uold = uold; a.unew = unew; a.rflux = rflux;
  a.P = make_phys(gamma, smallr, smallc, slope_theta, kNotRead, slope_type, niter);
  a.dt = dt; a.dx = dx; a.inv_dx = 1.0 / dx;
  int ex;
  a.dx_pow2 = (std::frexp(dx, &ex) == 0.5) ? 1 : 0;
  a.interpol_type = interpol_type; a.difmag = difmag; a.nps = 0; a.flux_only = 0; a.rflux_index = nullptr; a.dt_dev = nullptr;
  const int nb = (nact + AMR_OPB - 1) / AMR_OPB, nt = AMR_TPO * AMR_OPB;
#define RUN(ND, RS)                                                              \
  do {                                                                          \
    if (difmag > 0.0) emulate_launch(amr_godfine_kernel<ND, RS, true, 0>, a, nb, nt); \
    else emulate_launch(amr_godfine_kernel<ND, RS, false, 0>, a, nb, nt);        \
  } while (0)
#define RUN_ND(ND)                                                                                              \
  do {                                                                                                          \
    if (solver == RIEMANN_LLF) RUN(ND, RIEMANN_LLF); else if (solver == RIEMANN_EXACT) RUN(ND, RIEMANN_EXACT);   \
    else if (solver == RIEMANN_ACOUSTIC) RUN(ND, RIEMANN_ACOUSTIC); else if (solver == RIEMANN_HLLC) RUN(ND, RIEMANN_HLLC); \
    else RUN(ND, RIEMANN_HLL);                                                                                  \
  } while (0)
  if (ndim == 1) RUN_ND(1); else if (ndim == 2) RUN_ND(2); else RUN_ND(3);
#undef RUN_ND
#undef RUN
}

// godunov_fine of one level with the plain oct-batch kernel: kernel + coarse reflux pass with the bind-time schedule (what
// rgpu_godunov_fine does in AMR mode).  uold/unew [nvar][ncell], nvar = ndim+2.
void devnum_amr_godunov(int ndim, int solver, int ncoarse, int ngridmax, int nx, int ny, int nz, const int* son, const int* father,
                        const int* nbor, const int* active, int nact, int ilevel, const double* uold, double* unew, double dt, double dx,
                        int interpol_type, int slope_type, double slope_theta, double gamma, double smallr, double smallc, int niter,
                        int nvector) {
  const int nvar = ndim + 2, TW = 2 * ndim, NSF = 1 << (ndim - 1);
  std::vector<double> rflux((size_t)std::max(1, nact) * TW * NSF * nvar, 0.0);
  devnum_amr_godfine(ndim, solver, ncoarse, ngridmax, nx, ny, nz, son, father, nbor, active, nact, ilevel, uold, unew, rflux.data(), dt, dx,
                     interpol_type, slope_type, slope_theta, gamma, smallr, smallc, niter, 0.0);
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
}

// ---- poisson / pressure_fix (the SRC instantiation of the oct-batch kernel and the list passes of set_unew / set_uold) ------------
// unew holds nvar+2 columns when pfix (divu, enew behind the state); rflux [nact][2*ndim][2^(ndim-1)][nvar(+2)]
void devnum_amr_godfine_src(int ndim, int solver, int ncoarse, int ngridmax, int nx, int ny, int nz, const int* son, const int* father,
                            const int* nbor, const int* active, int nact, int ilevel, const double* uold, double* unew, double* rflux,
                            double dt, double dx, int interpol_type, int slope_type, double slope_theta, double gamma, double smallr,
                            double smallc, int niter, const double* force, int pfix, int nvector_reflux) {
  AmrSweepArgs a;
  std::memset(&a, 0, sizeof a);
  a.t.son = son - 1; a.t.father = father - 1; a.t.nbor = nbor; a.t.ncoarse = ncoarse; a.t.ngridmax = ngridmax;
  a.t.nx = nx; a.t.ny = ny; a.t.nz = nz; a.t.ncell = (long long)ncoarse + (long long)(1 << ndim) * ngridmax;
  a.active = active; a.nact = nact; a.ilevel = ilevel; a.uold = uold; a.unew = unew; a.rflux = rflux;
  a.P = make_phys(gamma, smallr, smallc, slope_theta, kNotRead, slope_type, niter);
  a.dt = dt; a.dx = dx; a.inv_dx = 1.0 / dx;
  int ex;
  a.dx_pow2 = (std::frexp(dx, &ex) == 0.5) ? 1 : 0;
  a.interpol_type = interpol_type; a.force = force; a.pfix = pfix; a.nvr = ndim + 2 + (pfix ? 2 : 0);
  const int nb = (nact + AMR_OPB - 1) / AMR_OPB, nt = AMR_TPO * AMR_OPB;
#define RUN(ND, RS) emulate_launch(amr_godfine_kernel<ND, RS, false, 0, true>, a, nb, nt)
#define RUN_ND(ND)                                                                                              \
  do {                                                                                                          \
    if (solver == RIEMANN_LLF) RUN(ND, RIEMANN_LLF); else if (solver == RIEMANN_EXACT) RUN(ND, RIEMANN_EXACT);   \
    else if (solver == RIEMANN_ACOUSTIC) RUN(ND, RIEMANN_ACOUSTIC); else if (solver == RIEMANN_HLLC) RUN(ND, RIEMANN_HLLC); \
    else RUN(ND, RIEMANN_HLL);                                                                                  \
  } while (0)
  if (ndim == 1) RUN_ND(1); else if (ndim == 2) RUN_ND(2); else RUN_ND(3);
#undef RUN_ND
#undef RUN
  // coarse reflux of the state AND of divu / enew (hydro/godunov_fine.f90:798-908) with the schedule rgpu_api.cu builds at bind time
  std::vector<int> cells, start, srcs, src;
  build_reflux_schedule(ndim, nvector_reflux, nact, active, nbor, son, ngridmax, cells, start, srcs, src);
  if (!cells.empty()) {
    RefluxArgs r;
    std::memset(&r, 0, sizeof r);
    r.nent = (int)cells.size(); r.cell = cells.data(); r.start = start.data(); r.src = srcs.data(); r.rflux = rflux; r.unew = unew;
    r.ncell = a.t.ncell; r.nvar = a.nvr; r.nsides = 2 * ndim; r.nsf = 1 << (ndim - 1); r.oneontwotondim = 1.0 / (double)(1 << ndim);
    emulate_serial(amr_reflux_kernel, r, (r.nent * r.nvar + 127) / 128, 128);
  }
}

// kind 0: amr_pfix_init_kernel, 1: amr_gravity_src_kernel, 2: amr_pdv_kernel, 3: amr_pfix_switch_kernel -- run thread after thread
void devnum_amr_src_pass(int kind, int ndim, int ncoarse, int ngridmax, int nx, int ny, int nz, const int* son, const int* father,
                         const int* nbor, const int* active, int nact, double* uold, double* unew, double* divu, double* enew,
                         const double* force, double gamma, double smallr, double beta_fix, double dx, double dt) {
  AmrTree t;
  std::memset(&t, 0, sizeof t);
  t.son = son - 1; t.father = father - 1; t.nbor = nbor; t.ncoarse = ncoarse; t.ngridmax = ngridmax; t.nx = nx; t.ny = ny; t.nz = nz;
  t.ncell = (long long)ncoarse + (long long)(1 << ndim) * ngridmax;
  const int T = 1 << ndim, n = nact * T, nb = (n + 127) / 128;
  for (int b = 0; b < nb; b++)
    for (int th = 0; th < 128; th++) {
      threadIdx = {(unsigned)th, 0, 0}; blockIdx = {(unsigned)b, 0, 0}; blockDim = {128, 1, 1}; gridDim = {(unsigned)nb, 1, 1};
      if (kind == 0) amr_pfix_init_kernel(uold, divu, enew, active, nact, ncoarse, ngridmax, t.ncell, T, ndim, smallr);
      else if (kind == 1) amr_gravity_src_kernel(uold, unew, force, active, nact, ncoarse, ngridmax, t.ncell, T, ndim, smallr, dt, nullptr);
      else if (kind == 2) amr_pdv_kernel(t, uold, enew, active, nact, ndim, gamma, smallr, dx, dt, nullptr);
      else amr_pfix_switch_kernel(uold, divu, enew, active, nact, ncoarse, ngridmax, t.ncell, T, ndim, smallr, beta_fix, dx, dt, nullptr);
    }
}

// n cells: dt = cmpdt_cell(u, dx, sum|g|)
void devnum_cmpdt_grav(int ndim, int n, const double* u, const double* gsum, double dx, double* dt, double gamma, double smallr,
                       double smallc, double cfl) {
  const Phys P = make_phys(gamma, smallr, smallc, kNotRead, cfl, 1, 10);
  const int nv = ndim + 2;
  for (int i = 0; i < n; i++) {
    double ei;
    if (ndim == 1) dt[i] = cmpdt_cell<1>(u + i * nv, dx, P, ei, gsum[i]);
    else if (ndim == 2) dt[i] = cmpdt_cell<2>(u + i * nv, dx, P, ei, gsum[i]);
    else dt[i] = cmpdt_cell<3>(u + i * nv, dx, P, ei, gsum[i]);
  }
}

// n Riemann problems, internal-energy flux fgdnv(nvar+1) only (pressure_fix)
void devnum_riemann_eflux(int ndim, int solver, int n, const double* ql, const double* qr, double* fe, double gamma, double smallr,
                          double smallc, int niter) {
  const Phys P = make_phys(gamma, smallr, smallc, kNotRead, kNotRead, 1, niter);
  const int nv = ndim + 2;
  for (int i = 0; i < n; i++) {
    double fg[5];
#define RE(ND)                                                                                                      \
    switch (solver) {                                                                                               \
      case RIEMANN_LLF: riemann<ND, RIEMANN_LLF>(ql + i * nv, qr + i * nv, fg, P, fe + i); break;                    \
      case RIEMANN_EXACT: riemann<ND, RIEMANN_EXACT>(ql + i * nv, qr + i * nv, fg, P, fe + i); break;                \
      case RIEMANN_ACOUSTIC: riemann<ND, RIEMANN_ACOUSTIC>(ql + i * nv, qr + i * nv, fg, P, fe + i); break;          \
      case RIEMANN_HLLC: riemann<ND, RIEMANN_HLLC>(ql + i * nv, qr + i * nv, fg, P, fe + i); break;                  \
      default: riemann<ND, RIEMANN_HLL>(ql + i * nv, qr + i * nv, fg, P, fe + i); break;                             \
    }
    if (ndim == 1) { RE(1) } else if (ndim == 2) { RE(2) } else { RE(3) }
#undef RE
  }
}

static MPhys make_mphys(double gamma, double smallr, double smallc, double slope_theta, double courant_factor) {
  MPhys M;
  M.gamma = gamma; M.smallr = smallr; M.smallc = smallc; M.slope_theta = slope_theta; M.courant_factor = courant_factor;
  M.smallp = smallr * (smallc * smallc) / gamma;
  M.slope_type = 1; M.slope_mag_type = 1;
  return M;
}

// ---- ideal MHD in AMR mode (mhd_amr.cuh): godunov_fine of one level = godfine kernel + Euler reflux + (2-D) EMF reflux, with the
// schedules of amr_schedules.h exactly as rgpu_api.cu builds them at bind time.  uold/unew [11][ncell].
void devnum_mhd_amr_godunov(int ndim, int ncoarse, int ngridmax, int nx, int ny, int nz, const int* son, const int* father, const int* nbor,
                            const int* active, int nact, int ilevel, const double* uold, double* unew, double dt, double dx,
                            int interpol_type, int interpol_mag_type, int riemann, int riemann2d, int slope_type, int slope_mag_type,
                            double gamma, double smallr, double smallc, int nvector) {
  MhdAmrArgs a;
  std::memset(&a, 0, sizeof a);
  a.t.son = son - 1; a.t.father = father - 1; a.t.nbor = nbor; a.t.ncoarse = ncoarse; a.t.ngridmax = ngridmax;
  a.t.nx = nx; a.t.ny = ny; a.t.nz = nz; a.t.ncell = (long long)ncoarse + (long long)(1 << ndim) * ngridmax;
  const int TW = 2 * ndim, NSF = 1 << (ndim - 1);
  std::vector<double> rflux((size_t)std::max(1, nact) * TW * NSF * MNV, 0.0), remf((size_t)std::max(1, nact) * (ndim == 3 ? 81 : 4), 0.0);
  a.active = active; a.nact = nact; a.ilevel = ilevel; a.uold = uold; a.unew = unew; a.rflux = rflux.data(); a.remf = remf.data();
  a.P = make_mphys(gamma, smallr, smallc, kNotRead, kNotRead);   // the AMR kernels build slopes 0-2 and no Courant step
  a.P.slope_type = slope_type; a.P.slope_mag_type = slope_mag_type;
  a.dt = dt; a.dx = dx; a.dt_dev = nullptr;
  a.interpol_type = interpol_type; a.interpol_mag_type = interpol_mag_type < 0 ? interpol_type : interpol_mag_type;
  a.riemann = riemann; a.riemann2d = riemann2d;
  if (ndim == 1) emulate_serial(mhd_amr1_godfine_kernel, a, (nact + 63) / 64, 64);
  else if (ndim == 2) emulate_launch(mhd_amr2_godfine_kernel, a, nact, MHD2_TPO);
  else emulate_launch(mhd_amr3_godfine_kernel, a, nact, MHD3_TPO, 1, sizeof(Mhd3Sm) / sizeof(double) + 1);
  std::vector<int> cells, start, srcs, src;
  build_reflux_schedule(ndim, nvector, nact, active, nbor, son, ngridmax, cells, start, srcs, src);
  if (!cells.empty()) {
    RefluxArgs r;
    std::memset(&r, 0, sizeof r);
    r.nent = (int)cells.size(); r.cell = cells.data(); r.start = start.data(); r.src = srcs.data(); r.rflux = rflux.data(); r.unew = unew;
    r.ncell = a.t.ncell; r.nvar = MNVS; r.nsides = TW; r.nsf = NSF; r.oneontwotondim = 1.0 / (double)(1 << ndim);
    emulate_serial(mhd_amr_reflux_kernel, r, (r.nent * MNVS + 127) / 128, 128);
  }
  if (ndim == 2 && nact > 0) {
    std::vector<int> nfc((size_t)nact * 9);
    for (int i = 0; i < nact; i++) {
      int f[27], ng[8];
      amr_get3cubefather<2>(a.t, active[i], ilevel, f, ng);
      for (int j = 0; j < 9; j++) nfc[(size_t)i * 9 + j] = f[j];
    }
    std::vector<int> ec, ev, es, ecode;
    build_emf_schedule_2d(nvector, nact, nfc.data(), son, ec, ev, es, ecode);
    if (!ec.empty()) {
      EmfRefluxArgs r;
      std::memset(&r, 0, sizeof r);
      r.nent = (int)ec.size(); r.cell = ec.data(); r.var = ev.data(); r.start = es.data(); r.code = ecode.data(); r.remf = remf.data();
      r.unew = unew; r.ncell = a.t.ncell;
      emulate_serial(mhd_amr_emf_reflux_kernel, r, (r.nent + 127) / 128, 128);
    }
  }
  if (ndim == 3 && nact > 0) {
    std::vector<int> nfc((size_t)nact * 27);
    for (int i = 0; i < nact; i++) {
      int f[27], ng[8];
      amr_get3cubefather<3>(a.t, active[i], ilevel, f, ng);
      for (int j = 0; j < 27; j++) nfc[(size_t)i * 27 + j] = f[j];
    }
    std::vector<int> ec, ev, es, ecode;
    build_emf_schedule_3d(nvector, nact, nfc.data(), son, ec, ev, es, ecode);
    if (!ec.empty()) {
      Emf3RefluxArgs r;
      std::memset(&r, 0, sizeof r);
      r.nent = (int)ec.size(); r.cell = ec.data(); r.var = ev.data(); r.start = es.data(); r.code = ecode.data(); r.remf = remf.data();
      r.unew = unew; r.ncell = a.t.ncell;
      const MhdEdge3Host* E = mhd_edges3();
      for (int e = 0; e < 12; e++) {
        r.edir[e] = (signed char)E[e].dir;
        r.ec0[e] = (signed char)(((E[e].c[0][2] - 1) * 3 + (E[e].c[0][1] - 1)) * 3 + (E[e].c[0][0] - 1));
        r.ec1[e] = (signed char)(((E[e].c[1][2] - 1) * 3 + (E[e].c[1][1] - 1)) * 3 + (E[e].c[1][0] - 1));
      }
      emulate_serial(mhd_amr_emf3_reflux_kernel, r, (r.nent + 127) / 128, 128);
    }
  }
}

// kind 0: upload_fine (both passes), 1: make_boundary_hydro (NDIM = 1; dir, bkind), 2: per-cell Courant steps of the leaf cells -> dtc[nact*T]
void devnum_mhd_amr_pass(int kind, int ndim, int ncoarse, int ngridmax, int nx, int ny, int nz, const int* son, const int* father,
                         const int* nbor, const int* list, int n, double* u, double gamma, double smallr, double smallc, double cfl,
                         double dx, int dir, int bkind, double* dtc) {
  AmrTree t;
  std::memset(&t, 0, sizeof t);
  t.son = son - 1; t.father = father - 1; t.nbor = nbor; t.ncoarse = ncoarse; t.ngridmax = ngridmax; t.nx = nx; t.ny = ny; t.nz = nz;
  t.ncell = (long long)ncoarse + (long long)(1 << ndim) * ngridmax;
  const int T = 1 << ndim;
  const MPhys P = make_mphys(gamma, smallr, smallc, kNotRead, cfl);
  if (kind == 0) {
    for (int pass = 0; pass < 2; pass++)
      for (int b = 0; b < (n * T + 127) / 128; b++)
        for (int th = 0; th < 128; th++) {
          threadIdx = {(unsigned)th, 0, 0}; blockIdx = {(unsigned)b, 0, 0}; blockDim = {128, 1, 1}; gridDim = {1, 1, 1};
          mhd_amr_upload_kernel(u, t, list, n, ndim, smallr, pass);
        }
  } else if (kind == 1) {
    MhdAmrBoundArgs bb;
    bb.n = n; bb.igrid = list; bb.dir = dir; bb.kind = bkind; bb.smallr = smallr;
    for (int b = 0; b < (n * 2 + 127) / 128; b++)
      for (int th = 0; th < 128; th++) {
        threadIdx = {(unsigned)th, 0, 0}; blockIdx = {(unsigned)b, 0, 0}; blockDim = {128, 1, 1}; gridDim = {1, 1, 1};
        mhd_amr1_boundary_kernel(u, t, bb);
      }
  } else {
    for (int o = 0; o < n; o++)
      for (int ind = 0; ind < T; ind++) {
        const int ic = amr_cell(t, ind, list[o]);
        double uu[MNVS];
        for (int k = 0; k < MNVS; k++) uu[k] = u[(size_t)k * t.ncell + ic - 1];
        dtc[o * T + ind] = (t.son[ic] != 0) ? 1e300 : mhd_cmpdt_cell_nd(P, uu, dx, ndim);
      }
  }
}

// n MHD Riemann problems in solver order (rho, P, v_n, B_n, v_t1, B_t1, v_t2, B_t2): fg [n][9]
void devnum_mhd_riemann(int solver, int n, const double* ql, const double* qr, double* fg, double gamma, double smallr, double smallc) {
  const MPhys M = make_mphys(gamma, smallr, smallc, kNotRead, kNotRead);
  for (int i = 0; i < n; i++) {
    real l[8], r[8], f[9];
    for (int k = 0; k < 8; k++) { l[k] = ql[i * 8 + k]; r[k] = qr[i * 8 + k]; }
    switch (solver) {
      case MHD_LLF: riemann1d<MHD_LLF>(M, l, r, f); break;
      case MHD_ROE: riemann1d<MHD_ROE>(M, l, r, f); break;
      case MHD_HLL: riemann1d<MHD_HLL>(M, l, r, f); break;
      case MHD_HLLD: riemann1d<MHD_HLLD>(M, l, r, f); break;
      case MHD_UPWIND: riemann1d<MHD_UPWIND>(M, l, r, f); break;
      default: riemann1d<MHD_HYDRO>(M, l, r, f); break;
    }
    for (int k = 0; k < 9; k++) fg[i * 9 + k] = (double)f[k];
  }
}

// n corner EMFs from the four states (qLL, qRL, qLR, qRR) [n][8] in cmp_mag_flx's solver order
void devnum_mhd_emf(int solver2d, int n, const double* qLL, const double* qRL, const double* qLR, const double* qRR, double* emf,
                    double gamma, double smallr, double smallc) {
  const MPhys M = make_mphys(gamma, smallr, smallc, kNotRead, kNotRead);
  for (int i = 0; i < n; i++) {
    real a[8], b[8], c[8], d[8];
    for (int k = 0; k < 8; k++) { a[k] = qLL[i * 8 + k]; b[k] = qRL[i * 8 + k]; c[k] = qLR[i * 8 + k]; d[k] = qRR[i * 8 + k]; }
    real e;
    switch (solver2d) {
      case MHD2D_LLF: e = emf_edge<MHD2D_LLF>(M, a, b, c, d); break;
      case MHD2D_ROE: e = emf_edge<MHD2D_ROE>(M, a, b, c, d); break;
      case MHD2D_UPWIND: e = emf_edge<MHD2D_UPWIND>(M, a, b, c, d); break;
      case MHD2D_HLL: e = emf_edge<MHD2D_HLL>(M, a, b, c, d); break;
      case MHD2D_HLLA: e = emf_edge<MHD2D_HLLA>(M, a, b, c, d); break;
      default: e = emf_edge<MHD2D_HLLD>(M, a, b, c, d); break;
    }
    emf[i] = (double)e;
  }
}

// the six passes of the dense MHD sweep (mhd_dense.cuh) in the order of launch_mhd_sweep (mhd_inst_misc.cu) on a periodic cube
// of N^3 cells: uin/uout in the device layout [11][8][nslot] (cell_offset of sweep_dense.cuh), N even
// on a box of n[0] x n[1] x n[2] owned cells, each axis periodic or with a 2-cell ghost shell (box_geom)
void devnum_mhd_sweep_box(const int* n, const int* shell, int r1d, int r2d, int sl, const double* uin, double* uout, double dt,
                          double dx, double gamma, double smallr, double smallc, int slope_type, int slope_mag_type, double slope_theta,
                          double courant_factor) {
  MhdArgs a;
  std::memset(&a, 0, sizeof a);
  a.g = box_geom(3, n, shell);
  const DenseGeom& g = a.g;
  a.uin = uin; a.uout = uout;
  a.P = make_mphys(gamma, smallr, smallc, slope_theta, courant_factor);
  a.P.slope_type = slope_type; a.P.slope_mag_type = slope_mag_type;
  a.dt_dev = &dt; a.dx = dx; a.nc = (long long)g.ncx * g.ncy * g.ncz;
  std::vector<double> W((size_t)MW_NCOMP * a.nc, 0.0), part(5 * 64, 0.0);
  a.W = W.data(); a.part = part.data();
  const long long nb256 = (a.nc + 255) / 256, nb128 = (a.nc + 127) / 128;
  emulate_serial(mhd_prim_kernel, a, nb256, 256);
  emulate_serial(mhd_efield_kernel, a, nb256, 256);
  if (sl) emulate_serial(mhd_trace_kernel<true>, a, nb256, 256); else emulate_serial(mhd_trace_kernel<false>, a, nb256, 256);
#define FLUX(R)                                                                                   \
  case R: if (sl) emulate_serial(mhd_flux_kernel<R, true, 2>, a, nb128, 128); else emulate_serial(mhd_flux_kernel<R, false, 2>, a, nb128, 128); break;
  switch (r1d) { FLUX(MHD_LLF) FLUX(MHD_ROE) FLUX(MHD_HLL) FLUX(MHD_HLLD) FLUX(MHD_UPWIND) FLUX(MHD_HYDRO) }
#undef FLUX
#define EMF(R)                                                                                    \
  case R: if (sl) emulate_serial(mhd_emf_kernel<R, true, 2>, a, nb128, 128); else emulate_serial(mhd_emf_kernel<R, false, 2>, a, nb128, 128); break;
  switch (r2d) { EMF(MHD2D_LLF) EMF(MHD2D_ROE) EMF(MHD2D_UPWIND) EMF(MHD2D_HLL) EMF(MHD2D_HLLA) EMF(MHD2D_HLLD) }
#undef EMF
  emulate_serial(mhd_update_kernel, a, 8, 256);
}

// the stand-alone MHD Courant scan (mhd_courant_kernel, mhd_dense.cuh) on a box laid out like devnum_mhd_sweep_box, launched with
// nblocks CTAs of 256 threads like launch_mhd_courant: part[5][nblocks] = per-block min dt, sum rho, sum E, sum eint, sum emag
struct MhdCourantHost { const double* u; DenseGeom g; MPhys P; double dx; double* part; };
void devnum_mhd_courant(const int* n, const int* shell, int nblocks, const double* u, double dx, double gamma, double smallr,
                        double smallc, double cfl, double* part) {
  MhdCourantHost a;
  a.u = u; a.g = box_geom(3, n, shell); a.P = make_mphys(gamma, smallr, smallc, kNotRead, cfl); a.dx = dx; a.part = part;
  emulate_launch([](const MhdCourantHost& c) { mhd_courant_kernel(c.u, c.g, c.P, c.dx, c.part); }, a, nblocks, 256);
}

// make_boundary_hydro of the dense MHD path (mhd_boundary_kernel) for one boundary region of such a box: the MhdBoundArgs that
// launch_boundaries (rgpu_api.cu) builds for boundary type bt and the region's oct slots; u [11][8][nslot] is updated in place
void devnum_mhd_boundary(const int* n, const int* shell, int bt, const int* slots, int nreg, double* u, double smallr) {
  static const int ref_x[8] = {2, 1, 4, 3, 6, 5, 8, 7}, ref_y[8] = {3, 4, 1, 2, 7, 8, 5, 6}, ref_z[8] = {5, 6, 7, 8, 1, 2, 3, 4};
  static const int fre[6][8] = {{1, 1, 3, 3, 5, 5, 7, 7}, {2, 2, 4, 4, 6, 6, 8, 8}, {1, 2, 1, 2, 5, 6, 5, 6},
                                {3, 4, 3, 4, 7, 8, 7, 8}, {1, 2, 3, 4, 1, 2, 3, 4}, {5, 6, 7, 8, 5, 6, 7, 8}};
  static const int alt_[6][8] = {{-2, -1, -2, -1, -2, -1, -2, -1}, {1, 2, 1, 2, 1, 2, 1, 2}, {-2, -2, -1, -1, -2, -2, -1, -1},
                                 {1, 1, 2, 2, 1, 1, 2, 2}, {-2, -2, -2, -2, -1, -1, -1, -1}, {1, 1, 1, 1, 2, 2, 2, 2}};
  const DenseGeom g = box_geom(3, n, shell);
  const long long str[3] = {1, g.nox, (long long)g.nox * g.noy};
  const int dir = bt - 10 * (bt / 10), d = (dir - 1) / 2;
  MhdBoundArgs m;
  std::memset(&m, 0, sizeof m);
  m.n = nreg; m.slots = slots; m.nslot = g.nslot;
  m.nbr_off = (dir % 2 == 1) ? str[d] : -str[d];
  const int* ir = (bt / 10 == 0) ? (d == 0 ? ref_x : d == 1 ? ref_y : ref_z) : fre[dir - 1];
  for (int i = 0; i < 8; i++) { m.ind_ref[i] = ir[i]; m.ind_normal[i] = fre[dir - 1][i]; m.alt[i] = alt_[dir - 1][i]; }
  m.gs[0] = m.gs[1] = m.gs[2] = 1.0;
  if (bt >= 1 && bt <= 6) m.gs[d] = -1.0;
  m.kind = bt / 10; m.gdim = d + 1;
  m.iperp1 = (dir % 2 == 1) ? 4 + m.gdim : 7 + m.gdim;
  m.smallr = smallr;
  struct B { double* u; MhdBoundArgs m; } b{u, m};
  emulate_serial([](const B& x) { mhd_boundary_kernel(x.u, x.m); }, b, (nreg * 8 + 127) / 128, 128);
}

void devnum_mhd_sweep(int N, int r1d, int r2d, int sl, const double* uin, double* uout, double dt, double dx, double gamma,
                      double smallr, double smallc, int slope_type, int slope_mag_type, double slope_theta, double courant_factor) {
  const int n[3] = {N, N, N};
  devnum_mhd_sweep_box(n, k_no_shell, r1d, r2d, sl, uin, uout, dt, dx, gamma, smallr, smallc, slope_type, slope_mag_type, slope_theta,
                       courant_factor);
}

// the fused dense-box sweep (sweep_dense_kernel: persistent CTAs of 32 x BY threads, cp.async staging, warp shuffles in x, shared
// memory exchange in y, plane carry in z, fused set_unew / update / set_uold / Courant scan) on a periodic box of N^ndim cells,
// state in the device layout [nvar][2^ndim][nslot]; nblocks persistent CTAs share the work like on the GPU
// on a box of n[0] x n[1] x n[2] owned cells (1 beyond ndim), each axis periodic or with a 2-cell ghost shell (box_geom)
int devnum_sweep_dense_box(int ndim, int solver, const int* n, const int* shell, int nblocks, const double* uin, double* uout,
                           double dt, double dx, int slope_type, double slope_theta, double courant_factor, double gamma,
                           double smallr, double smallc, int niter, double* part, int late) {
  SweepArgs a;
  std::memset(&a, 0, sizeof a);
  a.g = box_geom(ndim, n, shell);
  const DenseGeom& g = a.g;
  a.uin = uin; a.uout = uout;
  a.P = make_phys(gamma, smallr, smallc, slope_theta, courant_factor, slope_type, niter);
  a.dt_dev = nullptr; a.dt_val = dt; a.dx = dx; a.inv_dx = 1.0 / dx;
  int ex;
  a.dx_pow2 = (std::frexp(dx, &ex) == 0.5) ? 1 : 0;
  const int by = tile_by_default(ndim, solver);
  const int txo = 30, tyo = ndim > 1 ? by - 2 : 1;                          // rgpu_bind_level (rgpu_api.cu)
  a.ntx = (g.ox1 - g.ox0 + txo - 1) / txo;
  a.nty = ndim > 1 ? (g.oy1 - g.oy0 + tyo - 1) / tyo : 1;
  a.nwork = (long long)a.ntx * a.nty * (ndim > 2 ? (g.oz1 - g.oz0) : 1);
  if (nblocks > a.nwork) nblocks = (int)a.nwork;
  a.part = part; a.refined = nullptr;
#define SW(ND, RS, BY)                                                                                                            \
  do {                                                                                                                           \
    if (late) emulate_launch(sweep_dense_kernel<ND, RS, -1, 32, BY, false, true>, a, nblocks, 32, BY, SweepSmem<ND, 32, BY>::doubles + (ND + 2) * 32 * BY); \
    else emulate_launch(sweep_dense_kernel<ND, RS, -1, 32, BY, false, false>, a, nblocks, 32, BY, SweepSmem<ND, 32, BY>::doubles); \
  } while (0)
#define SW_ND(ND, BY)                                                                                    \
  do {                                                                                                   \
    if (solver == RIEMANN_LLF) SW(ND, RIEMANN_LLF, BY); else if (solver == RIEMANN_EXACT) SW(ND, RIEMANN_EXACT, BY);   \
    else if (solver == RIEMANN_ACOUSTIC) SW(ND, RIEMANN_ACOUSTIC, BY); else if (solver == RIEMANN_HLLC) SW(ND, RIEMANN_HLLC, BY); \
    else SW(ND, RIEMANN_HLL, BY);                                                                        \
  } while (0)
  if (ndim == 1) SW_ND(1, 1); else if (ndim == 2) SW_ND(2, 8); else SW_ND(3, 12);
#undef SW_ND
#undef SW
  return nblocks;   // CTAs actually used: part is [4][nblocks]
}

int devnum_sweep_dense(int ndim, int solver, int N, int nblocks, const double* uin, double* uout, double dt, double dx,
                        int slope_type, double slope_theta, double courant_factor, double gamma, double smallr, double smallc, int niter,
                        double* part, int late) {
  const int n[3] = {N, ndim > 1 ? N : 1, ndim > 2 ? N : 1};
  return devnum_sweep_dense_box(ndim, solver, n, k_no_shell, nblocks, uin, uout, dt, dx, slope_type, slope_theta, courant_factor, gamma,
                                smallr, smallc, niter, part, late);
}

// the AMR variant of the dense sweep (AMRV=true: fluxes through faces of refined cells reset to zero, the update ACCUMULATES into
// uout which already holds unew) on a fully refined periodic level of N^3 cells; refined[8][nslot] = son(cell)>0
void devnum_sweep_dense_amr_box(int solver, const int* n, const int* shell, int nblocks, const double* uin, double* uout,
                                const unsigned char* refined, double dt, double dx, int slope_type, double slope_theta, double gamma,
                                double smallr, double smallc, int niter) {
  SweepArgs a;
  std::memset(&a, 0, sizeof a);
  a.g = box_geom(3, n, shell);
  const DenseGeom& g = a.g;
  a.uin = uin; a.uout = uout; a.refined = refined;
  a.P = make_phys(gamma, smallr, smallc, slope_theta, kNotRead, slope_type, niter);   // part = NULL: no Courant partials
  a.dt_dev = nullptr; a.dt_val = dt; a.dx = dx; a.inv_dx = 1.0 / dx;
  int ex;
  a.dx_pow2 = (std::frexp(dx, &ex) == 0.5) ? 1 : 0;
  a.ntx = (g.ox1 - g.ox0 + 29) / 30; a.nty = (g.oy1 - g.oy0 + 9) / 10; a.nwork = (long long)a.ntx * a.nty * (g.oz1 - g.oz0);
  if (nblocks > a.nwork) nblocks = (int)a.nwork;
  a.part = nullptr;
#define SWA(RS) emulate_launch(sweep_dense_kernel<3, RS, -1, 32, 12, true, false>, a, nblocks, 32, 12, SweepSmem<3, 32, 12>::doubles)
  if (solver == RIEMANN_LLF) SWA(RIEMANN_LLF); else if (solver == RIEMANN_EXACT) SWA(RIEMANN_EXACT);
  else if (solver == RIEMANN_ACOUSTIC) SWA(RIEMANN_ACOUSTIC); else if (solver == RIEMANN_HLLC) SWA(RIEMANN_HLLC); else SWA(RIEMANN_HLL);
#undef SWA
}

void devnum_sweep_dense_amr(int solver, int N, int nblocks, const double* uin, double* uout, const unsigned char* refined, double dt,
                            double dx, int slope_type, double slope_theta, double gamma, double smallr, double smallc, int niter) {
  const int n[3] = {N, N, N};
  devnum_sweep_dense_amr_box(solver, n, k_no_shell, nblocks, uin, uout, refined, dt, dx, slope_type, slope_theta, gamma, smallr, smallc,
                             niter);
}


// lane-generic solvers of hydro_vec.cuh: n 3-D Riemann problems through (a) the branch-free scalar form riemann_v<R,double>
// and (b) the 3-lane form riemann_v<R,V3> (problems i, i+1, i+2 in lanes a, b, c; n must be a multiple of 3)
void devnum_riemann_vec(int solver, int n, const double* ql, const double* qr, double* fg_scalar, double* fg_v3, double gamma,
                        double smallr, double smallc, int niter) {
  const Phys P = make_phys(gamma, smallr, smallc, kNotRead, kNotRead, 1, niter);
  auto run1 = [&](const double* l, const double* r, double* f) {
    switch (solver) {
      case RIEMANN_LLF: riemann_v<RIEMANN_LLF, double>(l, r, f, P); break;
      case RIEMANN_EXACT: riemann_v<RIEMANN_EXACT, double>(l, r, f, P); break;
      case RIEMANN_ACOUSTIC: riemann_v<RIEMANN_ACOUSTIC, double>(l, r, f, P); break;
      case RIEMANN_HLLC: riemann_v<RIEMANN_HLLC, double>(l, r, f, P); break;
      default: riemann_v<RIEMANN_HLL, double>(l, r, f, P); break;
    }
  };
  auto run3 = [&](const V3* l, const V3* r, V3* f) {
    switch (solver) {
      case RIEMANN_LLF: riemann_v<RIEMANN_LLF, V3>(l, r, f, P); break;
      case RIEMANN_EXACT: riemann_v<RIEMANN_EXACT, V3>(l, r, f, P); break;
      case RIEMANN_ACOUSTIC: riemann_v<RIEMANN_ACOUSTIC, V3>(l, r, f, P); break;
      case RIEMANN_HLLC: riemann_v<RIEMANN_HLLC, V3>(l, r, f, P); break;
      default: riemann_v<RIEMANN_HLL, V3>(l, r, f, P); break;
    }
  };
  for (int i = 0; i < n; i++) run1(ql + i * 5, qr + i * 5, fg_scalar + i * 5);
  for (int i = 0; i + 2 < n; i += 3) {
    V3 l[5], r[5], f[5];
    for (int k = 0; k < 5; k++) {
      l[k] = {ql[i * 5 + k], ql[(i + 1) * 5 + k], ql[(i + 2) * 5 + k]};
      r[k] = {qr[i * 5 + k], qr[(i + 1) * 5 + k], qr[(i + 2) * 5 + k]};
    }
    run3(l, r, f);
    for (int k = 0; k < 5; k++) { fg_v3[i * 5 + k] = f[k].a; fg_v3[(i + 1) * 5 + k] = f[k].b; fg_v3[(i + 2) * 5 + k] = f[k].c; }
  }
}

// sweep3_kernel (sweep_dense3.cuh) on a periodic box of N^3 cells, emulated launch; by in {8, 12, 16}, vec in {0, 1, 2}
// on a box of n[0] x n[1] x n[2] owned cells, each axis periodic or with a 2-cell ghost shell (box_geom)
int devnum_sweep3_box(int solver, const int* n, const int* shell, int nblocks, const double* uin, double* uout, double dt, double dx,
                      int slope_type, double slope_theta, double courant_factor, double gamma, double smallr, double smallc, int niter,
                      double* part, int by, int vec) {
  SweepArgs a;
  std::memset(&a, 0, sizeof a);
  a.g = box_geom(3, n, shell);
  const DenseGeom& g = a.g;
  a.uin = uin; a.uout = uout;
  a.P = make_phys(gamma, smallr, smallc, slope_theta, courant_factor, slope_type, niter);
  a.dt_dev = nullptr; a.dt_val = dt; a.dx = dx; a.inv_dx = 1.0 / dx;
  int ex;
  a.dx_pow2 = (std::frexp(dx, &ex) == 0.5) ? 1 : 0;
  a.ntx = (g.ox1 - g.ox0 + 29) / 30; a.nty = (g.oy1 - g.oy0 + by - 3) / (by - 2);   // rgpu_bind_level (rgpu_api.cu)
  a.nwork = (long long)a.ntx * a.nty * (g.oz1 - g.oz0);
  if (nblocks > a.nwork) nblocks = (int)a.nwork;
  a.part = part; a.refined = nullptr;
#define S3(RS, BY, VEC) emulate_launch(sweep3_kernel<RS, -1, BY, 1, VEC>, a, nblocks, 32, BY, Sweep3Smem<BY>::doubles)
#define S3C(RS, BY) emulate_launch(sweep3_kernel<RS, -1, BY, 1, 2, true>, a, nblocks, 32, BY, Sweep3Smem<BY>::doubles)
#define S4(RS, BY, ORD) emulate_launch(sweep4_kernel<RS, -1, BY, 2, ORD>, a, nblocks, 32, BY, Sweep4Smem<BY>::doubles)
#define S3V(RS, BY) do { if (vec == 0) S3(RS, BY, 0); else if (vec == 1) S3(RS, BY, 1); else if (vec == 12) S3C(RS, BY); else if (vec == 40) S4(RS, BY, 0); \
                         else if (vec == 41) S4(RS, BY, 1); else if (vec == 42) S4(RS, BY, 2); else S3(RS, BY, 2); } while (0)
#define S3B(RS) do { if (by == 8) S3V(RS, 8); else if (by == 16) S3V(RS, 16); else S3V(RS, 12); } while (0)
  if (solver == RIEMANN_LLF) S3B(RIEMANN_LLF); else if (solver == RIEMANN_EXACT) S3B(RIEMANN_EXACT);
  else if (solver == RIEMANN_ACOUSTIC) S3B(RIEMANN_ACOUSTIC); else if (solver == RIEMANN_HLLC) S3B(RIEMANN_HLLC); else S3B(RIEMANN_HLL);
#undef S3B
#undef S3V
#undef S3
  return nblocks;
}

int devnum_sweep3(int solver, int N, int nblocks, const double* uin, double* uout, double dt, double dx, int slope_type,
                  double slope_theta, double courant_factor, double gamma, double smallr, double smallc, int niter, double* part, int by,
                  int vec) {
  const int n[3] = {N, N, N};
  return devnum_sweep3_box(solver, n, k_no_shell, nblocks, uin, uout, dt, dx, slope_type, slope_theta, courant_factor, gamma, smallr,
                           smallc, niter, part, by, vec);
}

void devnum_mhd_cmpdt(int n, const double* u, double dx, double* dt, double gamma, double smallr, double smallc, double cfl) {
  const MPhys M = make_mphys(gamma, smallr, smallc, kNotRead, cfl);
  for (int i = 0; i < n; i++) {
    real uu[11];
    for (int k = 0; k < 11; k++) uu[k] = u[i * 11 + k];
    dt[i] = (double)mhd_cmpdt_cell(M, uu, dx);
  }
}

}  // extern "C"
#pragma GCC visibility pop
