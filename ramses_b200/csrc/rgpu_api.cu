// rgpu_api.cu -- host side of the C-ABI declared in include/ramses_gpu.h.
//
// Mirrors the reference's per-level driver routines (hydro/godunov_fine.f90,
// hydro/courant_fine.f90, hydro/hydro_boundary.f90, amr/virtual_boundaries.f90)
// on device-resident "level stores": for every bound level the octs named by the
// communicator lists are renumbered into lattice order ("slots") and the state
// lives as u[ivar][cell-in-oct][slot] -- the oct-tree layout of the reference
// (hydro/hydro_commons.f90:4) with contiguous, spatially ordered octs.
#include <cuda_runtime.h>
#include <nccl.h>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <vector>
#include "../../include/ramses_gpu.h"
#include "sweep_dense.cuh"
#include "sweep_dense3.cuh"
#include "sweep_dense4.cuh"
#include "amr_kernels.cuh"
#include "mhd_amr.cuh"
#include "amr_schedules.h"
#include "mhd_dense.cuh"

namespace rgpu {
// launchers instantiated in sweep_inst_*.cu
template <int NDIM, int RIEMANN> cudaError_t launch_sweep_dense(const SweepArgs& a, int nblocks, cudaStream_t st, int by);
#define DECL(ND, R) extern template cudaError_t launch_sweep_dense<ND, R>(const SweepArgs&, int, cudaStream_t, int);
DECL(1, 0) DECL(1, 1) DECL(1, 2) DECL(1, 3) DECL(1, 4)
DECL(2, 0) DECL(2, 1) DECL(2, 2) DECL(2, 3) DECL(2, 4)
DECL(3, 0) DECL(3, 1) DECL(3, 2) DECL(3, 3) DECL(3, 4)
#undef DECL
// round-2 form of the 3-D sweep (sweep_dense3.cuh), instantiated in sweep3_inst_*.cu
#define DECL(R) extern template cudaError_t launch_sweep3<R>(const SweepArgs&, int, cudaStream_t, int); \
                extern template cudaError_t launch_sweep4<R>(const SweepArgs&, int, cudaStream_t, int);
DECL(0) DECL(1) DECL(2) DECL(3) DECL(4)
#undef DECL
template <int NDIM, int RIEMANN> cudaError_t launch_sweep_dense_amr(const SweepArgs& a, int nblocks, cudaStream_t st);
}  // namespace rgpu
// FAST arithmetic mode: the same kernels built with FMA contraction under namespace rgpu_fast (sweep3_fast_inst_*.cu)
extern "C" {
cudaError_t rgpu_fast_launch_sweep3_llf(const void*, int, cudaStream_t, int);
cudaError_t rgpu_fast_launch_sweep3_exact(const void*, int, cudaStream_t, int);
cudaError_t rgpu_fast_launch_sweep3_acoustic(const void*, int, cudaStream_t, int);
cudaError_t rgpu_fast_launch_sweep3_hllc(const void*, int, cudaStream_t, int);
cudaError_t rgpu_fast_launch_sweep3_hll(const void*, int, cudaStream_t, int);
}
namespace rgpu {
#define DECL(R) extern template cudaError_t launch_sweep_dense_amr<3, R>(const SweepArgs&, int, cudaStream_t);
DECL(0) DECL(1) DECL(2) DECL(3) DECL(4)
#undef DECL
// poisson: the GRAV instantiations of the dense sweep (sweep_grav_inst_*.cu)
#define DECL(ND, R, AMRV) extern template cudaError_t launch_sweep_dense_grav<ND, R, AMRV>(const SweepArgs&, int, cudaStream_t);
DECL(1, 0, false) DECL(1, 1, false) DECL(1, 2, false) DECL(1, 3, false) DECL(1, 4, false)
DECL(2, 0, false) DECL(2, 1, false) DECL(2, 2, false) DECL(2, 3, false) DECL(2, 4, false)
DECL(3, 0, false) DECL(3, 1, false) DECL(3, 2, false) DECL(3, 3, false) DECL(3, 4, false)
DECL(3, 0, true) DECL(3, 1, true) DECL(3, 2, true) DECL(3, 3, true) DECL(3, 4, true)
#undef DECL
// pressure_fix: the PFIX instantiations of the 3-D AMR variant, without and with poisson (sweep_pfix_inst_3d_*.cu)
#define DECL(R, GRAV) extern template cudaError_t launch_sweep_dense_pfix<R, GRAV>(const SweepArgs&, int, cudaStream_t);
DECL(0, false) DECL(1, false) DECL(2, false) DECL(3, false) DECL(4, false)
DECL(0, true) DECL(1, true) DECL(2, true) DECL(3, true) DECL(4, true)
#undef DECL
// pressure_fix outside AMR mode: the plain PFIX instantiations (sweep_pfix_inst_12d.cu, sweep_pfix_inst_plain3d_*.cu)
#define DECL(ND, R) extern template cudaError_t launch_sweep_dense_pfix_plain<ND, R>(const SweepArgs&, int, cudaStream_t);
DECL(1, 0) DECL(1, 1) DECL(1, 2) DECL(1, 3) DECL(1, 4)
DECL(2, 0) DECL(2, 1) DECL(2, 2) DECL(2, 3) DECL(2, 4)
DECL(3, 0) DECL(3, 1) DECL(3, 2) DECL(3, 3) DECL(3, 4)
#undef DECL
}  // namespace rgpu

using namespace rgpu;

namespace {

constexpr int MAXLEVEL = 32;
char g_err[512] = "";

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
#define CUDA_OK(x)                                                                                        \
  do {                                                                                                    \
    cudaError_t e_ = (x);                                                                                 \
    if (e_ != cudaSuccess) return fail(RGPU_ECUDA, "%s:%d %s: %s", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); \
  } while (0)
#define NCCL_OK(x)                                                                                        \
  do {                                                                                                    \
    ncclResult_t r_ = (x);                                                                                \
    if (r_ != ncclSuccess) return fail(RGPU_ENCCL, "%s:%d %s: %s", __FILE__, __LINE__, #x, ncclGetErrorString(r_)); \
  } while (0)

struct BoundRegion {
  int type = 0;          // boundary_type(ibound)
  int n = 0;             // octs
  int* d_slots = nullptr;
};

struct PeerList {        // one peer rank
  int nrecv = 0, nemit = 0;
  int* d_recv = nullptr; // slots of reception (ghost) octs, in the order of reception(icpu,ilevel)%igrid
  int* d_emit = nullptr; // slots of emission octs
  double* d_sbuf = nullptr;
  double* d_rbuf = nullptr;
};

struct Level {
  bool bound = false;
  bool dense = false;
  DenseGeom g{};
  int lo[3] = {0, 0, 0};             // box origin in oct units (global oct coordinates)
  int gmin = 0, gmax = 0;            // igrid range covered by the level (host mirror window)
  long long nslot = 0;
  std::vector<int> slot_igrid;       // igrid of every slot (0: empty)
  std::vector<std::vector<int>> h_bslots, h_rslots, h_eslots;   // boundary / reception / emission octs as slots
  std::vector<int> h_btype;
  int* d_slot_igrid = nullptr;
  double* d_mirror = nullptr;        // host-layout window [nvar][2^ndim][gmax-gmin+1]
  double* d_u[2] = {nullptr, nullptr};
  int cur = 0;                       // d_u[cur] = uold, d_u[1-cur] = unew
  bool unew_valid = false;
  std::vector<BoundRegion> regions;
  std::vector<PeerList> peers;
  int ntx = 0, nty = 0, nblocks = 0, by = 1;
  int variant = 0;                   // 3-D hydro: sweep3_kernel variant (100*BY + 10*MINB + VEC); 0: round-1 kernel
  // fused forward ghost exchange: every peer's emission / reception slots in one list, one send and one receive buffer with a
  // contiguous segment per peer ([plane][oct] inside a segment): one pack kernel, one NCCL group, one unpack kernel per exchange
  int *d_emit_all = nullptr, *d_recv_all = nullptr;
  long long *d_emit_off = nullptr, *d_recv_off = nullptr;   // [npeer+1] first oct of every peer's segment
  double *d_sbuf_all = nullptr, *d_rbuf_all = nullptr;
  std::vector<long long> emit_off, recv_off;
  // overlap of the exchange with the interior of the next sweep (rgpu_level_steps, multi-rank): interior / frame work maps
  bool overlap = false;
  int reserve_sms = 0;
  SweepWork wk_int{}, wk_frame{};
  long long nwork_int = 0, nwork_frame = 0;
  cudaEvent_t ev_x = nullptr, ev_s = nullptr;
  // Level-0 pipeline (rgpu_godunov_fine on host arrays): z-slabs of oct planes; per slab the igrid ranges to upload (every oct
  // of the slab) and to download (its active octs).  Empty when the oct numbering is too scattered (serial path then).
  struct Range { int lo, n, stride, count; };   // `count` runs of n consecutive igrids, `stride` igrids apart (count 1: one run)
  struct Slab { int oz_a = 0, oz_b = 0; std::vector<Range> up, down; };
  std::vector<Slab> slabs;
  std::vector<cudaEvent_t> ev_in, ev_c;
  long long nwork = 0;
  double* d_part = nullptr;          // [5][part_cap]
  double* d_mhdw = nullptr;          // MHD work arrays [MW_NCOMP][ncell_box]
  unsigned char* d_refined = nullptr;  // AMR mode: son(cell)>0 per box cell [2^ndim][nslot]
  double* d_f = nullptr;             // poisson: the acceleration f [ndim][2^ndim][nslot] (rgpu_upload_force; AMR mode: gathered per call)
  double* d_pfix = nullptr;          // pressure_fix: divu and enew [2][2^ndim][nslot] (AMR mode: gathered from / scattered to d_unew per call)
  bool pfix_ready = false;           // pressure_fix, levelmin=levelmax: set_unew has initialised divu / enew for the next sweep
  bool f_valid = false;              // poisson, levelmin=levelmax: f uploaded since the bind
  double dt_last = 0.0;              // dt of the last godunov_fine (rgpu_set_uold's gravity source term needs it)
  int mhd_nb = 0;                    // CTAs of the MHD update kernel
  int part_cap = 0;
  double* d_dt = nullptr;            // [1] dt used by the next sweep
  double* d_out = nullptr;           // [5] dt, mass, etot, eint (, emag) of the last scan
  double* d_hist = nullptr; int hist_cap = 0;
  long long launches = 0;
  double dt_by_value = 0.0, dt_stage = 0.0;   // rgpu_godunov_fine_dev: time step of the pending launch (hydro: passed by value)
  double last_sweep_ms = 0;
  double last_steps_ms = 0;
  double dx = 0;
};

// AMR mode (levelmin < levelmax): the device mirrors the reference arrays, every level is a list of octs
struct AmrRegion { int type = 0, n = 0; int* d_igrid = nullptr; };
struct AmrPeer { int nrecv = 0, nemit = 0; int *d_recv = nullptr, *d_emit = nullptr; double *d_sbuf = nullptr, *d_rbuf = nullptr; };
struct AmrLevel {
  bool bound = false;
  int nact = 0;
  int* d_active = nullptr;
  std::vector<AmrRegion> regions;
  std::vector<AmrPeer> peers;
  double* d_rflux = nullptr;
  int nent = 0;                       // coarse cells that receive refluxes from this level
  int *d_rcell = nullptr, *d_rstart = nullptr, *d_rsrc = nullptr;
  double* d_part = nullptr; double* d_out = nullptr; double* d_dt = nullptr;
  long long launches = 0;
  double dx = 0;
  double dt_last = 0;                 // dtnew(ilevel) of the last godunov_fine (set_uold's source terms need it)
  // MHD, NDIM = 2: corner EMFs of every oct and their coarse-reflux schedule (mhd/godunov_fine.f90:1176-1270)
  double* d_remf = nullptr;
  int nemf = 0;
  int *d_ecell = nullptr, *d_evar = nullptr, *d_estart = nullptr, *d_ecode = nullptr;
  double last_steps_ms = 0;           // CUDA-event duration of the last rgpu_amr_steps call (recorded on the levelmin entry)
  bool dense_sweep = false;           // the level is a Cartesian box: godunov_fine runs the dense kernel (AMR variant)
  bool patch = false;                 // ... with a prolongated ghost shell and coarse refluxes (refined patch)
  int nsurf = 0;                      // octs at the surface of the patch (they own the refluxed faces)
  int *d_surf_igrid = nullptr, *d_surf_io = nullptr, *d_act_slot = nullptr, *d_shell_father = nullptr;
  std::vector<int> h_surf_io;
};

struct Context {
  bool init = false;
  bool amr = false;
  int* d_son = nullptr; int* d_son_base = nullptr; int* d_father = nullptr; int* d_nbor = nullptr;
  double* d_uold = nullptr; double* d_unew = nullptr;
  double bvar[64][8] = {{0}};        // boundary_var(ibound, 1:nvar) of the imposed boundaries (rgpu_set_boundary_var)
  bool bvar_set[64] = {false};
  double* d_force = nullptr;         // poisson: f[ndim][ncell] (rgpu_upload_force)
  int nvn = 0;                       // columns of d_unew: nvar, + divu and enew with pressure_fix
  long long ncell = 0;
  int interpol_type = 1, interpol_var = 0;
  int interpol_mag_type = -1;        // -1: interpol_type (hydro/read_hydro_params.f90:531)
  // one coarse step of rgpu_amr_steps as a CUDA graph (single rank, mesh unchanged since the capture): ~200 short launches per
  // coarse step of a 4-level run replay without per-launch CPU work or inter-kernel launch gaps
  cudaGraphExec_t amr_graph = nullptr;
  int amr_graph_levelmin = 0; int amr_graph_nsub[MAXLEVEL + 2] = {0};
  long long amr_graph_launches[MAXLEVEL + 1] = {0};   // kernel launches per level inside one captured coarse step
  AmrLevel alev[MAXLEVEL + 1];
  double* d_dtn = nullptr; double* d_dto = nullptr;   // device-resident dtnew/dtold(0:MAXLEVEL+1) of rgpu_amr_steps
  int numbtot[MAXLEVEL + 2] = {0};                    // numbtot(1,ilevel): octs of a level over ALL ranks (amr_commons.f90)
  int* d_numb = nullptr;
  rgpu_params p{};
  Phys phys{};
  MPhys mphys{};
  int nvs = 0;                       // stored variables per cell: nvar (hydro) or nvar+3 (MHD)
  int myid = 1, ncpu = 1, device = 0;
  int nsm = 132;                     // SMs of the bound device (rgpu_init); 132 on an H100 SXM for host-only planning
  cudaStream_t stream = nullptr;
  cudaStream_t s_in = nullptr, s_out = nullptr;   // copy streams of the Level-0 pipeline (H2D / D2H run on both DMA engines)
  cudaStream_t s_x = nullptr;                     // ghost exchange stream (overlaps the interior sweep)
  ncclComm_t comm_x = nullptr;                    // communicator of the exchange stream (split of `comm`)
  cudaEvent_t ev_pipe = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev2 = nullptr, ev3 = nullptr;
  bool timing = false;
  bool pipeline = true;              // Level-0 call: slab pipeline allowed (rgpu_set_pipeline)
  int ncoarse = 0, ngridmax = 0;
  const int *son = nullptr, *father = nullptr, *nbor = nullptr;
  Level lev[MAXLEVEL + 1];
  ncclComm_t comm = nullptr;
  int nranks = 1, rank = 0;
} G;

// grid of the grid-stride scans (Courant partials, self-test): eight CTAs per SM
inline int reduce_blocks() { return G.nsm * 8; }

// ----------------------------------------------------------------------------- kernels
__global__ void gather_slots_kernel(const double* __restrict__ mirror, double* __restrict__ u, const int* __restrict__ slot_igrid,
                                    long long nslot, int gmin, long long gspan, int nplanes, long long s0 = 0, long long s1 = -1) {
  const long long s = s0 + blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (s >= (s1 < 0 ? nslot : s1)) return;
  const int ig = slot_igrid[s];
  if (ig <= 0) return;
  for (int pl = 0; pl < nplanes; pl++) u[(size_t)pl * nslot + s] = mirror[(size_t)pl * gspan + (ig - gmin)];
}
__global__ void scatter_slots_kernel(double* __restrict__ mirror, const double* __restrict__ u, const int* __restrict__ slot_igrid,
                                     long long nslot, int gmin, long long gspan, int nplanes, int owned_only, DenseGeom g,
                                     long long s0 = 0, long long s1 = -1) {
  const long long s = s0 + blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (s >= (s1 < 0 ? nslot : s1)) return;
  const int ig = slot_igrid[s];
  if (ig <= 0) return;
  if (owned_only) {   // only the active octs (owned cell range) are written back
    const int ox = (int)(s % g.nox), oy = (int)((s / g.nox) % g.noy), oz = (int)(s / ((long long)g.nox * g.noy));
    if (2 * ox < g.ox0 || 2 * ox >= g.ox1) return;
    if (g.ncy > 1 && (2 * oy < g.oy0 || 2 * oy >= g.oy1)) return;
    if (g.ncz > 1 && (2 * oz < g.oz0 || 2 * oz >= g.oz1)) return;
  }
  for (int pl = 0; pl < nplanes; pl++) mirror[(size_t)pl * gspan + (ig - gmin)] = u[(size_t)pl * nslot + s];
}

// set_unew on the owned cells: unew = uold (hydro/godunov_fine.f90:58-66); ghost octs: unew = 0 (:93-100)
__global__ void copy_state_kernel(const double* __restrict__ src, double* __restrict__ dst, size_t n) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[i];
}
__global__ void zero_octs_kernel(double* __restrict__ u, const int* __restrict__ slots, int n, long long nslot, int nplanes) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  for (int pl = 0; pl < nplanes; pl++) u[(size_t)pl * nslot + slots[i]] = 0.0;
}

// carry a list of octs from one state buffer to the other (ghost / boundary shells across the uold<->unew swap)
__global__ void copy_octs_kernel(const double* __restrict__ src, double* __restrict__ dst, const int* __restrict__ slots, int n,
                                 long long nslot, int nplanes) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)n * nplanes) return;
  const size_t a = (size_t)(i / n) * nslot + slots[i % n];
  dst[a] = src[a];
}

// AMR mode, dense levels: reference-layout arrays u[ivar][icell] <-> level store u[ivar][cell-in-oct][slot]
__global__ void amr_gather_slots_kernel(const double* __restrict__ src, double* __restrict__ u, const int* __restrict__ slot_igrid, long long nslot,
                                        int ncoarse, int ngridmax, long long ncell, int nvar, int T) {
  const long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (s >= nslot) return;
  const int ig = slot_igrid[s];
  if (ig <= 0) return;
  for (int iv = 0; iv < nvar; iv++)
    for (int ind = 0; ind < T; ind++)
      u[((size_t)iv * T + ind) * nslot + s] = src[(size_t)iv * ncell + ncoarse + (size_t)ind * ngridmax + ig - 1];
}
__global__ void amr_scatter_slots_kernel(double* __restrict__ dst, const double* __restrict__ u, const int* __restrict__ slot_igrid, long long nslot,
                                         int ncoarse, int ngridmax, long long ncell, int nvar, int T, DenseGeom g) {
  const long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (s >= nslot) return;
  const int ig = slot_igrid[s];
  if (ig <= 0) return;
  const int ox = (int)(s % g.nox), oy = (int)((s / g.nox) % g.noy), oz = (int)(s / ((long long)g.nox * g.noy));
  if (2 * ox < g.ox0 || 2 * ox >= g.ox1) return;      // active octs only
  if (g.ncy > 1 && (2 * oy < g.oy0 || 2 * oy >= g.oy1)) return;
  if (g.ncz > 1 && (2 * oz < g.oz0 || 2 * oz >= g.oz1)) return;
  for (int iv = 0; iv < nvar; iv++)
    for (int ind = 0; ind < T; ind++)
      dst[(size_t)iv * ncell + ncoarse + (size_t)ind * ngridmax + ig - 1] = u[((size_t)iv * T + ind) * nslot + s];
}
__global__ void amr_refined_mask_kernel(const int* __restrict__ son0 /*son(1:ncell), 0-based*/, unsigned char* __restrict__ mask,
                                        const int* __restrict__ slot_igrid, long long nslot, int ncoarse, int ngridmax, int T) {
  const long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (s >= nslot) return;
  const int ig = slot_igrid[s];
  for (int ind = 0; ind < T; ind++)
    mask[(size_t)ind * nslot + s] = (ig > 0 && son0[ncoarse + (size_t)ind * ngridmax + ig - 1] > 0) ? 1 : 0;
}

// make_boundary_hydro (hydro/hydro_boundary.f90:5-269) for one boundary region.
struct BoundArgs {
  int n; const int* slots; long long nslot; long long nbr_off; // slot offset of the reference oct (towards the domain)
  int ind_ref[8]; double gs[3]; int kind;  // 0 wall (reflexive), 1 free (outflow), 2 imposed (boundary_var, default boundana)
  int ndim, nvar; double smallr;
  double bvar[8];
};
__global__ void boundary_kernel(double* __restrict__ u, const BoundArgs b) {
  const int T = 1 << b.ndim;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= b.n * T) return;
  const int o = i / T, ind = i % T;
  const long long s = b.slots[o], sr = s + b.nbr_off;
  const int indr = b.ind_ref[ind] - 1;
  if (b.kind == 2) {   // :229-252 with the default boundana (hydro/boundana.f90): u = boundary_var(ibound, :)
    for (int iv = 0; iv < b.nvar; iv++) u[((size_t)iv * T + ind) * b.nslot + s] = b.bvar[iv];
    return;
  }
  double uu[8];
  for (int iv = 0; iv < b.nvar; iv++) uu[iv] = u[((size_t)iv * T + indr) * b.nslot + sr];
  if (b.kind == 0) {   // :141-157
    for (int iv = 0; iv < b.nvar; iv++) {
      double sw = 1.0;
      if (iv >= 1 && iv <= b.ndim) sw = b.gs[iv - 1];
      u[((size_t)iv * T + ind) * b.nslot + s] = uu[iv] * sw;
    }
  } else {             // :160-211 (no_inflow = .false.)
    double ekin = 0.0;
    double d = fmx(uu[0], b.smallr);
    for (int idim = 0; idim < b.ndim; idim++) { const double v = uu[idim + 1] / d; ekin = ekin + 0.5 * d * (v * v); }
    uu[b.ndim + 1] = uu[b.ndim + 1] - ekin;
    ekin = 0.0;
    d = fmx(uu[0], b.smallr);
    for (int idim = 0; idim < b.ndim; idim++) { const double v = uu[idim + 1] / d; ekin = ekin + 0.5 * d * (v * v); }
    uu[b.ndim + 1] = uu[b.ndim + 1] + ekin;
    for (int iv = 0; iv < b.nvar; iv++) u[((size_t)iv * T + ind) * b.nslot + s] = uu[iv];
  }
}

// stand-alone courant_fine scan over the owned cells (hydro/courant_fine.f90:1-159); GRAV (poisson): gg = f, the acceleration in
// the level-store layout (:75-83)
template <int NDIM, bool GRAV = false>
__global__ void courant_kernel(const double* __restrict__ u, DenseGeom g, Phys P, double dx, double* __restrict__ part,
                               const double* __restrict__ force = nullptr) {
  constexpr int NV = NDIM + 2, T = 1 << NDIM;
  __shared__ double red[4][32];
  const long long nx = g.ox1 - g.ox0, ny = NDIM > 1 ? g.oy1 - g.oy0 : 1, nz = NDIM > 2 ? g.oz1 - g.oz0 : 1;
  const long long ncell = nx * ny * nz;
  double my_dt = 1e300, m0 = 0, m1 = 0, m2 = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < ncell; i += (long long)gridDim.x * blockDim.x) {
    const int x = g.ox0 + (int)(i % nx), y = NDIM > 1 ? g.oy0 + (int)((i / nx) % ny) : 0, z = NDIM > 2 ? g.oz0 + (int)(i / (nx * ny)) : 0;
    const long long off = cell_offset<NDIM>(g, x, y, z);
    double uu[NV];
#pragma unroll
    for (int n = 0; n < NV; n++) uu[n] = u[(size_t)n * T * g.nslot + off];
    double ei;
    double gs = -1.0;
    if (GRAV) {   // the same sum as amr_courant_kernel (amr_kernels.cuh)
      gs = 0.0;
#pragma unroll
      for (int d = 0; d < NDIM; d++) gs = gs + fabs(force[(size_t)d * T * g.nslot + off]);
    }
    const double dtc = cmpdt_cell<NDIM>(uu, dx, P, ei, gs);
    my_dt = dtc < my_dt ? dtc : my_dt;
    m0 += uu[0]; m1 += uu[NDIM + 1];
    m2 += ei;
  }
  my_dt = warp_min(my_dt); m0 = warp_sum(m0); m1 = warp_sum(m1); m2 = warp_sum(m2);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { red[0][w] = my_dt; red[1][w] = m0; red[2][w] = m1; red[3][w] = m2; }
  __syncthreads();
  if (w == 0) {
    const int nw = blockDim.x >> 5;
    double v0 = l < nw ? red[0][l] : 1e300, v1 = l < nw ? red[1][l] : 0, v2 = l < nw ? red[2][l] : 0, v3 = l < nw ? red[3][l] : 0;
    v0 = warp_min(v0); v1 = warp_sum(v1); v2 = warp_sum(v2); v3 = warp_sum(v3);
    if (l == 0) {
      const size_t nb = gridDim.x;
      part[0 * nb + blockIdx.x] = v0; part[1 * nb + blockIdx.x] = v1; part[2 * nb + blockIdx.x] = v2; part[3 * nb + blockIdx.x] = v3;
    }
  }
}

// set_uold's add_gravity_source_terms (hydro/godunov_fine.f90:159-161,237-289) on the owned cells of a dense level store
template <int NDIM>
__global__ void dense_gravity_src_kernel(const double* __restrict__ uold, double* __restrict__ unew, const double* __restrict__ force,
                                         DenseGeom g, double smallr, double dt) {
  constexpr int T = 1 << NDIM;
  const long long nx = g.ox1 - g.ox0, ny = NDIM > 1 ? g.oy1 - g.oy0 : 1, nz = NDIM > 2 ? g.oz1 - g.oz0 : 1;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= nx * ny * nz) return;
  const int x = g.ox0 + (int)(i % nx), y = NDIM > 1 ? g.oy0 + (int)((i / nx) % ny) : 0, z = NDIM > 2 ? g.oz0 + (int)(i / (nx * ny)) : 0;
  const long long off = cell_offset<NDIM>(g, x, y, z);
  const size_t vs = (size_t)T * g.nslot;
  double un[NDIM + 2], f[NDIM];
#pragma unroll
  for (int n = 0; n < NDIM + 2; n++) un[n] = unew[n * vs + off];
#pragma unroll
  for (int d = 0; d < NDIM; d++) f[d] = force[d * vs + off];
  gravity_src_cell(un[0], un[1], un[1 + 1 % NDIM], un[1 + 2 % NDIM], un[NDIM + 1], fmx(uold[off], smallr), f[0], f[1 % NDIM], f[2 % NDIM],
                   NDIM, smallr, dt);
#pragma unroll
  for (int n = 1; n < NDIM + 2; n++) unew[n * vs + off] = un[n];
}

// AMR patch mode, poisson: the empty shell slots of a refined patch take the f of their father cell (straight injection,
// hydro/godunov_fine.f90:637-647); force = f[ndim][ncell] of the tree, f = level store [ndim][8][nslot]
__global__ void amr_fill_shell_force_kernel(const double* __restrict__ force, double* __restrict__ f, const int* __restrict__ shell_father,
                                            long long nslot, long long ncell, int ndim) {
  const long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (s >= nslot) return;
  const int fc = shell_father[s];
  if (fc <= 0) return;
  for (int d = 0; d < ndim; d++) {
    const double v = force[(size_t)d * ncell + fc - 1];
    for (int is = 0; is < 8; is++) f[((size_t)d * 8 + is) * nslot + s] = v;
  }
}

// final reduction of the per-CTA partials: dt = min(dt_cap, courant_factor*dx/smallc, min dtcell)
// (cmpdt godunov_utils.f90:113-118, courant_fine.f90:121-123,155); fixed summation order.
__global__ void courant_reduce_kernel(const double* __restrict__ part, int nb, double dt_cap, double dt_floor0, double vol,
                                      double* __restrict__ out /*[5]*/, double* __restrict__ dt_dev, double* __restrict__ hist, int has_emag = 0) {
  __shared__ double red[5][32];
  double v0 = 1e300, v1 = 0, v2 = 0, v3 = 0, v4 = 0;
  for (int i = threadIdx.x; i < nb; i += blockDim.x) {
    v0 = part[i] < v0 ? part[i] : v0; v1 += part[(size_t)nb + i]; v2 += part[2 * (size_t)nb + i]; v3 += part[3 * (size_t)nb + i];
    if (has_emag) v4 += part[4 * (size_t)nb + i];
  }
  v0 = warp_min(v0); v1 = warp_sum(v1); v2 = warp_sum(v2); v3 = warp_sum(v3); v4 = warp_sum(v4);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { red[0][w] = v0; red[1][w] = v1; red[2][w] = v2; red[3][w] = v3; red[4][w] = v4; }
  __syncthreads();
  if (w == 0) {
    const int nw = blockDim.x >> 5;
    v0 = l < nw ? red[0][l] : 1e300; v1 = l < nw ? red[1][l] : 0; v2 = l < nw ? red[2][l] : 0; v3 = l < nw ? red[3][l] : 0; v4 = l < nw ? red[4][l] : 0;
    v0 = warp_min(v0); v1 = warp_sum(v1); v2 = warp_sum(v2); v3 = warp_sum(v3); v4 = warp_sum(v4);
    if (l == 0) {
      double dt = dt_floor0 < v0 ? dt_floor0 : v0;
      dt = dt_cap < dt ? dt_cap : dt;
      out[0] = dt; out[1] = v1 * vol; out[2] = v2 * vol; out[3] = v3 * vol; out[4] = v4 * vol;
      if (dt_dev) *dt_dev = dt;
      if (hist) *hist = dt;
    }
  }
}

// pack / unpack of ghost-oct exchange buffers: all variables of one peer in one message
// (replaces the per-variable messages of make_virtual_fine_dp, amr/virtual_boundaries.f90:454-464,492-506)
__global__ void pack_kernel(const double* __restrict__ u, const int* __restrict__ slots, int n, long long nslot, int nplanes, double* __restrict__ buf) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)n * nplanes) return;
  const int o = (int)(i % n), pl = (int)(i / n);
  buf[i] = u[(size_t)pl * nslot + slots[o]];
}
__global__ void unpack_kernel(double* __restrict__ u, const int* __restrict__ slots, int n, long long nslot, int nplanes, const double* __restrict__ buf, int accumulate) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)n * nplanes) return;
  const int o = (int)(i % n), pl = (int)(i / n);
  const size_t a = (size_t)pl * nslot + slots[o];
  if (accumulate) u[a] = u[a] + buf[i]; else u[a] = buf[i];
}

// fused forward exchange: all peers in one launch.  off[p] = first oct of peer p's segment, buffer segment p = [plane][oct]
__device__ __forceinline__ int seg_of(const long long* __restrict__ off, int nseg, long long o) {
  int p = 0;
  while (p + 1 < nseg && o >= off[p + 1]) p++;
  return p;
}
__global__ void pack_all_kernel(const double* __restrict__ u, const int* __restrict__ slots, long long ntot, long long nslot, int nplanes,
                                double* __restrict__ buf, const long long* __restrict__ off, int nseg) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= ntot * nplanes) return;
  const long long o = i % ntot;
  const int pl = (int)(i / ntot);
  const int p = seg_of(off, nseg, o);
  const long long n = off[p + 1] - off[p];
  buf[off[p] * nplanes + (long long)pl * n + (o - off[p])] = u[(size_t)pl * nslot + slots[o]];
}
__global__ void unpack_all_kernel(double* __restrict__ u, const int* __restrict__ slots, long long ntot, long long nslot, int nplanes,
                                  const double* __restrict__ buf, const long long* __restrict__ off, int nseg) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= ntot * nplanes) return;
  const long long o = i % ntot;
  const int pl = (int)(i / ntot);
  const int p = seg_of(off, nseg, o);
  const long long n = off[p + 1] - off[p];
  u[(size_t)pl * nslot + slots[o]] = buf[off[p] * nplanes + (long long)pl * n + (o - off[p])];
}

// self test of div_rn(a, b, rcp_rn(b)) == a / b (IEEE) on pseudo-random and adversarial operand pairs
__device__ __forceinline__ unsigned long long xs64(unsigned long long& s) { s ^= s << 13; s ^= s >> 7; s ^= s << 17; return s; }
__global__ void selftest_div_kernel(long long n_per_thread, unsigned long long seed, unsigned long long* mismatches) {
  unsigned long long s = seed + 0x9E3779B97F4A7C15ull * (blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x + 1);
  unsigned long long bad = 0;
  for (long long i = 0; i < n_per_thread; i++) {
    const unsigned long long ra = xs64(s), rb = xs64(s), rc = xs64(s);
    // significands: uniform, or adversarial (near 1, near 2, long runs of ones / zeros)
    unsigned long long ma = ra & 0xFFFFFFFFFFFFFull, mb = rb & 0xFFFFFFFFFFFFFull;
    const int mode = (int)(rc & 7);
    if (mode == 1) { ma &= 0xFFull; mb |= 0xFFFFFFFFFFF00ull; }
    else if (mode == 2) { ma |= 0xFFFFFFFFFFF00ull; mb &= 0xFFull; }
    else if (mode == 3) { ma = (ma & 0x3ull) | (0xFFFFFFFFFFFFFull << (rc >> 8 & 31) & 0xFFFFFFFFFFFFFull); mb &= ~0ull << (rc >> 16 & 31); }
    else if (mode == 4) { mb = 0xFFFFFFFFFFFFFull - (rb & 0xFull); }
    const int ea = 1023 + (int)((rc >> 24) % 201) - 100, eb = 1023 + (int)((rc >> 40) % 201) - 100;
    const double a = __longlong_as_double((long long)(((unsigned long long)ea << 52) | ma | ((rc >> 60 & 1ull) << 63)));
    const double b = __longlong_as_double((long long)(((unsigned long long)eb << 52) | mb | ((rc >> 61 & 1ull) << 63)));
    const double q1 = div_rn(a, b, rcp_rn(b));
    const double q2 = a / b;
    if (__double_as_longlong(q1) != __double_as_longlong(q2)) bad++;
    if (__double_as_longlong(rcp_rn(b)) != __double_as_longlong(1.0 / b)) bad++;
    const double aa = fabs(a);
    if (__double_as_longlong(sqrt_rn(aa)) != __double_as_longlong(sqrt(aa))) bad++;
  }
  if (bad) atomicAdd(mismatches, bad);
}

// ----------------------------------------------------------------------------- helpers
inline int T_() { return 1 << G.p.ndim; }
inline size_t nplanes_() { return (size_t)G.nvs * T_(); }

double level_dx(int ilevel) {  // godunov_fine.f90:532-534
  const int nx_loc = G.p.icoarse_max - G.p.icoarse_min + 1;
  const double scale = G.p.boxlen / (double)nx_loc;
  return std::pow(0.5, ilevel) * scale;
}

// integer position of an oct (units of its own size): walk the father chain (amr_commons: father(igrid)
// = father cell; cell index = ncoarse + (ind-1)*ngridmax + igrid)
void oct_pos(int ilevel, int igrid, int pos[3]) {
  int chain[MAXLEVEL];
  int g = igrid;
  int n = 0;
  for (int l = ilevel; l > 1; l--) {
    const int ic = G.father[g - 1];
    const int ind = (ic - G.ncoarse - 1) / G.ngridmax;
    g = ic - G.ncoarse - ind * G.ngridmax;
    chain[n++] = ind;
  }
  const int ic = G.father[g - 1];
  const int nxny = G.p.nx * G.p.ny;
  int pz = (ic - 1) / nxny, py = (ic - 1 - pz * nxny) / G.p.nx, px = ic - 1 - py * G.p.nx - pz * nxny;
  for (int i = n - 1; i >= 0; i--) {
    px = 2 * px + (chain[i] & 1);
    py = 2 * py + ((chain[i] >> 1) & 1);
    pz = 2 * pz + ((chain[i] >> 2) & 1);
  }
  pos[0] = px; pos[1] = py; pos[2] = pz;
}

void free_level(Level& L) {
  cudaFree(L.d_emit_all); cudaFree(L.d_recv_all); cudaFree(L.d_emit_off); cudaFree(L.d_recv_off); cudaFree(L.d_sbuf_all); cudaFree(L.d_rbuf_all);
  if (L.ev_x) cudaEventDestroy(L.ev_x);
  if (L.ev_s) cudaEventDestroy(L.ev_s);
  for (auto e : L.ev_in) cudaEventDestroy(e);
  for (auto e : L.ev_c) cudaEventDestroy(e);
  cudaFree(L.d_slot_igrid); cudaFree(L.d_mirror); cudaFree(L.d_u[0]); cudaFree(L.d_u[1]);
  cudaFree(L.d_part); cudaFree(L.d_dt); cudaFree(L.d_out); cudaFree(L.d_hist); cudaFree(L.d_mhdw); cudaFree(L.d_refined);
  cudaFree(L.d_f); cudaFree(L.d_pfix);
  for (auto& r : L.regions) cudaFree(r.d_slots);
  for (auto& p : L.peers) { cudaFree(p.d_recv); cudaFree(p.d_emit); cudaFree(p.d_sbuf); cudaFree(p.d_rbuf); }
  L = Level();
}

int check_level(int ilevel, Level** out) {
  if (!G.init) return fail(RGPU_EINVAL, "rgpu_init has not been called");
  if (ilevel < 1 || ilevel > MAXLEVEL) return fail(RGPU_EINVAL, "ilevel %d out of range", ilevel);
  Level& L = G.lev[ilevel];
  if (!L.bound) return fail(RGPU_EINVAL, "level %d is not bound (rgpu_bind_level)", ilevel);
  if (!L.dense) return fail(RGPU_EUNSUPPORTED, "level %d is not a dense box; the AMR oct-batch path is not built yet", ilevel);
  *out = &L;
  return RGPU_OK;
}

template <int ND>
cudaError_t dispatch_sweep_nd(int riemann, const SweepArgs& a, int nb, cudaStream_t st, int by) {
  switch (riemann) {
    case RGPU_RIEMANN_LLF: return launch_sweep_dense<ND, RIEMANN_LLF>(a, nb, st, by);
    case RGPU_RIEMANN_EXACT: return launch_sweep_dense<ND, RIEMANN_EXACT>(a, nb, st, by);
    case RGPU_RIEMANN_ACOUSTIC: return launch_sweep_dense<ND, RIEMANN_ACOUSTIC>(a, nb, st, by);
    case RGPU_RIEMANN_HLLC: return launch_sweep_dense<ND, RIEMANN_HLLC>(a, nb, st, by);
    default: return launch_sweep_dense<ND, RIEMANN_HLL>(a, nb, st, by);
  }
}
// poisson: the GRAV instantiations (runtime slope switch, default tile height); AMRV: the 3-D AMR variant
template <int ND, bool AMRV>
cudaError_t dispatch_sweep_grav(int riemann, const SweepArgs& a, int nb, cudaStream_t st) {
  switch (riemann) {
    case RGPU_RIEMANN_LLF: return launch_sweep_dense_grav<ND, RIEMANN_LLF, AMRV>(a, nb, st);
    case RGPU_RIEMANN_EXACT: return launch_sweep_dense_grav<ND, RIEMANN_EXACT, AMRV>(a, nb, st);
    case RGPU_RIEMANN_ACOUSTIC: return launch_sweep_dense_grav<ND, RIEMANN_ACOUSTIC, AMRV>(a, nb, st);
    case RGPU_RIEMANN_HLLC: return launch_sweep_dense_grav<ND, RIEMANN_HLLC, AMRV>(a, nb, st);
    default: return launch_sweep_dense_grav<ND, RIEMANN_HLL, AMRV>(a, nb, st);
  }
}
// pressure_fix: the PFIX instantiations of the 3-D AMR variant; GRAV: with poisson
template <bool GRAV>
cudaError_t dispatch_sweep_pfix(int riemann, const SweepArgs& a, int nb, cudaStream_t st) {
  switch (riemann) {
    case RGPU_RIEMANN_LLF: return launch_sweep_dense_pfix<RIEMANN_LLF, GRAV>(a, nb, st);
    case RGPU_RIEMANN_EXACT: return launch_sweep_dense_pfix<RIEMANN_EXACT, GRAV>(a, nb, st);
    case RGPU_RIEMANN_ACOUSTIC: return launch_sweep_dense_pfix<RIEMANN_ACOUSTIC, GRAV>(a, nb, st);
    case RGPU_RIEMANN_HLLC: return launch_sweep_dense_pfix<RIEMANN_HLLC, GRAV>(a, nb, st);
    default: return launch_sweep_dense_pfix<RIEMANN_HLL, GRAV>(a, nb, st);
  }
}
// pressure_fix outside AMR mode: the plain PFIX instantiations (runtime slope switch, default tile height)
template <int ND>
cudaError_t dispatch_sweep_pfix_plain(int riemann, const SweepArgs& a, int nb, cudaStream_t st) {
  switch (riemann) {
    case RGPU_RIEMANN_LLF: return launch_sweep_dense_pfix_plain<ND, RIEMANN_LLF>(a, nb, st);
    case RGPU_RIEMANN_EXACT: return launch_sweep_dense_pfix_plain<ND, RIEMANN_EXACT>(a, nb, st);
    case RGPU_RIEMANN_ACOUSTIC: return launch_sweep_dense_pfix_plain<ND, RIEMANN_ACOUSTIC>(a, nb, st);
    case RGPU_RIEMANN_HLLC: return launch_sweep_dense_pfix_plain<ND, RIEMANN_HLLC>(a, nb, st);
    default: return launch_sweep_dense_pfix_plain<ND, RIEMANN_HLL>(a, nb, st);
  }
}
inline int need_force(const Level& L) {
  if (G.p.poisson && !L.f_valid) return fail(RGPU_EINVAL, "poisson: no rgpu_upload_force since the level was bound (the sweep and the Courant "
                                                         "scan need the acceleration f)");
  return RGPU_OK;
}

// zlo/zhi >= 0: sweep only the owned cell planes [zlo, zhi) (Level-0 pipeline; no Courant partials then)
// part: 0 whole level, 1 interior, 2 frame (Level::wk_int / wk_frame; Courant partials of 1 and 2 share one array)
// gsrc (poisson): set_uold's gravity source term and the gravity term of the Courant scan are fused into the sweep
int launch_sweep(Level& L, int zlo = -1, int zhi = -1, int part = 0, bool gsrc = false) {
  if (G.p.mhd) {
    MhdArgs m{};
    m.uin = L.d_u[L.cur]; m.uout = L.d_u[1 - L.cur]; m.g = L.g; m.P = G.mphys; m.dt_dev = L.d_dt; m.dx = L.dx;
    m.W = L.d_mhdw; m.nc = (long long)L.g.ncx * L.g.ncy * L.g.ncz; m.part = L.d_part;
    if (G.timing) cudaEventRecord(G.ev0, G.stream);
    const bool sl = !(G.mphys.slope_type == 0 && G.mphys.slope_mag_type == 0);
    cudaError_t e = launch_mhd_sweep(m, G.p.riemann, G.p.riemann2d, sl, L.mhd_nb, G.stream);
    if (e != cudaSuccess) return fail(RGPU_ECUDA, "MHD sweep launch: %s", cudaGetErrorString(e));
    if (G.timing) {
      cudaEventRecord(G.ev1, G.stream);
      cudaEventSynchronize(G.ev1);
      float ms = 0;
      cudaEventElapsedTime(&ms, G.ev0, G.ev1);
      L.last_sweep_ms = ms;
    }
    L.launches += 6;
    return RGPU_OK;
  }
  { const int rc = need_force(L); if (rc) return rc; }
  SweepArgs a{};
  a.uin = L.d_u[L.cur];
  a.uout = L.d_u[1 - L.cur];
  a.g = L.g;
  a.P = G.phys;
  if (G.p.poisson) { a.force = L.d_f; a.gsrc = gsrc ? 1 : 0; }
  a.dt_dev = L.d_dt;
  if (L.dt_by_value > 0.0) { a.dt_dev = nullptr; a.dt_val = L.dt_by_value; }
  a.dx = L.dx;
  a.inv_dx = 1.0 / L.dx;   // correctly rounded reciprocal (IEEE division on the host)
  int ex;
  a.dx_pow2 = (std::frexp(L.dx, &ex) == 0.5) ? 1 : 0;
  a.ntx = L.ntx; a.nty = L.nty; a.nwork = L.nwork;
  a.part = L.d_part;
  int nblocks = L.nblocks;
  if (part) {
    a.wk = part == 1 ? L.wk_int : L.wk_frame;
    a.nwork = part == 1 ? L.nwork_int : L.nwork_frame;
    nblocks = (int)std::min<long long>(L.nblocks, a.nwork);
    // the interior launch leaves a few SMs to the pack / NCCL / unpack kernels of the exchange stream: a persistent CTA per SM
    // holds the whole register file, nothing else could become resident before the interior ends (RGPU_OVERLAP_RESERVE)
    if (part == 1 && nblocks > 4 * L.reserve_sms) nblocks -= L.reserve_sms;
    a.part_stride = 2 * L.nblocks; a.part_off = part == 1 ? 0 : L.nblocks;
  }
  if (zlo >= 0) {
    a.g.oz0 = std::max(L.g.oz0, zlo); a.g.oz1 = std::min(L.g.oz1, zhi);
    if (a.g.oz1 <= a.g.oz0) return RGPU_OK;
    a.nwork = (long long)L.ntx * L.nty * (a.g.oz1 - a.g.oz0);
    nblocks = (int)std::min<long long>(L.nblocks, a.nwork);
    a.part = nullptr;
  }
  if (G.p.pressure_fix) {   // divu / enew accumulate into the PFIX store; the Courant scan runs after set_uold's energy switch
    a.pfix = L.d_pfix;
    a.part = nullptr;
  }
  if (G.timing) cudaEventRecord(G.ev0, G.stream);
  cudaError_t e;
  if (G.p.pressure_fix) {   // round-1 kernel with pressure_fix (3-D: variant 0, FAST ignored; rgpu_bind_level)
    if (G.p.ndim == 1) e = dispatch_sweep_pfix_plain<1>(G.p.riemann, a, nblocks, G.stream);
    else if (G.p.ndim == 2) e = dispatch_sweep_pfix_plain<2>(G.p.riemann, a, nblocks, G.stream);
    else e = dispatch_sweep_pfix_plain<3>(G.p.riemann, a, nblocks, G.stream);
  }
  else if (G.p.poisson) {   // round-1 kernel with gravity (3-D: variant 0, FAST ignored; rgpu_bind_level)
    if (G.p.ndim == 1) e = dispatch_sweep_grav<1, false>(G.p.riemann, a, nblocks, G.stream);
    else if (G.p.ndim == 2) e = dispatch_sweep_grav<2, false>(G.p.riemann, a, nblocks, G.stream);
    else e = dispatch_sweep_grav<3, false>(G.p.riemann, a, nblocks, G.stream);
  }
  else if (G.p.ndim == 1) e = dispatch_sweep_nd<1>(G.p.riemann, a, nblocks, G.stream, L.by);
  else if (G.p.ndim == 2) e = dispatch_sweep_nd<2>(G.p.riemann, a, nblocks, G.stream, L.by);
  else if (L.variant && G.p.fast) {
    switch (G.p.riemann) {
      case RGPU_RIEMANN_LLF: e = rgpu_fast_launch_sweep3_llf(&a, nblocks, G.stream, L.variant); break;
      case RGPU_RIEMANN_EXACT: e = rgpu_fast_launch_sweep3_exact(&a, nblocks, G.stream, L.variant); break;
      case RGPU_RIEMANN_ACOUSTIC: e = rgpu_fast_launch_sweep3_acoustic(&a, nblocks, G.stream, L.variant); break;
      case RGPU_RIEMANN_HLLC: e = rgpu_fast_launch_sweep3_hllc(&a, nblocks, G.stream, L.variant); break;
      default: e = rgpu_fast_launch_sweep3_hll(&a, nblocks, G.stream, L.variant); break;
    }
  }
  else if (L.variant >= 40000) {   // one-barrier loop (sweep_dense4.cuh): tuning builds
    switch (G.p.riemann) {
      case RGPU_RIEMANN_LLF: e = launch_sweep4<RIEMANN_LLF>(a, nblocks, G.stream, L.variant); break;
      case RGPU_RIEMANN_EXACT: e = launch_sweep4<RIEMANN_EXACT>(a, nblocks, G.stream, L.variant); break;
      case RGPU_RIEMANN_ACOUSTIC: e = launch_sweep4<RIEMANN_ACOUSTIC>(a, nblocks, G.stream, L.variant); break;
      case RGPU_RIEMANN_HLLC: e = launch_sweep4<RIEMANN_HLLC>(a, nblocks, G.stream, L.variant); break;
      default: e = launch_sweep4<RIEMANN_HLL>(a, nblocks, G.stream, L.variant); break;
    }
  }
  else if (L.variant) {
    switch (G.p.riemann) {
      case RGPU_RIEMANN_LLF: e = launch_sweep3<RIEMANN_LLF>(a, nblocks, G.stream, L.variant); break;
      case RGPU_RIEMANN_EXACT: e = launch_sweep3<RIEMANN_EXACT>(a, nblocks, G.stream, L.variant); break;
      case RGPU_RIEMANN_ACOUSTIC: e = launch_sweep3<RIEMANN_ACOUSTIC>(a, nblocks, G.stream, L.variant); break;
      case RGPU_RIEMANN_HLLC: e = launch_sweep3<RIEMANN_HLLC>(a, nblocks, G.stream, L.variant); break;
      default: e = launch_sweep3<RIEMANN_HLL>(a, nblocks, G.stream, L.variant); break;
    }
  }
  else e = dispatch_sweep_nd<3>(G.p.riemann, a, nblocks, G.stream, L.by);
  if (e != cudaSuccess) return fail(RGPU_ECUDA, "sweep launch: %s", cudaGetErrorString(e));
  if (G.timing) {
    cudaEventRecord(G.ev1, G.stream);
    cudaEventSynchronize(G.ev1);
    float ms = 0;
    cudaEventElapsedTime(&ms, G.ev0, G.ev1);
    L.last_sweep_ms = ms;
  }
  L.launches++;
  return RGPU_OK;
}

// reduce partials of the last sweep / courant scan into d_out and d_dt
int launch_reduce(Level& L, int nb, double dt_cap, double* hist_slot) {
  const double vol = std::pow(L.dx, G.p.ndim);
  const double dt0 = G.p.courant_factor * L.dx / G.p.smallc;   // cmpdt: dt = courant_factor*dx/smallc
  courant_reduce_kernel<<<1, 1024, 0, G.stream>>>(L.d_part, nb, dt_cap, dt0, vol, L.d_out, L.d_dt, hist_slot, G.p.mhd ? 1 : 0);
  CUDA_OK(cudaGetLastError());
  L.launches++;
  return RGPU_OK;
}

int launch_courant(Level& L, double dt_cap, double* hist_slot) {
  const int nb = std::min(L.part_cap, reduce_blocks());
  if (G.p.mhd) {
    cudaError_t e = launch_mhd_courant(L.d_u[L.cur], L.g, G.mphys, L.dx, L.d_part, nb, G.stream);
    if (e != cudaSuccess) return fail(RGPU_ECUDA, "MHD courant launch: %s", cudaGetErrorString(e));
    L.launches++;
    return launch_reduce(L, nb, dt_cap, hist_slot);
  }
  if (G.p.poisson) {   // gg = f (courant_fine.f90:75-83)
    const int rc = need_force(L); if (rc) return rc;
    if (G.p.ndim == 1) courant_kernel<1, true><<<nb, 256, 0, G.stream>>>(L.d_u[L.cur], L.g, G.phys, L.dx, L.d_part, L.d_f);
    else if (G.p.ndim == 2) courant_kernel<2, true><<<nb, 256, 0, G.stream>>>(L.d_u[L.cur], L.g, G.phys, L.dx, L.d_part, L.d_f);
    else courant_kernel<3, true><<<nb, 256, 0, G.stream>>>(L.d_u[L.cur], L.g, G.phys, L.dx, L.d_part, L.d_f);
  }
  else if (G.p.ndim == 1) courant_kernel<1><<<nb, 256, 0, G.stream>>>(L.d_u[L.cur], L.g, G.phys, L.dx, L.d_part);
  else if (G.p.ndim == 2) courant_kernel<2><<<nb, 256, 0, G.stream>>>(L.d_u[L.cur], L.g, G.phys, L.dx, L.d_part);
  else courant_kernel<3><<<nb, 256, 0, G.stream>>>(L.d_u[L.cur], L.g, G.phys, L.dx, L.d_part);
  CUDA_OK(cudaGetLastError());
  L.launches++;
  return launch_reduce(L, nb, dt_cap, hist_slot);
}

// pressure_fix passes on the owned cells of a dense level (sweep_dense.cuh).  dt_dev != NULL: the time step of rgpu_level_steps
// (device resident), otherwise dt.  PFIX_INIT: set_unew's divu = 0, enew = e_int of uold; PFIX_PDV: add_pdv_source_terms from
// uold, whose ghost and boundary shells must be current; PFIX_SWITCH: set_uold's energy switch on the new state (after the swap)
enum PfixPass { PFIX_INIT, PFIX_PDV, PFIX_SWITCH };
int launch_pfix_pass(Level& L, PfixPass k, double dt, const double* dt_dev) {
  long long n = L.g.ox1 - L.g.ox0;
  if (G.p.ndim > 1) n *= L.g.oy1 - L.g.oy0;
  if (G.p.ndim > 2) n *= L.g.oz1 - L.g.oz0;
  const unsigned nb = (unsigned)((n + 127) / 128);
  const double* uo = L.d_u[L.cur];
#define PFIX_LAUNCH(ND)                                                                                                          \
  do {                                                                                                                           \
    if (k == PFIX_INIT) dense_pfix_init_kernel<ND><<<nb, 128, 0, G.stream>>>(uo, L.d_pfix, L.g, G.p.smallr);                    \
    else if (k == PFIX_PDV) dense_pdv_kernel<ND><<<nb, 128, 0, G.stream>>>(uo, L.d_pfix, L.g, G.p.gamma, G.p.smallr, L.dx, dt, dt_dev); \
    else dense_pfix_switch_kernel<ND><<<nb, 128, 0, G.stream>>>(L.d_u[L.cur], L.d_pfix, L.g, G.p.smallr, G.p.beta_fix, L.dx, dt, dt_dev); \
  } while (0)
  if (G.p.ndim == 1) PFIX_LAUNCH(1);
  else if (G.p.ndim == 2) PFIX_LAUNCH(2);
  else PFIX_LAUNCH(3);
#undef PFIX_LAUNCH
  CUDA_OK(cudaGetLastError());
  L.launches++;
  return RGPU_OK;
}

int launch_boundaries(Level& L, double* u) {
  // boundaries are applied in the order ibound = 1..nboundary like the reference loop
  // (hydro_boundary.f90:53): corner octs read neighbours that a later region refreshes.
  static const int ref_x[8] = {2, 1, 4, 3, 6, 5, 8, 7}, ref_y[8] = {3, 4, 1, 2, 7, 8, 5, 6}, ref_z[8] = {5, 6, 7, 8, 1, 2, 3, 4};
  static const int fre[6][8] = {{1, 1, 3, 3, 5, 5, 7, 7}, {2, 2, 4, 4, 6, 6, 8, 8}, {1, 2, 1, 2, 5, 6, 5, 6},
                                {3, 4, 3, 4, 7, 8, 7, 8}, {1, 2, 3, 4, 1, 2, 3, 4}, {5, 6, 7, 8, 5, 6, 7, 8}};
  int ibr = -1;
  for (auto& r : L.regions) {
    ibr++;
    if (r.n == 0) continue;
    const int bt = r.type, dir = bt - 10 * (bt / 10);
    if (bt / 10 > 2 || (bt / 10 == 2 && G.p.mhd)) return fail(RGPU_EUNSUPPORTED, "boundary type %d not supported", bt);
    if (bt / 10 == 2 && !G.bvar_set[ibr]) return fail(RGPU_EINVAL, "imposed boundary %d: call rgpu_set_boundary_var first", ibr + 1);
    const long long str[3] = {1, L.g.nox, (long long)L.g.nox * L.g.noy};
    const int d = (dir - 1) / 2;
    if (G.p.mhd) {   // mhd/hydro_boundary.f90:53-139
      static const int alt_[6][8] = {{-2, -1, -2, -1, -2, -1, -2, -1}, {1, 2, 1, 2, 1, 2, 1, 2}, {-2, -2, -1, -1, -2, -2, -1, -1},
                                     {1, 1, 2, 2, 1, 1, 2, 2}, {-2, -2, -2, -2, -1, -1, -1, -1}, {1, 1, 1, 1, 2, 2, 2, 2}};
      MhdBoundArgs m{};
      m.n = r.n; m.slots = r.d_slots; m.nslot = L.nslot;
      m.nbr_off = (dir % 2 == 1) ? str[d] : -str[d];
      const int* ir = (bt / 10 == 0) ? (d == 0 ? ref_x : d == 1 ? ref_y : ref_z) : fre[dir - 1];
      for (int i = 0; i < 8; i++) { m.ind_ref[i] = ir[i]; m.ind_normal[i] = fre[dir - 1][i]; m.alt[i] = alt_[dir - 1][i]; }
      m.gs[0] = m.gs[1] = m.gs[2] = 1.0;
      if (bt >= 1 && bt <= 6) m.gs[d] = -1.0;
      m.kind = bt / 10; m.gdim = d + 1;
      m.iperp1 = (dir % 2 == 1) ? 4 + m.gdim : 7 + m.gdim;   // left-face (6..8) / right-face (nvar+1..) component, 0-based
      m.smallr = G.p.smallr;
      cudaError_t e = launch_mhd_boundary(u, m, G.stream);
      if (e != cudaSuccess) return fail(RGPU_ECUDA, "MHD boundary launch: %s", cudaGetErrorString(e));
      L.launches++;
      continue;
    }
    BoundArgs b{};
    b.n = r.n; b.slots = r.d_slots; b.nslot = L.nslot;
    b.nbr_off = (dir % 2 == 1) ? str[d] : -str[d];   // boundary at the min face looks towards +d
    const int* ir = (bt / 10 == 0) ? (d == 0 ? ref_x : d == 1 ? ref_y : ref_z) : fre[dir - 1];
    for (int i = 0; i < 8; i++) b.ind_ref[i] = ir[i];
    b.gs[0] = b.gs[1] = b.gs[2] = 1.0;
    if (bt >= 1 && bt <= 6) b.gs[d] = -1.0;
    b.kind = bt / 10;
    b.ndim = G.p.ndim; b.nvar = G.p.nvar; b.smallr = G.p.smallr;
    for (int iv = 0; iv < 8; iv++) b.bvar[iv] = G.bvar[ibr][iv];
    const int nthr = r.n * T_();
    boundary_kernel<<<(nthr + 127) / 128, 128, 0, G.stream>>>(u, b);
    CUDA_OK(cudaGetLastError());
    L.launches++;
  }
  return RGPU_OK;
}


// ----------------------------------------------------------------------------- AMR mode host glue
AmrTree amr_tree() {
  AmrTree t{};
  t.son = G.d_son - 1;         // 1-based indexing like the Fortran arrays
  t.father = G.d_father - 1;
  t.nbor = G.d_nbor;
  t.ncoarse = G.ncoarse; t.ngridmax = G.ngridmax; t.nx = G.p.nx; t.ny = G.p.ny; t.nz = G.p.nz;
  t.ncell = G.ncell;
  return t;
}
inline bool src_terms() { return G.p.poisson || G.p.pressure_fix; }
inline void drop_amr_graph() { if (G.amr_graph) { cudaGraphExecDestroy(G.amr_graph); G.amr_graph = nullptr; } }
inline double* d_divu() { return G.d_unew + (size_t)G.p.nvar * G.ncell; }
inline double* d_enew() { return G.d_unew + (size_t)(G.p.nvar + 1) * G.ncell; }
void free_amr_level(AmrLevel& A) {
  cudaFree(A.d_active); cudaFree(A.d_rflux); cudaFree(A.d_rcell); cudaFree(A.d_rstart); cudaFree(A.d_rsrc);
  cudaFree(A.d_part); cudaFree(A.d_out); cudaFree(A.d_dt);
  cudaFree(A.d_surf_igrid); cudaFree(A.d_surf_io); cudaFree(A.d_act_slot); cudaFree(A.d_shell_father);
  cudaFree(A.d_remf); cudaFree(A.d_ecell); cudaFree(A.d_evar); cudaFree(A.d_estart); cudaFree(A.d_ecode);
  for (auto& r : A.regions) cudaFree(r.d_igrid);
  for (auto& p : A.peers) { cudaFree(p.d_recv); cudaFree(p.d_emit); cudaFree(p.d_sbuf); cudaFree(p.d_rbuf); }
  A = AmrLevel();
}
int check_amr_level(int ilevel, AmrLevel** out) {
  if (!G.init) return fail(RGPU_EINVAL, "rgpu_init has not been called");
  if (ilevel < 1 || ilevel > MAXLEVEL) return fail(RGPU_EINVAL, "ilevel %d out of range", ilevel);
  if (!G.d_son) return fail(RGPU_EINVAL, "AMR mode: rgpu_bind_tree has not been called");
  AmrLevel& A = G.alev[ilevel];
  if (!A.bound) return fail(RGPU_EINVAL, "level %d is not bound (rgpu_bind_level)", ilevel);
  *out = &A;
  return RGPU_OK;
}
int amr_bind_level(int ilevel, int ngrid_active, const int* igrid_active, int ncpu, const int* ngrid_recv, const int* const* igrid_recv,
                   const int* ngrid_emit, const int* const* igrid_emit, int nboundary, const int* boundary_type,
                   const int* ngrid_bound, const int* const* igrid_bound) {
  AmrLevel& A = G.alev[ilevel];
  drop_amr_graph();
  if (A.bound) free_amr_level(A);
  if (ncpu > 1 && ngrid_recv && igrid_recv && ngrid_emit && igrid_emit) {
    const size_t per = (size_t)G.nvn * T_();     // the reverse exchange of unew carries divu and enew too
    A.peers.resize(ncpu);
    for (int cpu = 0; cpu < ncpu; cpu++) {
      if (cpu == G.myid - 1) continue;
      AmrPeer& P = A.peers[cpu];
      P.nrecv = ngrid_recv[cpu]; P.nemit = ngrid_emit[cpu];
      if (P.nrecv) {
        CUDA_OK(cudaMalloc(&P.d_recv, sizeof(int) * P.nrecv));
        CUDA_OK(cudaMemcpy(P.d_recv, igrid_recv[cpu], sizeof(int) * P.nrecv, cudaMemcpyHostToDevice));
        CUDA_OK(cudaMalloc(&P.d_rbuf, sizeof(double) * per * P.nrecv));
      }
      if (P.nemit) {
        CUDA_OK(cudaMalloc(&P.d_emit, sizeof(int) * P.nemit));
        CUDA_OK(cudaMemcpy(P.d_emit, igrid_emit[cpu], sizeof(int) * P.nemit, cudaMemcpyHostToDevice));
        CUDA_OK(cudaMalloc(&P.d_sbuf, sizeof(double) * per * P.nemit));
      }
    }
  }
  const int nd = G.p.ndim, nvar = G.p.nvar, TW = 2 * nd, NSF = 1 << (nd - 1);
  A.dx = level_dx(ilevel);
  A.nact = ngrid_active;
  CUDA_OK(cudaMalloc(&A.d_active, sizeof(int) * std::max(1, ngrid_active)));
  if (ngrid_active > 0) CUDA_OK(cudaMemcpy(A.d_active, igrid_active, sizeof(int) * ngrid_active, cudaMemcpyHostToDevice));
  CUDA_OK(cudaMalloc(&A.d_rflux, sizeof(double) * (size_t)std::max(1, ngrid_active) * TW * NSF * G.nvn));
  (void)nvar;
  A.regions.resize(nboundary);
  for (int b = 0; b < nboundary; b++) {
    A.regions[b].type = boundary_type[b];
    A.regions[b].n = ngrid_bound[b];
    if (ngrid_bound[b] > 0) {
      CUDA_OK(cudaMalloc(&A.regions[b].d_igrid, sizeof(int) * ngrid_bound[b]));
      CUDA_OK(cudaMemcpy(A.regions[b].d_igrid, igrid_bound[b], sizeof(int) * ngrid_bound[b], cudaMemcpyHostToDevice));
    }
  }
  // reflux schedule (hydro/godunov_fine.f90:798-908): contributions in the order the reference visits them (amr_schedules.h)
  {
    std::vector<int> cells, start, srcs, src;
    build_reflux_schedule(nd, G.p.nvector, ngrid_active, igrid_active, G.nbor, G.son, G.ngridmax, cells, start, srcs, src);
    A.nent = (int)cells.size();
    {   // octs that own at least one refluxed face, in active-list order
      std::vector<char> mark((size_t)std::max(1, ngrid_active), 0);
      for (int sv : src) mark[(size_t)(sv >> 6)] = 1;
      A.h_surf_io.clear();
      for (int i = 0; i < ngrid_active; i++) if (mark[i]) A.h_surf_io.push_back(i);
    }
    if (A.nent > 0) {
      if (ngrid_active >= (1 << 25)) return fail(RGPU_EUNSUPPORTED, "too many octs for the packed reflux schedule");
      CUDA_OK(cudaMalloc(&A.d_rcell, sizeof(int) * cells.size()));
      CUDA_OK(cudaMalloc(&A.d_rstart, sizeof(int) * start.size()));
      CUDA_OK(cudaMalloc(&A.d_rsrc, sizeof(int) * srcs.size()));
      CUDA_OK(cudaMemcpy(A.d_rcell, cells.data(), sizeof(int) * cells.size(), cudaMemcpyHostToDevice));
      CUDA_OK(cudaMemcpy(A.d_rstart, start.data(), sizeof(int) * start.size(), cudaMemcpyHostToDevice));
      CUDA_OK(cudaMemcpy(A.d_rsrc, srcs.data(), sizeof(int) * srcs.size(), cudaMemcpyHostToDevice));
    }
  }
  CUDA_OK(cudaMalloc(&A.d_part, sizeof(double) * 4 * reduce_blocks()));
  CUDA_OK(cudaMalloc(&A.d_out, sizeof(double) * 5));
  CUDA_OK(cudaMalloc(&A.d_dt, sizeof(double)));
  A.bound = true;
  return RGPU_OK;
}
template <int ND>
cudaError_t dispatch_amr_nd(int riemann, const AmrSweepArgs& a, cudaStream_t st) {
  switch (riemann) {
    case RGPU_RIEMANN_LLF: return launch_amr_godfine<ND, RIEMANN_LLF>(a, st);
    case RGPU_RIEMANN_EXACT: return launch_amr_godfine<ND, RIEMANN_EXACT>(a, st);
    case RGPU_RIEMANN_ACOUSTIC: return launch_amr_godfine<ND, RIEMANN_ACOUSTIC>(a, st);
    case RGPU_RIEMANN_HLLC: return launch_amr_godfine<ND, RIEMANN_HLLC>(a, st);
    default: return launch_amr_godfine<ND, RIEMANN_HLL>(a, st);
  }
}
// godunov_fine of a fully refined level inside an AMR run through the dense kernel: gather uold (all octs of the box) and
// unew (it carries the refluxes of the finer level) into the level store, masked sweep, scatter unew of the active octs
int amr_godunov_dense(AmrLevel& A, int ilevel, double dt, const double* dt_dev) {
  Level& L = G.lev[ilevel];
  const int nthr = 256;
  const unsigned nb = (unsigned)((L.nslot + nthr - 1) / nthr);
  amr_gather_slots_kernel<<<nb, nthr, 0, G.stream>>>(G.d_uold, L.d_u[0], L.d_slot_igrid, L.nslot, G.ncoarse, G.ngridmax, G.ncell, G.p.nvar, T_());
  amr_gather_slots_kernel<<<nb, nthr, 0, G.stream>>>(G.d_unew, L.d_u[1], L.d_slot_igrid, L.nslot, G.ncoarse, G.ngridmax, G.ncell, G.p.nvar, T_());
  CUDA_OK(cudaGetLastError());
  if (G.p.pressure_fix) {   // divu, enew (columns nvar, nvar+1 of unew: set_unew's values + the finer level's refluxes)
    amr_gather_slots_kernel<<<nb, nthr, 0, G.stream>>>(d_divu(), L.d_pfix, L.d_slot_igrid, L.nslot, G.ncoarse, G.ngridmax, G.ncell, 2, T_());
    CUDA_OK(cudaGetLastError());
    A.launches++;
  }
  if (G.p.poisson) {   // f of every oct of the box (the host may upload a new f every step); a patch's empty shell slots take the
                       // f of their father cell (gloc gather, godunov_fine.f90:637-647)
    amr_gather_slots_kernel<<<nb, nthr, 0, G.stream>>>(G.d_force, L.d_f, L.d_slot_igrid, L.nslot, G.ncoarse, G.ngridmax, G.ncell, G.p.ndim, T_());
    CUDA_OK(cudaGetLastError());
    A.launches++;
    if (A.patch) {
      amr_fill_shell_force_kernel<<<nb, nthr, 0, G.stream>>>(G.d_force, L.d_f, A.d_shell_father, L.nslot, G.ncell, G.p.ndim);
      CUDA_OK(cudaGetLastError());
      A.launches++;
    }
  }
  if (A.patch) {   // ghost shell: prolongation from level l-1 (what godfine1 does for every missing neighbour oct, :583-593)
    const long long n = L.nslot * G.p.nvar;
    if (G.interpol_var != 0 || G.interpol_type == 4)
      amr_fill_shell_coupled_kernel<<<(unsigned)((L.nslot + nthr - 1) / nthr), nthr, 0, G.stream>>>(amr_tree(), G.d_uold, L.d_u[0], A.d_shell_father, L.nslot,
                                                                                              ilevel, G.interpol_type, G.interpol_var, G.p.smallr);
    else
    amr_fill_shell_kernel<<<(unsigned)((n + nthr - 1) / nthr), nthr, 0, G.stream>>>(amr_tree(), G.d_uold, L.d_u[0], A.d_shell_father, L.nslot, ilevel,
                                                                                G.p.nvar, G.interpol_type);
    CUDA_OK(cudaGetLastError());
    A.launches++;
  }
  SweepArgs a{};
  a.uin = L.d_u[0]; a.uout = L.d_u[1]; a.g = L.g; a.P = G.phys; a.dt_dev = dt_dev; a.dt_val = dt; a.dx = L.dx; a.inv_dx = 1.0 / L.dx;
  int ex;
  a.dx_pow2 = (std::frexp(L.dx, &ex) == 0.5) ? 1 : 0;
  a.ntx = L.ntx; a.nty = L.nty; a.nwork = L.nwork; a.part = nullptr; a.refined = L.d_refined;
  cudaError_t e;
  if (G.p.poisson) { a.force = L.d_f; a.gsrc = 0; }   // predictor only: set_uold and courant_fine apply the gravity terms
                                                      // through their list kernels
  if (G.p.pressure_fix) {   // tmp1 / tmp2 into divu / enew; set_uold's pdV source and energy switch run as list kernels
    a.pfix = L.d_pfix;
    e = G.p.poisson ? dispatch_sweep_pfix<true>(G.p.riemann, a, L.nblocks, G.stream)
                    : dispatch_sweep_pfix<false>(G.p.riemann, a, L.nblocks, G.stream);
  } else if (G.p.poisson) {
    e = dispatch_sweep_grav<3, true>(G.p.riemann, a, L.nblocks, G.stream);
  } else
  switch (G.p.riemann) {
    case RGPU_RIEMANN_LLF: e = launch_sweep_dense_amr<3, RIEMANN_LLF>(a, L.nblocks, G.stream); break;
    case RGPU_RIEMANN_EXACT: e = launch_sweep_dense_amr<3, RIEMANN_EXACT>(a, L.nblocks, G.stream); break;
    case RGPU_RIEMANN_ACOUSTIC: e = launch_sweep_dense_amr<3, RIEMANN_ACOUSTIC>(a, L.nblocks, G.stream); break;
    case RGPU_RIEMANN_HLLC: e = launch_sweep_dense_amr<3, RIEMANN_HLLC>(a, L.nblocks, G.stream); break;
    default: e = launch_sweep_dense_amr<3, RIEMANN_HLL>(a, L.nblocks, G.stream); break;
  }
  if (e != cudaSuccess) return fail(RGPU_ECUDA, "dense AMR sweep launch: %s", cudaGetErrorString(e));
  amr_scatter_slots_kernel<<<nb, nthr, 0, G.stream>>>(G.d_unew, L.d_u[1], L.d_slot_igrid, L.nslot, G.ncoarse, G.ngridmax, G.ncell, G.p.nvar, T_(), L.g);
  CUDA_OK(cudaGetLastError());
  A.launches += 4;
  if (G.p.pressure_fix) {
    amr_scatter_slots_kernel<<<nb, nthr, 0, G.stream>>>(d_divu(), L.d_pfix, L.d_slot_igrid, L.nslot, G.ncoarse, G.ngridmax, G.ncell, 2, T_(), L.g);
    CUDA_OK(cudaGetLastError());
    A.launches++;
  }
  if (A.patch && A.nsurf > 0) {   // fluxes through the outer faces of the surface octs, then the coarse reflux pass
    AmrSweepArgs s{};
    s.t = amr_tree();
    s.active = A.d_surf_igrid; s.nact = A.nsurf; s.ilevel = ilevel;
    s.uold = G.d_uold; s.unew = G.d_unew; s.rflux = A.d_rflux;
    s.P = G.phys; s.dt = dt; s.dt_dev = dt_dev; s.dx = A.dx; s.inv_dx = 1.0 / A.dx; s.dx_pow2 = a.dx_pow2;
    s.interpol_type = G.interpol_type; s.interpol_var = G.interpol_var; s.difmag = 0.0; s.nps = 0;
    s.flux_only = 1; s.rflux_index = A.d_surf_io;
    // the refluxed faces carry the gravity predictor and, with pressure_fix, tmp1 / tmp2 behind the fluxes
    s.force = G.p.poisson ? G.d_force : nullptr; s.pfix = G.p.pressure_fix ? 1 : 0; s.nvr = G.nvn;
    e = dispatch_amr_nd<3>(G.p.riemann, s, G.stream);
    if (e != cudaSuccess) return fail(RGPU_ECUDA, "patch surface flux launch: %s", cudaGetErrorString(e));
    A.launches++;
  }
  if (A.nent > 0) {
    RefluxArgs r{};
    r.nent = A.nent; r.cell = A.d_rcell; r.start = A.d_rstart; r.src = A.d_rsrc; r.rflux = A.d_rflux; r.unew = G.d_unew;
    r.ncell = G.ncell; r.nvar = G.nvn; r.nsides = 2 * G.p.ndim; r.nsf = 1 << (G.p.ndim - 1);   // nvn: divu / enew reflux like variables
    r.oneontwotondim = 1.0 / (double)(1 << G.p.ndim);
    const int n = A.nent * G.nvn;
    amr_reflux_kernel<<<(n + 127) / 128, 128, 0, G.stream>>>(r);
    CUDA_OK(cudaGetLastError());
    A.launches++;
  }
  return RGPU_OK;
}

int mhd_amr_godunov(AmrLevel& A, int ilevel, double dt, const double* dt_dev);
int amr_godunov(AmrLevel& A, int ilevel, double dt, const double* dt_dev = nullptr) {
  A.dt_last = dt;
  if (A.nact == 0) return RGPU_OK;
  if (G.p.mhd) return mhd_amr_godunov(A, ilevel, dt, dt_dev);
  if (A.dense_sweep) return amr_godunov_dense(A, ilevel, dt, dt_dev);
  AmrSweepArgs a{};
  a.dt_dev = dt_dev;
  a.t = amr_tree();
  a.active = A.d_active; a.nact = A.nact; a.ilevel = ilevel;
  a.uold = G.d_uold; a.unew = G.d_unew; a.rflux = A.d_rflux;
  a.P = G.phys; a.dt = dt; a.dx = A.dx; a.inv_dx = 1.0 / A.dx;
  int ex;
  a.dx_pow2 = (std::frexp(A.dx, &ex) == 0.5) ? 1 : 0;
  a.interpol_type = G.interpol_type; a.interpol_var = G.interpol_var;
  a.difmag = G.p.difmag;
  a.nps = G.p.nvar - (G.p.ndim + 2);
  a.force = G.p.poisson ? G.d_force : nullptr; a.pfix = G.p.pressure_fix ? 1 : 0; a.nvr = G.nvn;
  cudaError_t e;
  if (G.p.ndim == 1) e = dispatch_amr_nd<1>(G.p.riemann, a, G.stream);
  else if (G.p.ndim == 2) e = dispatch_amr_nd<2>(G.p.riemann, a, G.stream);
  else e = dispatch_amr_nd<3>(G.p.riemann, a, G.stream);
  if (e != cudaSuccess) return fail(RGPU_ECUDA, "amr sweep launch: %s", cudaGetErrorString(e));
  A.launches++;
  if (A.nent > 0) {
    RefluxArgs r{};
    r.nent = A.nent; r.cell = A.d_rcell; r.start = A.d_rstart; r.src = A.d_rsrc; r.rflux = A.d_rflux; r.unew = G.d_unew;
    r.ncell = G.ncell; r.nvar = G.nvn; r.nsides = 2 * G.p.ndim; r.nsf = 1 << (G.p.ndim - 1);   // nvn: divu / enew reflux like variables
    r.oneontwotondim = 1.0 / (double)(1 << G.p.ndim);
    const int n = A.nent * G.nvn;
    amr_reflux_kernel<<<(n + 127) / 128, 128, 0, G.stream>>>(r);
    CUDA_OK(cudaGetLastError());
    A.launches++;
  }
  return RGPU_OK;
}
int amr_copy(AmrLevel& A, const double* src, double* dst) {
  if (A.nact == 0) return RGPU_OK;
  const long long n = (long long)A.nact * T_() * G.nvs;
  amr_copy_octs_kernel<<<(unsigned)((n + 255) / 256), 256, 0, G.stream>>>(src, dst, A.d_active, A.nact, G.ncoarse, G.ngridmax, G.ncell, T_(), G.nvs);
  CUDA_OK(cudaGetLastError());
  A.launches++;
  return RGPU_OK;
}
// make_virtual_fine_dp (forward: emission octs -> peers' reception octs, copy) / make_virtual_reverse_dp (reverse:
// reception octs -> owners' emission octs, accumulate in peer order) on the mirrored arrays, one NCCL group per call
int amr_exchange(AmrLevel& A, double* u, bool reverse) {
  if (A.peers.empty()) return RGPU_OK;
  if (!G.comm) return fail(RGPU_EINVAL, "ghost exchange needs rgpu_comm_init");
  // reverse runs on unew: with pressure_fix its columns nvar, nvar+1 are divu and enew (amr_step.f90:397-404)
  const int T = T_(), nvar = (reverse && u == G.d_unew) ? G.nvn : G.nvs;
  const long long per = (long long)T * nvar;
  for (auto& P : A.peers) {
    const int n = reverse ? P.nrecv : P.nemit;
    if (!n) continue;
    amr_pack_kernel<<<(unsigned)((n * per + 255) / 256), 256, 0, G.stream>>>(u, reverse ? P.d_recv : P.d_emit, n, G.ncoarse, G.ngridmax, G.ncell, T, nvar,
                                                                            reverse ? P.d_rbuf : P.d_sbuf);
    CUDA_OK(cudaGetLastError());
    A.launches++;
  }
  NCCL_OK(ncclGroupStart());
  for (int cpu = 0; cpu < (int)A.peers.size(); cpu++) {
    AmrPeer& P = A.peers[cpu];
    const int nsend = reverse ? P.nrecv : P.nemit, nrecv = reverse ? P.nemit : P.nrecv;
    if (nsend) NCCL_OK(ncclSend(reverse ? P.d_rbuf : P.d_sbuf, (size_t)nsend * per, ncclDouble, cpu, G.comm, G.stream));
    if (nrecv) NCCL_OK(ncclRecv(reverse ? P.d_sbuf : P.d_rbuf, (size_t)nrecv * per, ncclDouble, cpu, G.comm, G.stream));
  }
  NCCL_OK(ncclGroupEnd());
  for (auto& P : A.peers) {
    const int n = reverse ? P.nemit : P.nrecv;
    if (!n) continue;
    amr_unpack_kernel<<<(unsigned)((n * per + 255) / 256), 256, 0, G.stream>>>(u, reverse ? P.d_emit : P.d_recv, n, G.ncoarse, G.ngridmax, G.ncell, T, nvar,
                                                                              reverse ? P.d_sbuf : P.d_rbuf, reverse ? 1 : 0);
    CUDA_OK(cudaGetLastError());
    A.launches++;
  }
  return RGPU_OK;
}
int amr_zero_ghost_unew(AmrLevel& A) {   // set_unew: unew (and divu, enew) = 0 in the reception octs (godunov_fine.f90:93-126)
  const long long per = (long long)T_() * G.nvn;
  for (auto& P : A.peers)
    if (P.nrecv) {
      amr_unpack_kernel<<<(unsigned)((P.nrecv * per + 255) / 256), 256, 0, G.stream>>>(G.d_unew, P.d_recv, P.nrecv, G.ncoarse, G.ngridmax, G.ncell, T_(), G.nvn,
                                                                                   nullptr, 2);
      CUDA_OK(cudaGetLastError());
      A.launches++;
    }
  return RGPU_OK;
}

// ---- ideal MHD in AMR mode, NDIM = 1, 2 (mhd_amr.cuh) -----------------------------------------------------------------------
int mhd_amr_bind_extra(AmrLevel& A, int ilevel, int ngrid_active, const int* igrid_active) {
  (void)igrid_active;
  if (G.p.ndim == 1 || ngrid_active == 0) return RGPU_OK;
  const int nd = G.p.ndim, N3 = nd == 2 ? 9 : 27, nemf = nd == 2 ? 4 : 81;
  CUDA_OK(cudaMalloc(&A.d_remf, sizeof(double) * nemf * (size_t)ngrid_active));
  // the 3^ndim father cells of every oct (device tree walk), then the schedule on the host in the reference's visiting order:
  // batch of nvector octs -> edge -> oct of the batch -> the statements of the edge (amr_schedules.h)
  std::vector<int> nfc((size_t)ngrid_active * N3);
  int* d_nfc = nullptr;
  CUDA_OK(cudaMalloc(&d_nfc, sizeof(int) * nfc.size()));
  if (nd == 2) amr_nfc_kernel<2><<<(ngrid_active + 127) / 128, 128, 0, G.stream>>>(amr_tree(), A.d_active, ngrid_active, ilevel, d_nfc);
  else amr_nfc_kernel<3><<<(ngrid_active + 127) / 128, 128, 0, G.stream>>>(amr_tree(), A.d_active, ngrid_active, ilevel, d_nfc);
  CUDA_OK(cudaGetLastError());
  CUDA_OK(cudaMemcpyAsync(nfc.data(), d_nfc, sizeof(int) * nfc.size(), cudaMemcpyDeviceToHost, G.stream));
  CUDA_OK(cudaStreamSynchronize(G.stream));
  cudaFree(d_nfc);
  if (ngrid_active >= (1 << 24)) return fail(RGPU_EUNSUPPORTED, "too many octs for the packed EMF reflux schedule");
  std::vector<int> cells, vars, start, codes;
  if (nd == 2) build_emf_schedule_2d(G.p.nvector, ngrid_active, nfc.data(), G.son, cells, vars, start, codes);
  else build_emf_schedule_3d(G.p.nvector, ngrid_active, nfc.data(), G.son, cells, vars, start, codes);
  A.nemf = (int)cells.size();
  if (A.nemf > 0) {
    CUDA_OK(cudaMalloc(&A.d_ecell, sizeof(int) * cells.size()));
    CUDA_OK(cudaMalloc(&A.d_evar, sizeof(int) * vars.size()));
    CUDA_OK(cudaMalloc(&A.d_estart, sizeof(int) * start.size()));
    CUDA_OK(cudaMalloc(&A.d_ecode, sizeof(int) * codes.size()));
    CUDA_OK(cudaMemcpy(A.d_ecell, cells.data(), sizeof(int) * cells.size(), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(A.d_evar, vars.data(), sizeof(int) * vars.size(), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(A.d_estart, start.data(), sizeof(int) * start.size(), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(A.d_ecode, codes.data(), sizeof(int) * codes.size(), cudaMemcpyHostToDevice));
  }
  return RGPU_OK;
}
int mhd_amr_godunov(AmrLevel& A, int ilevel, double dt, const double* dt_dev) {
  MhdAmrArgs a{};
  a.t = amr_tree(); a.active = A.d_active; a.nact = A.nact; a.ilevel = ilevel;
  a.uold = G.d_uold; a.unew = G.d_unew; a.rflux = A.d_rflux; a.remf = A.d_remf;
  a.P = G.mphys; a.dt = dt; a.dx = A.dx; a.dt_dev = dt_dev;
  a.interpol_type = G.interpol_type; a.interpol_mag_type = G.interpol_mag_type < 0 ? G.interpol_type : G.interpol_mag_type;
  a.riemann = G.p.riemann; a.riemann2d = G.p.riemann2d;
  if (G.p.ndim == 1) mhd_amr1_godfine_kernel<<<(A.nact + 63) / 64, 64, 0, G.stream>>>(a);
  else if (G.p.ndim == 2) mhd_amr2_godfine_kernel<<<A.nact, MHD2_TPO, 0, G.stream>>>(a);
  else {
    static bool attr = false;
    if (!attr) { CUDA_OK(cudaFuncSetAttribute(mhd_amr3_godfine_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(Mhd3Sm))); attr = true; }
    mhd_amr3_godfine_kernel<<<A.nact, MHD3_TPO, sizeof(Mhd3Sm), G.stream>>>(a);
  }
  CUDA_OK(cudaGetLastError());
  A.launches++;
  if (A.nent > 0) {   // Euler fluxes into the coarser level (:1030-1168)
    RefluxArgs r{};
    r.nent = A.nent; r.cell = A.d_rcell; r.start = A.d_rstart; r.src = A.d_rsrc; r.rflux = A.d_rflux; r.unew = G.d_unew;
    r.ncell = G.ncell; r.nvar = MNVS; r.nsides = 2 * G.p.ndim; r.nsf = 1 << (G.p.ndim - 1);
    r.oneontwotondim = 1.0 / (double)(1 << G.p.ndim);
    const int n = A.nent * MNVS;
    mhd_amr_reflux_kernel<<<(n + 127) / 128, 128, 0, G.stream>>>(r);
    CUDA_OK(cudaGetLastError());
    A.launches++;
  }
  if (A.nemf > 0) {   // corner EMFs into the coarser level (:1176-1270)
    if (G.p.ndim == 3) {
      Emf3RefluxArgs r{};
      r.nent = A.nemf; r.cell = A.d_ecell; r.var = A.d_evar; r.start = A.d_estart; r.code = A.d_ecode; r.remf = A.d_remf; r.unew = G.d_unew;
      r.ncell = G.ncell;
      const MhdEdge3Host* E = mhd_edges3();
      for (int e = 0; e < 12; e++) {
        r.edir[e] = (signed char)E[e].dir;
        r.ec0[e] = (signed char)(((E[e].c[0][2] - 1) * 3 + (E[e].c[0][1] - 1)) * 3 + (E[e].c[0][0] - 1));
        r.ec1[e] = (signed char)(((E[e].c[1][2] - 1) * 3 + (E[e].c[1][1] - 1)) * 3 + (E[e].c[1][0] - 1));
      }
      mhd_amr_emf3_reflux_kernel<<<(A.nemf + 127) / 128, 128, 0, G.stream>>>(r);
    } else {
    EmfRefluxArgs r{};
    r.nent = A.nemf; r.cell = A.d_ecell; r.var = A.d_evar; r.start = A.d_estart; r.code = A.d_ecode; r.remf = A.d_remf; r.unew = G.d_unew;
    r.ncell = G.ncell;
    mhd_amr_emf_reflux_kernel<<<(A.nemf + 127) / 128, 128, 0, G.stream>>>(r);
    }
    CUDA_OK(cudaGetLastError());
    A.launches++;
  }
  return RGPU_OK;
}
int mhd_amr_upload(AmrLevel& A) {
  if (A.nact == 0) return RGPU_OK;
  const int n = A.nact * T_();
  for (int pass = 0; pass < 2; pass++) {
    mhd_amr_upload_kernel<<<(n + 127) / 128, 128, 0, G.stream>>>(G.d_uold, amr_tree(), A.d_active, A.nact, G.p.ndim, G.p.smallr, pass);
    CUDA_OK(cudaGetLastError());
    A.launches++;
  }
  return RGPU_OK;
}
int mhd_amr_boundaries(AmrLevel& A) {
  for (auto& r : A.regions) {
    if (r.n == 0) continue;
    const int bt = r.type, dir = bt - 10 * (bt / 10);
    if (G.p.ndim != 1 || bt / 10 > 1) return fail(RGPU_EUNSUPPORTED, "MHD AMR mode: boundary type %d with NDIM=%d not supported (NDIM=1 reflexive / outflow; periodic otherwise)", bt, G.p.ndim);
    MhdAmrBoundArgs b{};
    b.n = r.n; b.igrid = r.d_igrid; b.dir = dir; b.kind = bt / 10; b.smallr = G.p.smallr;
    mhd_amr1_boundary_kernel<<<(r.n * 2 + 127) / 128, 128, 0, G.stream>>>(G.d_uold, amr_tree(), b);
    CUDA_OK(cudaGetLastError());
    A.launches++;
  }
  return RGPU_OK;
}

// set_unew (hydro/godunov_fine.f90:40-130): unew = uold on the active octs (+ divu = 0, enew = e_int), 0 on the reception octs
int amr_set_unew(AmrLevel& A) {
  int rc = amr_copy(A, G.d_uold, G.d_unew); if (rc) return rc;
  if (G.p.pressure_fix && A.nact > 0) {
    const int n = A.nact * T_();
    amr_pfix_init_kernel<<<(n + 127) / 128, 128, 0, G.stream>>>(G.d_uold, d_divu(), d_enew(), A.d_active, A.nact, G.ncoarse, G.ngridmax, G.ncell, T_(),
                                                             G.p.ndim, G.p.smallr);
    CUDA_OK(cudaGetLastError());
    A.launches++;
  }
  return amr_zero_ghost_unew(A);
}
// set_uold (hydro/godunov_fine.f90:135-232): gravity and pdV sources on unew / enew, scalar floor fix, uold = unew, energy switch
int amr_set_uold(AmrLevel& A, int ilevel, const double* dt_dev) {
  (void)ilevel;
  if (A.nact == 0) return RGPU_OK;
  const int n = A.nact * T_(), nb = (n + 127) / 128;
  if (src_terms() && !dt_dev && !(A.dt_last > 0)) return fail(RGPU_EINVAL, "set_uold with source terms before godunov_fine (dtnew(ilevel) unknown)");
  if (G.p.poisson) {
    amr_gravity_src_kernel<<<nb, 128, 0, G.stream>>>(G.d_uold, G.d_unew, G.d_force, A.d_active, A.nact, G.ncoarse, G.ngridmax, G.ncell, T_(), G.p.ndim,
                                                  G.p.smallr, A.dt_last, dt_dev);
    CUDA_OK(cudaGetLastError());
    A.launches++;
  }
  if (G.p.pressure_fix) {
    amr_pdv_kernel<<<nb, 128, 0, G.stream>>>(amr_tree(), G.d_uold, d_enew(), A.d_active, A.nact, G.p.ndim, G.p.gamma, G.p.smallr, A.dx, A.dt_last, dt_dev);
    CUDA_OK(cudaGetLastError());
    A.launches++;
  }
  const int nps = G.p.mhd ? 0 : G.p.nvar - (G.p.ndim + 2);
  if (nps > 0) {   // passive-scalar fix for floored densities, before the copy (godunov_fine.f90:176-190)
    amr_scalar_floor_kernel<<<nb, 128, 0, G.stream>>>(G.d_uold, G.d_unew, A.d_active, A.nact, G.ncoarse, G.ngridmax, G.ncell, T_(),
                                                   G.p.ndim + 2, G.p.nvar, G.p.smallr);
    CUDA_OK(cudaGetLastError());
    A.launches++;
  }
  int rc = amr_copy(A, G.d_unew, G.d_uold); if (rc) return rc;
  if (G.p.pressure_fix) {
    amr_pfix_switch_kernel<<<nb, 128, 0, G.stream>>>(G.d_uold, d_divu(), d_enew(), A.d_active, A.nact, G.ncoarse, G.ngridmax, G.ncell, T_(), G.p.ndim,
                                                  G.p.smallr, G.p.beta_fix, A.dx, A.dt_last, dt_dev);
    CUDA_OK(cudaGetLastError());
    A.launches++;
  }
  return RGPU_OK;
}
int amr_courant_launch(AmrLevel& A) {
  const int nb = reduce_blocks();
  if (G.p.mhd) {
    mhd_amr_courant_kernel<<<nb, 256, 0, G.stream>>>(G.d_uold, amr_tree(), A.d_active, A.nact, G.mphys, A.dx, G.p.ndim, A.d_part);
    CUDA_OK(cudaGetLastError());
    return RGPU_OK;
  }
  const double* f = G.p.poisson ? G.d_force : nullptr;
  if (G.p.ndim == 1) amr_courant_kernel<1><<<nb, 256, 0, G.stream>>>(G.d_uold, amr_tree(), A.d_active, A.nact, G.phys, A.dx, A.d_part, f);
  else if (G.p.ndim == 2) amr_courant_kernel<2><<<nb, 256, 0, G.stream>>>(G.d_uold, amr_tree(), A.d_active, A.nact, G.phys, A.dx, A.d_part, f);
  else amr_courant_kernel<3><<<nb, 256, 0, G.stream>>>(G.d_uold, amr_tree(), A.d_active, A.nact, G.phys, A.dx, A.d_part, f);
  CUDA_OK(cudaGetLastError());
  return RGPU_OK;
}

int amr_boundaries(AmrLevel& A) {
  if (G.p.mhd) return mhd_amr_boundaries(A);
  static const int ref_x[8] = {2, 1, 4, 3, 6, 5, 8, 7}, ref_y[8] = {3, 4, 1, 2, 7, 8, 5, 6}, ref_z[8] = {5, 6, 7, 8, 1, 2, 3, 4};
  static const int fre[6][8] = {{1, 1, 3, 3, 5, 5, 7, 7}, {2, 2, 4, 4, 6, 6, 8, 8}, {1, 2, 1, 2, 5, 6, 5, 6},
                                {3, 4, 3, 4, 7, 8, 7, 8}, {1, 2, 3, 4, 1, 2, 3, 4}, {5, 6, 7, 8, 5, 6, 7, 8}};
  static const int inb[7] = {0, 2, 1, 4, 3, 6, 5};
  int ibr = -1;
  for (auto& r : A.regions) {
    ibr++;
    if (r.n == 0) continue;
    const int bt = r.type, dir = bt - 10 * (bt / 10);
    if (bt / 10 > 2) return fail(RGPU_EUNSUPPORTED, "boundary type %d not supported", bt);
    if (bt / 10 == 2 && !G.bvar_set[ibr]) return fail(RGPU_EINVAL, "imposed boundary %d: call rgpu_set_boundary_var first", ibr + 1);
    AmrBoundArgs b{};
    b.n = r.n; b.igrid = r.d_igrid; b.inbor = inb[dir];
    const int d = (dir - 1) / 2;
    const int* ir = (bt / 10 == 0) ? (d == 0 ? ref_x : d == 1 ? ref_y : ref_z) : fre[dir - 1];
    for (int i = 0; i < 8; i++) b.ind_ref[i] = ir[i];
    b.gs[0] = b.gs[1] = b.gs[2] = 1.0;
    if (bt >= 1 && bt <= 6) b.gs[d] = -1.0;
    b.kind = bt / 10; b.ndim = G.p.ndim; b.nvar = G.p.nvar; b.smallr = G.p.smallr;
    for (int iv = 0; iv < 8; iv++) b.bvar[iv] = G.bvar[ibr][iv];
    const int nthr = r.n * T_();
    amr_boundary_kernel<<<(nthr + 127) / 128, 128, 0, G.stream>>>(G.d_uold, amr_tree(), b);
    CUDA_OK(cudaGetLastError());
    A.launches++;
  }
  return RGPU_OK;
}

int exchange_ghosts(Level& L, double* u, bool reverse);
int exchange_ghosts_fused(Level& L, double* u, cudaStream_t st, ncclComm_t comm);

// set_uold only touches the active cells: the boundary / ghost shells keep their uold values until the next
// make_boundary_hydro / make_virtual_fine.  With ping-pong buffers those values must be carried over explicitly
// (corner boundary octs read neighbours that are refreshed later in the same pass, hydro_boundary.f90:53).
int carry_shells(Level& L, const double* from, double* to, bool peers = true) {
  const long long np = (long long)nplanes_();
  for (auto& r : L.regions)
    if (r.n) {
      copy_octs_kernel<<<(unsigned)(((long long)r.n * np + 255) / 256), 256, 0, G.stream>>>(from, to, r.d_slots, r.n, L.nslot, (int)np);
      CUDA_OK(cudaGetLastError());
      L.launches++;
    }
  if (peers) for (auto& P : L.peers)
    if (P.nrecv) {
      copy_octs_kernel<<<(unsigned)(((long long)P.nrecv * np + 255) / 256), 256, 0, G.stream>>>(from, to, P.d_recv, P.nrecv, L.nslot, (int)np);
      CUDA_OK(cudaGetLastError());
      L.launches++;
    }
  return RGPU_OK;
}

}  // namespace

// ============================================================================= C ABI
extern "C" {

int rgpu_abi_version(void) { return RGPU_ABI_VERSION; }
const char* rgpu_last_error(void) { return g_err; }

int rgpu_init(const rgpu_params* p, int myid, int ncpu, int device) {
  if (!p) return fail(RGPU_EINVAL, "null params");
  if (p->ndim < 1 || p->ndim > 3) return fail(RGPU_EINVAL, "ndim=%d", p->ndim);
  if (p->mhd) {
    // NDIM = 3: dense levelmin=levelmax path (mhd_dense.cuh); NDIM = 1, 2: AMR mode (rgpu_set_amr; mhd_amr.cuh)
    if (p->nvar != 8) return fail(RGPU_EUNSUPPORTED, "MHD build: nvar=%d: passive scalars / NENER not supported (need nvar=8)", p->nvar);
    if (p->riemann < 0 || p->riemann > 5) return fail(RGPU_EINVAL, "unknown riemann solver");     // mhd/umuscl.f90:1435
    if (p->riemann2d < 0 || p->riemann2d > 5) return fail(RGPU_EINVAL, "unknown 2D riemann solver"); // mhd/umuscl.f90:1886
    const int smt = p->slope_mag_type == -1 ? p->slope_type : p->slope_mag_type;
    if (!(smt == 0 || smt == 1 || smt == 2)) return fail(RGPU_EINVAL, "Unknown mag. slope type %d", smt);   // mhd/umuscl.f90:2655
    if (!(p->slope_type == 0 || p->slope_type == 1 || p->slope_type == 2 || p->slope_type == 3 || p->slope_type == 7 || p->slope_type == 8))
      return fail(RGPU_EINVAL, "Unknown slope type %d", p->slope_type);                                      // mhd/umuscl.f90:2562
  } else {
  {
    const int nps = p->nvar - (p->ndim + 2);
    if (nps < 0) return fail(RGPU_EINVAL, "nvar=%d < ndim+2", p->nvar);
    if (nps > 0 && !(p->ndim == 3 && nps <= 2 && !(p->difmag > 0.0)))
      return fail(RGPU_EUNSUPPORTED, "nvar=%d: passive scalars are built for NDIM=3, at most 2 of them, difmag=0 (NENER not supported)", p->nvar);
  }
  if (p->riemann < 0 || p->riemann > 4) return fail(RGPU_EINVAL, "unknown Riemann solver %d", p->riemann);
  }
  if (p->scheme != RGPU_SCHEME_MUSCL) return fail(RGPU_EUNSUPPORTED, "scheme='plmde' not supported");
  if (p->pressure_fix || p->poisson) {   // built in the oct-batch kernel (rgpu_set_amr), hydro variables only
    if (p->mhd) return fail(RGPU_EUNSUPPORTED, "MHD build: poisson / pressure_fix not supported");
    if (p->nvar != p->ndim + 2 || p->difmag > 0.0)
      return fail(RGPU_EUNSUPPORTED, "poisson / pressure_fix: built for nvar=ndim+2 and difmag=0 (no passive scalars, NENER)");
    if (p->pressure_fix && !(p->beta_fix >= 0.0)) return fail(RGPU_EINVAL, "beta_fix=%g", p->beta_fix);
  }
  if (p->difmag > 0.0 && p->mhd) return fail(RGPU_EUNSUPPORTED, "MHD build: difmag>0 not supported");
  if (p->difmag < 0.0) return fail(RGPU_EINVAL, "difmag=%g", p->difmag);
  {
    const int st = p->slope_type;
    const bool ok = st == 0 || st == 1 || st == 2 || st == 3 || st == 7 || st == 8 || (p->ndim == 1 && st >= 4 && st <= 6);
    if (!ok) return fail(RGPU_EINVAL, "Unknown slope type %d", st);   // umuscl.f90:1083,1203,1476
  }
  if (G.init) rgpu_finalize();
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) return fail(RGPU_ECUDA, "no CUDA device: %s (there is no CPU fallback)", cudaGetErrorString(e));
  if (device < 0) {
    const char* lr = getenv("LOCAL_RANK");
    device = lr ? atoi(lr) % ndev : 0;
  }
  CUDA_OK(cudaSetDevice(device));
  G.p = *p; G.myid = myid; G.ncpu = ncpu; G.device = device;
  CUDA_OK(cudaDeviceGetAttribute(&G.nsm, cudaDevAttrMultiProcessorCount, device));
  CUDA_OK(cudaStreamCreateWithFlags(&G.stream, cudaStreamNonBlocking));
  CUDA_OK(cudaStreamCreateWithFlags(&G.s_in, cudaStreamNonBlocking));
  CUDA_OK(cudaStreamCreateWithFlags(&G.s_out, cudaStreamNonBlocking));
  CUDA_OK(cudaStreamCreateWithFlags(&G.s_x, cudaStreamNonBlocking));
  CUDA_OK(cudaEventCreateWithFlags(&G.ev_pipe, cudaEventDisableTiming));
  CUDA_OK(cudaEventCreate(&G.ev0));
  CUDA_OK(cudaEventCreate(&G.ev1));
  CUDA_OK(cudaEventCreate(&G.ev2));
  CUDA_OK(cudaEventCreate(&G.ev3));
  Phys& P = G.phys;
  P.gamma = p->gamma; P.smallr = p->smallr; P.smallc = p->smallc; P.slope_theta = p->slope_theta;
  P.courant_factor = p->courant_factor;
  P.smalle = p->smallc * p->smallc / p->gamma / (p->gamma - 1.0);
  P.smallp = p->smallc * p->smallc / p->gamma;
  P.smallpp = p->smallr * P.smallp;
  P.entho = 1.0 / (p->gamma - 1.0);
  P.gamma6 = (p->gamma + 1.0) / (2.0 * p->gamma);
  P.smallc2 = p->smallc * p->smallc;
  P.inv_gamma = 1.0 / p->gamma;
  P.cfl_g = 0.0001;
  P.cfl_rg = 1.0 / P.cfl_g;
  P.cfl_k = std::sqrt(1.0 + 2.0 * p->courant_factor * P.cfl_g) - 1.0;
  P.slope_type = p->slope_type; P.niter_riemann = p->niter_riemann;
  G.nvs = p->mhd ? p->nvar + 3 : p->nvar;
  G.nvn = G.nvs + (p->pressure_fix ? 2 : 0);
  for (int b = 0; b < 64; b++) G.bvar_set[b] = false;
  G.interpol_mag_type = -1;
  MPhys& M = G.mphys;
  M.gamma = p->gamma; M.smallr = p->smallr; M.smallc = p->smallc; M.slope_theta = p->slope_theta; M.courant_factor = p->courant_factor;
  M.smallp = p->smallr * (p->smallc * p->smallc) / p->gamma;
  M.slope_type = p->slope_type; M.slope_mag_type = p->slope_mag_type == -1 ? p->slope_type : p->slope_mag_type;
  G.init = true;
  return RGPU_OK;
}

int rgpu_finalize(void) {
  if (!G.init) return RGPU_OK;
  cudaStreamSynchronize(G.stream);
  drop_amr_graph();
  for (int l = 0; l <= MAXLEVEL; l++) if (G.lev[l].bound) free_level(G.lev[l]);
  for (int l = 0; l <= MAXLEVEL; l++) if (G.alev[l].bound) free_amr_level(G.alev[l]);
  cudaFree(G.d_son_base); cudaFree(G.d_father); cudaFree(G.d_nbor); cudaFree(G.d_uold); cudaFree(G.d_unew); cudaFree(G.d_force); G.d_force = nullptr; cudaFree(G.d_dtn); cudaFree(G.d_dto); cudaFree(G.d_numb);
  G.d_numb = nullptr; G.d_son_base = nullptr; G.d_son = G.d_father = G.d_nbor = nullptr; G.d_uold = G.d_unew = nullptr; G.d_dtn = G.d_dto = nullptr; G.ncell = 0; G.amr = false;
  if (G.comm_x) { ncclCommDestroy(G.comm_x); G.comm_x = nullptr; }
  if (G.comm) { ncclCommDestroy(G.comm); G.comm = nullptr; }
  cudaStreamDestroy(G.s_x);
  cudaEventDestroy(G.ev0); cudaEventDestroy(G.ev1); cudaEventDestroy(G.ev2); cudaEventDestroy(G.ev3);
  cudaEventDestroy(G.ev_pipe);
  cudaStreamDestroy(G.s_in); cudaStreamDestroy(G.s_out);
  cudaStreamDestroy(G.stream);
  G.init = false;
  return RGPU_OK;
}

int rgpu_set_amr(int on, int interpol_type, int interpol_var) {
  if (!G.init) return fail(RGPU_EINVAL, "rgpu_init has not been called");
  if (on && G.p.mhd && interpol_var != 0) return fail(RGPU_EUNSUPPORTED, "MHD build: interpol_var=%d not supported (0 only)", interpol_var);
  if (on && G.p.mhd && !(G.p.slope_type >= 0 && G.p.slope_type <= 2))
    return fail(RGPU_EUNSUPPORTED, "MHD AMR mode: slope_type=%d not supported (0, 1, 2)", G.p.slope_type);
  if (on && (interpol_var < 0 || interpol_var > 2)) return fail(RGPU_EINVAL, "interpol_var=%d (0, 1 or 2: hydro/interpol_hydro.f90:318-345)", interpol_var);
  if (on && (interpol_type < 0 || interpol_type > 4)) return fail(RGPU_EINVAL, "interpol_type=%d (0..4)", interpol_type);
  if (on && interpol_type == 4 && interpol_var != 2)
    return fail(RGPU_EINVAL, "interpol_type=4 (central slopes for the velocities) is designed for interpol_var=2 (hydro/interpol_hydro.f90:357-366)");
  drop_amr_graph();
  G.amr = on != 0;
  G.interpol_type = interpol_type; G.interpol_var = interpol_var;
  return RGPU_OK;
}

int rgpu_bind_tree(int ncoarse, int ngridmax, const int* son, const int* father, const int* nbor) {
  if (!G.init) return fail(RGPU_EINVAL, "rgpu_init has not been called");
  if (!son || !father || !nbor) return fail(RGPU_EINVAL, "null tree array");
  if (ncoarse != G.p.nx * G.p.ny * G.p.nz) return fail(RGPU_EINVAL, "ncoarse=%d != nx*ny*nz", ncoarse);
  drop_amr_graph();
  G.ncoarse = ncoarse; G.ngridmax = ngridmax; G.son = son; G.father = father; G.nbor = nbor;
  if (G.amr) {   // mirror the tree (read-only during a step; re-bind after every regrid)
    const long long ncell = (long long)ncoarse + (long long)T_() * ngridmax;
    const bool resized = ncell != G.ncell;
    if (resized) {
      cudaFree(G.d_son_base); cudaFree(G.d_father); cudaFree(G.d_nbor); cudaFree(G.d_uold); cudaFree(G.d_unew); cudaFree(G.d_force);
      G.d_son_base = nullptr; G.d_son = G.d_father = G.d_nbor = nullptr; G.d_uold = G.d_unew = nullptr; G.d_force = nullptr;
      // one leading zero: son(0) = 0 is what a missing neighbour father cell (nbor == 0 at an uncovered box corner) reads
      CUDA_OK(cudaMalloc(&G.d_son_base, sizeof(int) * (ncell + 1)));
      CUDA_OK(cudaMemset(G.d_son_base, 0, sizeof(int)));
      G.d_son = G.d_son_base + 1;
      CUDA_OK(cudaMalloc(&G.d_father, sizeof(int) * ngridmax));
      CUDA_OK(cudaMalloc(&G.d_nbor, sizeof(int) * (size_t)2 * G.p.ndim * ngridmax));
      CUDA_OK(cudaMalloc(&G.d_uold, sizeof(double) * G.nvs * ncell));
      CUDA_OK(cudaMalloc(&G.d_unew, sizeof(double) * G.nvn * ncell));
      CUDA_OK(cudaMemset(G.d_uold, 0, sizeof(double) * G.nvs * ncell));
      CUDA_OK(cudaMemset(G.d_unew, 0, sizeof(double) * G.nvn * ncell));
      if (G.p.poisson) {
        CUDA_OK(cudaMalloc(&G.d_force, sizeof(double) * G.p.ndim * ncell));
        CUDA_OK(cudaMemset(G.d_force, 0, sizeof(double) * G.p.ndim * ncell));
      }
      G.ncell = ncell;
    }
    // on the library's stream: after the kernels that still read the old tree, before the mask kernels below
    CUDA_OK(cudaMemcpyAsync(G.d_son, son, sizeof(int) * ncell, cudaMemcpyHostToDevice, G.stream));
    CUDA_OK(cudaMemcpyAsync(G.d_father, father, sizeof(int) * ngridmax, cudaMemcpyHostToDevice, G.stream));
    CUDA_OK(cudaMemcpyAsync(G.d_nbor, nbor, sizeof(int) * (size_t)2 * G.p.ndim * ngridmax, cudaMemcpyHostToDevice, G.stream));
    // the refined-cell mask of a dense AMR level is son(cell) > 0 of the level's own cells.  refine_fine(l) changes those sons
    // without changing level l's lists, so a level bound before its own refine_fine (the reference order: build_comm(l) runs
    // before refine_fine(l)) or never re-bound (a base level whose octs stay the same) would keep the mask of an older mesh.
    // A level bound against a tree of another size is skipped: its slots may name octs beyond ngridmax; it must be re-bound
    for (int l = 1; l <= MAXLEVEL && !resized; l++) {
      Level& L = G.lev[l];
      if (!G.alev[l].bound || !G.alev[l].dense_sweep || !L.d_refined) continue;
      amr_refined_mask_kernel<<<(unsigned)((L.nslot + 255) / 256), 256, 0, G.stream>>>(G.d_son, L.d_refined, L.d_slot_igrid, L.nslot, G.ncoarse,
                                                                                     G.ngridmax, T_());
      CUDA_OK(cudaGetLastError());
    }
    CUDA_OK(cudaStreamSynchronize(G.stream));
  }
  return RGPU_OK;
}

// Host-only planning of a level: oct positions from the father chain, dense-box detection, slot numbering,
// periodic unwrapping of ghost octs, boundary / reception / emission slot lists.  No CUDA call in here.
static int plan_level(Level& L, int ilevel, int ngrid_active, const int* igrid_active, int ncpu, const int* ngrid_recv,
                    const int* const* igrid_recv, const int* ngrid_emit, const int* const* igrid_emit, int nboundary,
                    const int* boundary_type, const int* ngrid_bound, const int* const* igrid_bound, bool isolated = false) {
  const int nd = G.p.ndim;
  L.dx = level_dx(ilevel);
  // ---- collect every oct of the level with its position -------------------------------------
  struct Rec { int ig; int pos[3]; int kind; int sub; };  // kind 0 active, 1 recv(peer sub), 2 boundary(region sub)
  std::vector<Rec> recs;
  recs.reserve((size_t)ngrid_active + 1024);
  auto add = [&](int ig, int kind, int sub) { Rec r; r.ig = ig; r.kind = kind; r.sub = sub; oct_pos(ilevel, ig, r.pos); recs.push_back(r); };
  for (int i = 0; i < ngrid_active; i++) add(igrid_active[i], 0, 0);
  if (ncpu > 1 && ngrid_recv && igrid_recv)
    for (int c = 0; c < ncpu; c++) if (c != G.myid - 1) for (int i = 0; i < ngrid_recv[c]; i++) add(igrid_recv[c][i], 1, c);
  for (int b = 0; b < nboundary; b++) for (int i = 0; i < ngrid_bound[b]; i++) add(igrid_bound[b][i], 2, b);
  // ---- owned box ------------------------------------------------------------------------------
  int alo[3] = {1 << 30, 1 << 30, 1 << 30}, ahi[3] = {-1, -1, -1};
  for (int i = 0; i < ngrid_active; i++)
    for (int d = 0; d < 3; d++) { alo[d] = std::min(alo[d], recs[i].pos[d]); ahi[d] = std::max(ahi[d], recs[i].pos[d]); }
  long long avol = 1;
  for (int d = 0; d < nd; d++) avol *= (ahi[d] - alo[d] + 1);
  // full extent of the level in octs per dimension (periodic images of ghost octs are unwrapped against it)
  const int ncoarse_d[3] = {G.p.nx, G.p.ny, G.p.nz};
  long long ext[3] = {1, 1, 1};
  for (int d = 0; d < nd; d++) ext[d] = (long long)ncoarse_d[d] << (ilevel - 1);
  // unwrap ghost octs that sit across a periodic boundary so that they become adjacent to the owned box
  for (size_t i = ngrid_active; i < recs.size(); i++)
    for (int d = 0; d < nd; d++) {
      if (recs[i].pos[d] > ahi[d] + 1 && recs[i].pos[d] - ext[d] >= alo[d] - 1) recs[i].pos[d] -= (int)ext[d];
      else if (recs[i].pos[d] < alo[d] - 1 && recs[i].pos[d] + ext[d] <= ahi[d] + 1) recs[i].pos[d] += (int)ext[d];
    }
  int lo[3] = {0, 0, 0}, hi[3] = {0, 0, 0};
  for (int d = 0; d < nd; d++) { lo[d] = alo[d]; hi[d] = ahi[d]; }
  bool in_shell = true;
  for (size_t i = ngrid_active; i < recs.size(); i++)
    for (int d = 0; d < nd; d++) {
      lo[d] = std::min(lo[d], recs[i].pos[d]); hi[d] = std::max(hi[d], recs[i].pos[d]);
      if (recs[i].pos[d] < alo[d] - 1 || recs[i].pos[d] > ahi[d] + 1) in_shell = false;
    }
  if (isolated)   // a refined patch: one layer of (mostly empty) shell slots wherever the box does not span the level
    for (int d = 0; d < nd; d++)
      if (!((long long)(ahi[d] - alo[d] + 1) == ext[d] && alo[d] == 0)) { lo[d] = std::min(lo[d], alo[d] - 1); hi[d] = std::max(hi[d], ahi[d] + 1); }
  L.bound = true;
  L.dense = (avol == ngrid_active) && in_shell;
  if (!L.dense) return RGPU_OK;
  // every dimension must either be periodic over the whole level (no shell) or carry a shell on both sides
  int wrap[3] = {0, 0, 0};
  for (int d = 0; d < nd; d++) {
    const bool shell_lo = lo[d] < alo[d], shell_hi = hi[d] > ahi[d];
    if (!shell_lo && !shell_hi) {
      if ((long long)(ahi[d] - alo[d] + 1) != ext[d] || alo[d] != 0) { L.dense = false; return RGPU_OK; }
      wrap[d] = 1;
    } else if (!(shell_lo && shell_hi)) { L.dense = false; return RGPU_OK; }
  }
  long long nslot = 1;
  int no[3] = {1, 1, 1};
  for (int d = 0; d < nd; d++) { no[d] = hi[d] - lo[d] + 1; nslot *= no[d]; }
  L.nslot = nslot;
  for (int d = 0; d < 3; d++) L.lo[d] = lo[d];
  DenseGeom& g = L.g;
  g.nox = no[0]; g.noy = no[1]; g.noz = no[2];
  g.ncx = 2 * no[0]; g.ncy = nd > 1 ? 2 * no[1] : 1; g.ncz = nd > 2 ? 2 * no[2] : 1;
  g.ox0 = 2 * (alo[0] - lo[0]); g.ox1 = 2 * (ahi[0] - lo[0] + 1);
  g.oy0 = nd > 1 ? 2 * (alo[1] - lo[1]) : 0; g.oy1 = nd > 1 ? 2 * (ahi[1] - lo[1] + 1) : 1;
  g.oz0 = nd > 2 ? 2 * (alo[2] - lo[2]) : 0; g.oz1 = nd > 2 ? 2 * (ahi[2] - lo[2] + 1) : 1;
  g.wrapx = wrap[0]; g.wrapy = wrap[1]; g.wrapz = wrap[2];
  g.nslot = nslot;
  // ---- slot maps ------------------------------------------------------------------------------
  L.slot_igrid.assign((size_t)nslot, 0);
  auto slot_of = [&](const int* pos) {
    long long s = pos[0] - lo[0];
    if (nd > 1) s += (long long)no[0] * (pos[1] - lo[1]);
    if (nd > 2) s += (long long)no[0] * no[1] * (pos[2] - lo[2]);
    return s;
  };
  L.gmin = 1 << 30; L.gmax = 0;
  std::vector<std::vector<int>>& bslots = L.h_bslots; std::vector<std::vector<int>>& rslots = L.h_rslots;
  bslots.assign(nboundary, {}); rslots.assign(ncpu > 1 ? ncpu : 0, {}); L.h_eslots.assign(ncpu > 1 ? ncpu : 0, {});
  L.h_btype.assign(boundary_type, boundary_type + nboundary);
  for (auto& r : recs) {
    const long long s = slot_of(r.pos);
    if (L.slot_igrid[s] != 0) return fail(RGPU_EINVAL, "level %d: two octs (%d,%d) at the same lattice site", ilevel, L.slot_igrid[s], r.ig);
    L.slot_igrid[s] = r.ig;
    L.gmin = std::min(L.gmin, r.ig); L.gmax = std::max(L.gmax, r.ig);
    if (r.kind == 2) bslots[r.sub].push_back((int)s);
    if (r.kind == 1) rslots[r.sub].push_back((int)s);
  }
  // emission octs as slots (the peer's reception list is sorted the same way by construction of build_comm)
  if (ncpu > 1 && ngrid_emit && igrid_emit)
    for (int c = 0; c < ncpu; c++) {
      if (c == G.myid - 1) continue;
      L.h_eslots[c].resize(ngrid_emit[c]);
      for (int i = 0; i < ngrid_emit[c]; i++) {
        int pos[3];
        oct_pos(ilevel, igrid_emit[c][i], pos);
        L.h_eslots[c][i] = (int)slot_of(pos);
      }
    }
  return RGPU_OK;
}

// Level-0 pipeline plan (host only): cut the box into slabs of oct planes along z; per slab the contiguous igrid ranges of
// its octs (upload) and of its active octs (download).  The reference numbers octs in creation order (amr/refine_utils.f90:
// 395-447: chunks of nvector father grids, cell position outermost inside a chunk), which scatters every slab over the whole
// igrid window in runs of ~4 octs -- then the plan is dropped and rgpu_godunov_fine keeps its serial H2D -> sweep -> D2H order.
// A spatially coherent numbering (lattice or Morton / Hilbert order) gives a handful of ranges per slab.
static void plan_slabs(Level& L) {
  L.slabs.clear();
  if (G.p.ndim != 3 || G.p.mhd || G.amr) return;
  const DenseGeom& g = L.g;
  int nsl = 64;   // fill (3 slabs up before the first sweep) + drain (2 slabs down after the last) cost 5/nsl of one direction
  if (const char* e = getenv("RGPU_E2E_SLABS")) nsl = atoi(e);
  nsl = std::min(nsl, g.noz / 4);
  if (nsl < 3) return;
  const size_t max_copies = 24576;   // cudaMemcpy2DAsync calls per direction and call (a few microseconds of host time each)
  const long long plane = (long long)g.nox * g.noy;
  std::vector<Level::Slab> slabs(nsl);
  size_t total = 0;
  std::vector<int> ig;
  // sorted igrids -> runs of consecutive igrids -> blocks of equally long, equally spaced runs (one pitched copy per block and
  // (variable, cell position): the owned octs of an oct plane of a rank's box are such a block in a lattice numbering)
  size_t ncopies = 0;
  auto coalesce = [&](std::vector<int>& v, std::vector<Level::Range>& out) {
    std::sort(v.begin(), v.end());
    std::vector<Level::Range> runs;
    for (size_t i = 0; i < v.size();) {
      size_t j = i + 1;
      while (j < v.size() && v[j] == v[j - 1] + 1) j++;
      runs.push_back({v[i], (int)(j - i), 0, 1});
      i = j;
    }
    for (size_t i = 0; i < runs.size();) {
      size_t j = i + 1;
      int stride = 0;
      if (j < runs.size() && runs[j].n == runs[i].n) {
        stride = runs[j].lo - runs[i].lo;
        while (j < runs.size() && runs[j].n == runs[i].n && runs[j].lo - runs[j - 1].lo == stride) j++;
      }
      const int cnt = (int)(j - i);
      if (cnt >= 3) { out.push_back({runs[i].lo, runs[i].n, stride, cnt}); ncopies += (size_t)G.nvs * T_(); i = j; }
      else { out.push_back(runs[i]); ncopies += (size_t)G.nvs; i++; }
    }
  };
  for (int sl = 0; sl < nsl; sl++) {
    Level::Slab& S = slabs[sl];
    S.oz_a = (int)((long long)g.noz * sl / nsl); S.oz_b = (int)((long long)g.noz * (sl + 1) / nsl);
    ig.clear();
    for (long long t = S.oz_a * plane; t < S.oz_b * plane; t++) if (L.slot_igrid[t] > 0) ig.push_back(L.slot_igrid[t]);
    coalesce(ig, S.up);
    ig.clear();
    for (int oz = S.oz_a; oz < S.oz_b; oz++) {
      if (2 * oz < g.oz0 || 2 * oz >= g.oz1) continue;
      for (int oy = g.oy0 / 2; oy < g.oy1 / 2; oy++)
        for (int ox = g.ox0 / 2; ox < g.ox1 / 2; ox++) {
          const int v = L.slot_igrid[ox + (long long)g.nox * (oy + (long long)g.noy * oz)];
          if (v > 0) ig.push_back(v);
        }
    }
    coalesce(ig, S.down);
    total = ncopies;
    if (total > 2 * max_copies) return;
  }
  L.slabs.swap(slabs);
}

// device side of a dense level store (after plan_level): slot map, state buffers, boundary / peer lists, tiling
static int alloc_dense_store(Level& L, int ncpu, int nboundary, const int* boundary_type) {
  const int nd = G.p.ndim;
  const long long nslot = L.nslot;
  DenseGeom& g = L.g;
  std::vector<std::vector<int>>& bslots = L.h_bslots; std::vector<std::vector<int>>& rslots = L.h_rslots;
  if (nslot >= (1LL << 31)) return fail(RGPU_EUNSUPPORTED, "level too large for 32-bit slots");
  const long long gspan = (long long)L.gmax - L.gmin + 1;
  const size_t np = nplanes_();
  CUDA_OK(cudaMalloc(&L.d_slot_igrid, sizeof(int) * nslot));
  CUDA_OK(cudaMemcpy(L.d_slot_igrid, L.slot_igrid.data(), sizeof(int) * nslot, cudaMemcpyHostToDevice));
  CUDA_OK(cudaMalloc(&L.d_mirror, sizeof(double) * np * gspan));
  CUDA_OK(cudaMalloc(&L.d_u[0], sizeof(double) * np * nslot));
  CUDA_OK(cudaMalloc(&L.d_u[1], sizeof(double) * np * nslot));
  CUDA_OK(cudaMemset(L.d_u[0], 0, sizeof(double) * np * nslot));
  CUDA_OK(cudaMemset(L.d_u[1], 0, sizeof(double) * np * nslot));
  L.f_valid = false;
  if (G.p.poisson) {
    CUDA_OK(cudaMalloc(&L.d_f, sizeof(double) * nd * T_() * nslot));
    CUDA_OK(cudaMemset(L.d_f, 0, sizeof(double) * nd * T_() * nslot));
  }
  if (G.p.pressure_fix) {
    CUDA_OK(cudaMalloc(&L.d_pfix, sizeof(double) * 2 * T_() * nslot));
    CUDA_OK(cudaMemset(L.d_pfix, 0, sizeof(double) * 2 * T_() * nslot));
  }
  L.regions.resize(nboundary);
  for (int b = 0; b < nboundary; b++) {
    L.regions[b].type = boundary_type[b];
    L.regions[b].n = (int)bslots[b].size();
    if (L.regions[b].n) {
      CUDA_OK(cudaMalloc(&L.regions[b].d_slots, sizeof(int) * bslots[b].size()));
      CUDA_OK(cudaMemcpy(L.regions[b].d_slots, bslots[b].data(), sizeof(int) * bslots[b].size(), cudaMemcpyHostToDevice));
    }
  }
  // ---- peers (ghost exchange lists) ----------------------------------------------------------
  // The exchange carries the state only.  pressure_fix's divu / enew need no ghost exchange and no reverse accumulation on a
  // full level: the pdV pass reads the neighbours' uold, and only a coarse-fine face (AMR mode) writes a neighbour's divu / enew.
  if (ncpu > 1) {
    L.peers.resize(ncpu);
    for (int c = 0; c < ncpu; c++) {
      if (c == G.myid - 1) continue;
      PeerList& P = L.peers[c];
      P.nrecv = (int)rslots[c].size();
      if (P.nrecv) {
        CUDA_OK(cudaMalloc(&P.d_recv, sizeof(int) * P.nrecv));
        CUDA_OK(cudaMemcpy(P.d_recv, rslots[c].data(), sizeof(int) * P.nrecv, cudaMemcpyHostToDevice));
        CUDA_OK(cudaMalloc(&P.d_rbuf, sizeof(double) * np * P.nrecv));
      }
      P.nemit = (int)L.h_eslots[c].size();
      if (P.nemit) {
        const std::vector<int>& es = L.h_eslots[c];
        CUDA_OK(cudaMalloc(&P.d_emit, sizeof(int) * P.nemit));
        CUDA_OK(cudaMemcpy(P.d_emit, es.data(), sizeof(int) * P.nemit, cudaMemcpyHostToDevice));
        CUDA_OK(cudaMalloc(&P.d_sbuf, sizeof(double) * np * P.nemit));
      }
    }
  }
  if (ncpu > 1) {   // fused forward exchange lists
    std::vector<int> eall, rall;
    L.emit_off.assign(1, 0); L.recv_off.assign(1, 0);
    for (int c = 0; c < ncpu; c++) {
      if (c != G.myid - 1) {
        eall.insert(eall.end(), L.h_eslots[c].begin(), L.h_eslots[c].end());
        rall.insert(rall.end(), rslots[c].begin(), rslots[c].end());
      }
      L.emit_off.push_back((long long)eall.size()); L.recv_off.push_back((long long)rall.size());
    }
    if (!eall.empty()) {
      CUDA_OK(cudaMalloc(&L.d_emit_all, sizeof(int) * eall.size()));
      CUDA_OK(cudaMemcpy(L.d_emit_all, eall.data(), sizeof(int) * eall.size(), cudaMemcpyHostToDevice));
      CUDA_OK(cudaMalloc(&L.d_sbuf_all, sizeof(double) * np * eall.size()));
    }
    if (!rall.empty()) {
      CUDA_OK(cudaMalloc(&L.d_recv_all, sizeof(int) * rall.size()));
      CUDA_OK(cudaMemcpy(L.d_recv_all, rall.data(), sizeof(int) * rall.size(), cudaMemcpyHostToDevice));
      CUDA_OK(cudaMalloc(&L.d_rbuf_all, sizeof(double) * np * rall.size()));
    }
    CUDA_OK(cudaMalloc(&L.d_emit_off, sizeof(long long) * (ncpu + 1)));
    CUDA_OK(cudaMalloc(&L.d_recv_off, sizeof(long long) * (ncpu + 1)));
    CUDA_OK(cudaMemcpy(L.d_emit_off, L.emit_off.data(), sizeof(long long) * (ncpu + 1), cudaMemcpyHostToDevice));
    CUDA_OK(cudaMemcpy(L.d_recv_off, L.recv_off.data(), sizeof(long long) * (ncpu + 1), cudaMemcpyHostToDevice));
    CUDA_OK(cudaEventCreateWithFlags(&L.ev_x, cudaEventDisableTiming));
    CUDA_OK(cudaEventCreateWithFlags(&L.ev_s, cudaEventDisableTiming));
  }
  // ---- tile decomposition of the owned range ----------------------------------------------------
  const int bx = 32;
  int by = tile_by_default(nd, G.p.riemann);
  // poisson, pressure_fix: the GRAV / PFIX instantiations exist for the default tile height of the round-1 kernel only (variant 0,
  // FAST ignored)
  if (nd == 3 && !G.p.poisson && !G.p.pressure_fix) { const char* e = getenv("RGPU_BY3"); if (e) { const int v = atoi(e); if (v == 8 || v == 12 || v == 16) by = v; } }
  int minb = 1;
  L.variant = 0;
  if (nd == 3 && !G.p.mhd && !G.amr && !G.p.poisson && !G.p.pressure_fix) {   // plain dense 3-D sweep: round-2 kernel; RGPU_SWEEP=old|<variant> for tuning runs
    // the two-barrier loop (sweep3_kernel, three scalar branch-free solves); profiles/tune_sweep.py times the variants
    L.variant = SWEEP3_DEFAULT_VARIANT;
    const char* e = getenv("RGPU_SWEEP");
    if (e) L.variant = (strcmp(e, "old") == 0) ? 0 : atoi(e);
    if ((long long)G.nvs * T_() * nslot >= (1LL << 32)) L.variant = 0;   // sweep3_kernel addresses the state with 32-bit element indices
    if (L.variant) { by = sweep3_by_of(L.variant); minb = (L.variant / 10) % 10; if (minb < 1 || minb == 9 || L.variant >= 40000) minb = 1; }
  }
  L.by = by;
  const int txo = bx - 2, tyo = nd > 1 ? by - 2 : 1;
  L.ntx = (g.ox1 - g.ox0 + txo - 1) / txo;
  L.nty = nd > 1 ? (g.oy1 - g.oy0 + tyo - 1) / tyo : 1;
  // persistent kernel: one CTA per SM, equal contiguous shares of the (column tile, z plane) space
  L.nwork = (long long)L.ntx * L.nty * (nd > 2 ? (g.oz1 - g.oz0) : 1);
  L.nblocks = (int)std::min<long long>((long long)G.nsm * minb, L.nwork);
  L.part_cap = std::max(2 * L.nblocks, reduce_blocks());
  // ---- interior / frame split (multi-rank 3-D hydro): a tile is interior when every cell it reads (2-cell halo) is owned
  L.overlap = false;
  if (nd == 3 && !G.p.mhd && !G.amr && ncpu > 1) {
    const char* e = getenv("RGPU_OVERLAP");
    if (const char* r = getenv("RGPU_OVERLAP_RESERVE")) L.reserve_sms = std::max(0, atoi(r));
    SweepWork wi{};
    wi.mode = 1;
    auto range = [](int n_owned, int tile, int ntile, int wrap, int& i0, int& i1) {
      if (wrap) { i0 = 0; i1 = ntile; return; }
      i0 = 1; i1 = n_owned >= tile + 2 + tile ? (n_owned - (tile + 2)) / tile + 1 : 0;
      if (i1 > ntile) i1 = ntile;
    };
    range(g.ox1 - g.ox0, txo, L.ntx, g.wrapx, wi.ix0, wi.ix1);
    range(g.oy1 - g.oy0, tyo, L.nty, g.wrapy, wi.iy0, wi.iy1);
    wi.iz0 = g.wrapz ? g.oz0 : g.oz0 + 2; wi.iz1 = g.wrapz ? g.oz1 : g.oz1 - 2;
    const long long nxi = wi.ix1 - wi.ix0, nyi = wi.iy1 - wi.iy0, nzi = wi.iz1 - wi.iz0;
    // at large sizes per rank the exchange is a small share of the step, and a NCCL kernel that becomes resident on one rank
    // before the persistent interior CTAs (and then spins for its peer) can cost more than the overlap gains -- default: overlap
    // only below 100 M owned cells (RGPU_OVERLAP=1 forces it; not re-measured on H100, profiles/mgpu_overlap_probe.py)
    const long long nown = (long long)(g.ox1 - g.ox0) * (g.oy1 - g.oy0) * (g.oz1 - g.oz0);
    const bool want = e ? atoi(e) != 0 : nown <= 100000000LL;
    if (want && nxi > 0 && nyi > 0 && nzi > 4) {
      L.wk_int = wi; L.wk_frame = wi; L.wk_frame.mode = 2;
      L.nwork_int = nxi * nyi * nzi;
      L.nwork_frame = ((long long)L.ntx * L.nty - nxi * nyi) * (g.oz1 - g.oz0) + nxi * nyi * ((wi.iz0 - g.oz0) + (g.oz1 - wi.iz1));
      L.overlap = L.nwork_frame > 0;
    }
  }
  if (G.p.mhd) {
    L.mhd_nb = reduce_blocks();
    L.nblocks = L.mhd_nb;   // CTAs that write Courant partials in the sweep
    L.part_cap = std::max(L.part_cap, L.mhd_nb);
    CUDA_OK(cudaMalloc(&L.d_mhdw, sizeof(double) * (size_t)MW_NCOMP * (size_t)g.ncx * g.ncy * g.ncz));
  }
  CUDA_OK(cudaMalloc(&L.d_part, sizeof(double) * 5 * L.part_cap));
  CUDA_OK(cudaMalloc(&L.d_dt, sizeof(double)));
  CUDA_OK(cudaMalloc(&L.d_out, sizeof(double) * 5));
  L.cur = 0; L.unew_valid = false;
  plan_slabs(L);
  for (size_t i = 0; i < L.slabs.size(); i++) {
    cudaEvent_t e1, e2;
    CUDA_OK(cudaEventCreateWithFlags(&e1, cudaEventDisableTiming));
    CUDA_OK(cudaEventCreateWithFlags(&e2, cudaEventDisableTiming));
    L.ev_in.push_back(e1); L.ev_c.push_back(e2);
  }
  return RGPU_OK;
}

int rgpu_bind_level(int ilevel, int ngrid_active, const int* igrid_active, int ncpu, const int* ngrid_recv,
                    const int* const* igrid_recv, const int* ngrid_emit, const int* const* igrid_emit, int nboundary,
                    const int* boundary_type, const int* ngrid_bound, const int* const* igrid_bound) {
  if (!G.init) return fail(RGPU_EINVAL, "rgpu_init has not been called");
  if (!G.son) return fail(RGPU_EINVAL, "rgpu_bind_tree has not been called");
  if (ilevel < 1 || ilevel > MAXLEVEL) return fail(RGPU_EINVAL, "ilevel %d out of range", ilevel);
  if (!G.amr && (ngrid_active <= 0 || !igrid_active)) return fail(RGPU_EINVAL, "level %d has no active oct", ilevel);
  if (G.amr) {
    int rc = amr_bind_level(ilevel, ngrid_active, igrid_active, ncpu, ngrid_recv, igrid_recv, ngrid_emit, igrid_emit, nboundary, boundary_type, ngrid_bound, igrid_bound);
    if (rc) return rc;
    if (G.p.mhd) return mhd_amr_bind_extra(G.alev[ilevel], ilevel, ngrid_active, igrid_active);
    // A level that is a complete Cartesian box and sends no refluxes to a coarser level (the fully refined base of the
    // run) is swept by the dense kernel: ~10x the throughput of the oct-batch kernel.  RGPU_AMR_DENSE=0 disables.
    AmrLevel& A = G.alev[ilevel];
    Level& L = G.lev[ilevel];
    if (L.bound) free_level(L);
    const char* env = getenv("RGPU_AMR_DENSE");
    const char* envp = getenv("RGPU_AMR_PATCH");
    // poisson: GRAV variant; pressure_fix: PFIX variant (both: GRAV+PFIX)
    const bool eligible = !(env && atoi(env) == 0) && G.p.ndim == 3 && !G.p.mhd && !(G.p.difmag > 0.0) && G.p.nvar == G.p.ndim + 2 &&
                          ngrid_active > 0;
    const bool base = eligible && A.nent == 0 && ncpu == 1;   // multi-rank AMR keeps the oct-batch kernel (tested path)
    // a refined level whose octs form a Cartesian box (nested / zoom refinement): dense kernel on the box + a prolongated
    // ghost shell; the octs at its surface go through the oct-batch kernel once more for the refluxed faces only
    const bool patch = eligible && A.nent > 0 && ncpu == 1 && nboundary == 0 && !(envp && atoi(envp) == 0);
    if (base || patch) {
      rc = plan_level(L, ilevel, ngrid_active, igrid_active, ncpu, ngrid_recv, igrid_recv, ngrid_emit, igrid_emit, nboundary,
                      boundary_type, ngrid_bound, igrid_bound, patch);
      if (rc == RGPU_OK && L.dense && L.nslot < (1LL << 31)) {
        rc = alloc_dense_store(L, ncpu, nboundary, boundary_type);
        if (rc) return rc;
        CUDA_OK(cudaMalloc(&L.d_refined, (size_t)T_() * L.nslot));
        amr_refined_mask_kernel<<<(unsigned)((L.nslot + 255) / 256), 256, 0, G.stream>>>(G.d_son, L.d_refined, L.d_slot_igrid, L.nslot, G.ncoarse,
                                                                                       G.ngridmax, T_());
        CUDA_OK(cudaGetLastError());
        if (patch) {
          std::vector<int> slot_of((size_t)G.ngridmax + 1, -1);
          for (long long s = 0; s < L.nslot; s++) if (L.slot_igrid[s] > 0) slot_of[L.slot_igrid[s]] = (int)s;
          std::vector<int> act_slot(ngrid_active), surf_ig(A.h_surf_io.size());
          for (int i = 0; i < ngrid_active; i++) act_slot[i] = slot_of[igrid_active[i]];
          for (size_t i = 0; i < A.h_surf_io.size(); i++) surf_ig[i] = igrid_active[A.h_surf_io[i]];
          A.nsurf = (int)A.h_surf_io.size();
          CUDA_OK(cudaMalloc(&A.d_act_slot, sizeof(int) * ngrid_active));
          CUDA_OK(cudaMemcpy(A.d_act_slot, act_slot.data(), sizeof(int) * ngrid_active, cudaMemcpyHostToDevice));
          CUDA_OK(cudaMalloc(&A.d_shell_father, sizeof(int) * L.nslot));
          CUDA_OK(cudaMemset(A.d_shell_father, 0, sizeof(int) * L.nslot));
          if (A.nsurf > 0) {
            CUDA_OK(cudaMalloc(&A.d_surf_igrid, sizeof(int) * A.nsurf));
            CUDA_OK(cudaMalloc(&A.d_surf_io, sizeof(int) * A.nsurf));
            CUDA_OK(cudaMemcpy(A.d_surf_igrid, surf_ig.data(), sizeof(int) * A.nsurf, cudaMemcpyHostToDevice));
            CUDA_OK(cudaMemcpy(A.d_surf_io, A.h_surf_io.data(), sizeof(int) * A.nsurf, cudaMemcpyHostToDevice));
          }
          amr_shell_father_kernel<<<(ngrid_active + 127) / 128, 128, 0, G.stream>>>(amr_tree(), A.d_active, A.d_act_slot, ngrid_active, ilevel, L.g.nox,
                                                                                L.g.noy, L.nslot, A.d_shell_father);
          CUDA_OK(cudaGetLastError());
          A.patch = true;
        }
        A.dense_sweep = true;
      } else {
        L = Level();   // not a box: the oct-batch kernel runs the level
      }
    }
    return RGPU_OK;
  }
  if (G.p.mhd && G.p.ndim != 3)
    return fail(RGPU_EUNSUPPORTED, "MHD build, NDIM=%d: built in AMR mode only -- call rgpu_set_amr(1, interpol_type, 0) after rgpu_init", G.p.ndim);
  // poisson and pressure_fix run through the dense sweep's GRAV / PFIX instantiations (rgpu_init admits them for nvar = ndim+2,
  // difmag = 0 only); both together have no plain form
  if (G.p.difmag > 0.0 || (!G.p.mhd && G.p.nvar != G.p.ndim + 2) || (G.p.pressure_fix && G.p.poisson))
    return fail(RGPU_EUNSUPPORTED, "difmag>0 (cmpdivu/consup), passive scalars (nvar>ndim+2) and pressure_fix together with poisson are "
                                   "built in AMR mode only: call rgpu_set_amr(1, interpol_type, 0) after rgpu_init (works for "
                                   "levelmin=levelmax runs too)");
  Level& L = G.lev[ilevel];
  if (L.bound) free_level(L);
  {
    const int rc = plan_level(L, ilevel, ngrid_active, igrid_active, ncpu, ngrid_recv, igrid_recv, ngrid_emit, igrid_emit, nboundary,
                              boundary_type, ngrid_bound, igrid_bound);
    if (rc) return rc;
  }
  if (!L.dense) return RGPU_OK;   // bound, but only the AMR path could run it
  if (G.p.pressure_fix) {
    // add_pdv_source_terms reads the face neighbours of every owned cell.  plan_level admits a shell with holes (it only bounds
    // the shell's extent); where a face-neighbour oct is missing the reference would read the father cell 1.5 dx away, which a
    // dense level does not hold: refuse such a level
    const DenseGeom& g = L.g;
    const int nd = G.p.ndim, wrap[3] = {g.wrapx, g.wrapy, g.wrapz};
    const int o0[3] = {g.ox0 / 2, g.oy0 / 2, g.oz0 / 2}, o1[3] = {g.ox1 / 2, nd > 1 ? g.oy1 / 2 : 1, nd > 2 ? g.oz1 / 2 : 1};
    const long long str[3] = {1, g.nox, (long long)g.nox * g.noy};
    for (int oz = o0[2]; oz < o1[2]; oz++)
      for (int oy = o0[1]; oy < o1[1]; oy++)
        for (int ox = o0[0]; ox < o1[0]; ox++) {
          const long long s0 = ox + str[1] * oy + str[2] * oz;
          for (int d = 0; d < nd; d++)
            for (int side = -1; side <= 1; side += 2)
              if (!wrap[d] && L.slot_igrid[s0 + side * str[d]] <= 0) {
                L = Level();
                return fail(RGPU_EUNSUPPORTED, "pressure_fix: an active oct of level %d has no neighbour oct across its %s face along "
                                               "dimension %d (outside AMR mode every face neighbour must be bound)", ilevel,
                            side < 0 ? "lower" : "upper", d + 1);
              }
        }
  }
  return alloc_dense_store(L, ncpu, nboundary, boundary_type);
}

// Host-only entry point: the level plan (dense-box geometry and slot numbering) without touching CUDA.
// Used by the CPU test-suite and for dry runs of a new mesh; needs no rgpu_init.
int rgpu_plan_level(const rgpu_params* p, int myid, int ncoarse, int ngridmax, const int* father, int ilevel, int ngrid_active, const int* igrid_active, int ncpu, const int* ngrid_recv,
                    const int* const* igrid_recv, const int* ngrid_emit, const int* const* igrid_emit, int nboundary,
                    const int* boundary_type, const int* ngrid_bound, const int* const* igrid_bound,
                    rgpu_level_info* info, int* slot_igrid_out, long long slot_cap) {
  if (!p || !father || !info) return fail(RGPU_EINVAL, "null argument");
  if (G.init) return fail(RGPU_EINVAL, "rgpu_plan_level is a dry-run entry point: call it before rgpu_init or after rgpu_finalize");
  G.p = *p; G.myid = myid; G.ncoarse = ncoarse; G.ngridmax = ngridmax; G.father = father;
  G.nvs = p->mhd ? p->nvar + 3 : p->nvar;
  Level L;
  const int rc = plan_level(L, ilevel, ngrid_active, igrid_active, ncpu, ngrid_recv, igrid_recv, ngrid_emit, igrid_emit, nboundary,
                            boundary_type, ngrid_bound, igrid_bound);
  G.father = nullptr;
  if (rc) return rc;
  memset(info, 0, sizeof(*info));
  info->dense = L.dense;
  if (L.dense) {
    info->ncell_box[0] = L.g.ncx; info->ncell_box[1] = L.g.ncy; info->ncell_box[2] = L.g.ncz;
    info->own_lo[0] = L.g.ox0; info->own_lo[1] = L.g.oy0; info->own_lo[2] = L.g.oz0;
    info->own_hi[0] = L.g.ox1; info->own_hi[1] = L.g.oy1; info->own_hi[2] = L.g.oz1;
    info->wrap[0] = L.g.wrapx; info->wrap[1] = L.g.wrapy; info->wrap[2] = L.g.wrapz;
    info->nslot = L.nslot;
    plan_slabs(L);                       // Level-0 pipeline plan (host only): 0 slabs = serial order
    info->pipeline_slabs = (int)L.slabs.size();
    if (slot_igrid_out) {
      if (slot_cap < L.nslot) return fail(RGPU_EINVAL, "slot_igrid_out too small (%lld < %lld)", slot_cap, L.nslot);
      memcpy(slot_igrid_out, L.slot_igrid.data(), sizeof(int) * L.nslot);
    }
  }
  return RGPU_OK;
}

int rgpu_host_register(void* ptr, size_t bytes) {
  if (!G.init) return fail(RGPU_EINVAL, "rgpu_init has not been called");
  CUDA_OK(cudaHostRegister(ptr, bytes, cudaHostRegisterPortable));
  return RGPU_OK;
}
int rgpu_host_unregister(void* ptr) {
  CUDA_OK(cudaHostUnregister(ptr));
  return RGPU_OK;
}

// host array [nv][ncell] (nv < 0: the G.nvs state variables) -> level store
static int upload_into(Level& L, const double* host, double* dst, int nv = -1) {
  const int T = T_();
  const long long gspan = (long long)L.gmax - L.gmin + 1;
  const size_t ncell = (size_t)G.ncoarse + (size_t)T * G.ngridmax;
  if (nv < 0) nv = G.nvs;
  for (int iv = 0; iv < nv; iv++)
    for (int ind = 0; ind < T; ind++) {
      const double* src = host + (size_t)iv * ncell + G.ncoarse + (size_t)ind * G.ngridmax + (L.gmin - 1);
      CUDA_OK(cudaMemcpyAsync(L.d_mirror + ((size_t)iv * T + ind) * gspan, src, sizeof(double) * gspan, cudaMemcpyHostToDevice, G.stream));
    }
  const int nthr = 256;
  gather_slots_kernel<<<(unsigned)((L.nslot + nthr - 1) / nthr), nthr, 0, G.stream>>>(L.d_mirror, dst, L.d_slot_igrid, L.nslot, L.gmin, gspan, nv * T);
  CUDA_OK(cudaGetLastError());
  L.launches++;
  return RGPU_OK;
}
// device level store -> host array.  owned_only: write back the active octs only (unew of godunov_fine);
// the mirror window is pre-loaded from the host whenever it also covers octs that must keep the host's values.
static int download_from(Level& L, double* host, const double* srcdev, bool owned_only) {
  const int T = T_();
  const long long gspan = (long long)L.gmax - L.gmin + 1;
  const size_t ncell = (size_t)G.ncoarse + (size_t)T * G.ngridmax;
  long long nown = (L.g.ox1 - L.g.ox0) / 2;
  if (G.p.ndim > 1) nown *= (L.g.oy1 - L.g.oy0) / 2;
  if (G.p.ndim > 2) nown *= (L.g.oz1 - L.g.oz0) / 2;
  const bool preload = (gspan != L.nslot) || (owned_only && nown != L.nslot);
  if (preload)
    for (int iv = 0; iv < G.nvs; iv++)
      for (int ind = 0; ind < T; ind++) {
        const double* src = host + (size_t)iv * ncell + G.ncoarse + (size_t)ind * G.ngridmax + (L.gmin - 1);
        CUDA_OK(cudaMemcpyAsync(L.d_mirror + ((size_t)iv * T + ind) * gspan, src, sizeof(double) * gspan, cudaMemcpyHostToDevice, G.stream));
      }
  const int nthr = 256;
  scatter_slots_kernel<<<(unsigned)((L.nslot + nthr - 1) / nthr), nthr, 0, G.stream>>>(L.d_mirror, srcdev, L.d_slot_igrid, L.nslot, L.gmin, gspan,
                                                                                  (int)nplanes_(), owned_only ? 1 : 0, L.g);
  CUDA_OK(cudaGetLastError());
  L.launches++;
  for (int iv = 0; iv < G.nvs; iv++)
    for (int ind = 0; ind < T; ind++) {
      double* dst = host + (size_t)iv * ncell + G.ncoarse + (size_t)ind * G.ngridmax + (L.gmin - 1);
      CUDA_OK(cudaMemcpyAsync(dst, L.d_mirror + ((size_t)iv * T + ind) * gspan, sizeof(double) * gspan, cudaMemcpyDeviceToHost, G.stream));
    }
  CUDA_OK(cudaStreamSynchronize(G.stream));
  return RGPU_OK;
}

// Level-0 call as a three-stream pipeline over z-slabs (plan_slabs): H2D of slab s+1 (stream s_in) runs while slab s is gathered
// into lattice slots, swept and scattered back (G.stream) and slab s-1 travels back to the host (s_out) -- PCIe is full duplex, so
// the call costs about one direction of the link instead of two plus the sweep.  The sweep of a slab needs one oct layer of its
// two neighbours: slabs are uploaded in the order N-1, 0, 1, ..., N-2 (the periodic wrap makes slab N-1 the lower neighbour of
// slab 0) and slab s is swept once slab s+1 has been gathered.  Same kernels, same arithmetic as the serial path; the result is
// bit-identical (tests/test_gpu_parity.py::test_level0_pipelined_equals_serial).
static int godunov_fine_pipelined(Level& L, const double* uold, double* unew) {
  const int T = T_(), nsl = (int)L.slabs.size();
  const long long gspan = (long long)L.gmax - L.gmin + 1;
  const size_t ncell = (size_t)G.ncoarse + (size_t)T * G.ngridmax;
  const long long plane = (long long)L.g.nox * L.g.noy;
  const int nthr = 256;
  double* uin = L.d_u[L.cur];
  double* uout = L.d_u[1 - L.cur];
  // the copy streams must not start before the work already queued on the main stream (previous call, dt upload)
  CUDA_OK(cudaEventRecord(G.ev_pipe, G.stream));
  CUDA_OK(cudaStreamWaitEvent(G.s_in, G.ev_pipe, 0));
  CUDA_OK(cudaStreamWaitEvent(G.s_out, G.ev_pipe, 0));
  auto h2d = [&](int sl) -> int {
    for (const auto& r : L.slabs[sl].up)
      for (int iv = 0; iv < G.nvs; iv++) {
        if (r.count == 1) {   // one run: the 2^ndim cell positions are the rows of one pitched copy
          CUDA_OK(cudaMemcpy2DAsync(L.d_mirror + (size_t)iv * T * gspan + (r.lo - L.gmin), sizeof(double) * gspan,
                                    uold + (size_t)iv * ncell + G.ncoarse + (r.lo - 1), sizeof(double) * G.ngridmax,
                                    sizeof(double) * r.n, T, cudaMemcpyHostToDevice, G.s_in));
        } else {              // a block of equally spaced runs: the runs are the rows, one copy per cell position
          for (int ind = 0; ind < T; ind++)
            CUDA_OK(cudaMemcpy2DAsync(L.d_mirror + ((size_t)iv * T + ind) * gspan + (r.lo - L.gmin), sizeof(double) * r.stride,
                                      uold + (size_t)iv * ncell + G.ncoarse + (size_t)ind * G.ngridmax + (r.lo - 1), sizeof(double) * r.stride,
                                      sizeof(double) * r.n, r.count, cudaMemcpyHostToDevice, G.s_in));
        }
      }
    CUDA_OK(cudaEventRecord(L.ev_in[sl], G.s_in));
    return RGPU_OK;
  };
  auto gather = [&](int sl) -> int {
    CUDA_OK(cudaStreamWaitEvent(G.stream, L.ev_in[sl], 0));
    const long long s0 = L.slabs[sl].oz_a * plane, s1 = L.slabs[sl].oz_b * plane;
    gather_slots_kernel<<<(unsigned)((s1 - s0 + nthr - 1) / nthr), nthr, 0, G.stream>>>(L.d_mirror, uin, L.d_slot_igrid, L.nslot, L.gmin, gspan,
                                                                                      (int)nplanes_(), s0, s1);
    CUDA_OK(cudaGetLastError());
    L.launches++;
    return RGPU_OK;
  };
  auto sweep_out = [&](int sl) -> int {
    int rc = launch_sweep(L, 2 * L.slabs[sl].oz_a, 2 * L.slabs[sl].oz_b); if (rc) return rc;
    const long long s0 = L.slabs[sl].oz_a * plane, s1 = L.slabs[sl].oz_b * plane;
    scatter_slots_kernel<<<(unsigned)((s1 - s0 + nthr - 1) / nthr), nthr, 0, G.stream>>>(L.d_mirror, uout, L.d_slot_igrid, L.nslot, L.gmin, gspan,
                                                                                       (int)nplanes_(), 1, L.g, s0, s1);
    CUDA_OK(cudaGetLastError());
    L.launches++;
    CUDA_OK(cudaEventRecord(L.ev_c[sl], G.stream));
    CUDA_OK(cudaStreamWaitEvent(G.s_out, L.ev_c[sl], 0));
    for (const auto& r : L.slabs[sl].down)
      for (int iv = 0; iv < G.nvs; iv++) {
        if (r.count == 1) {
          CUDA_OK(cudaMemcpy2DAsync(unew + (size_t)iv * ncell + G.ncoarse + (r.lo - 1), sizeof(double) * G.ngridmax,
                                    L.d_mirror + (size_t)iv * T * gspan + (r.lo - L.gmin), sizeof(double) * gspan,
                                    sizeof(double) * r.n, T, cudaMemcpyDeviceToHost, G.s_out));
        } else {
          for (int ind = 0; ind < T; ind++)
            CUDA_OK(cudaMemcpy2DAsync(unew + (size_t)iv * ncell + G.ncoarse + (size_t)ind * G.ngridmax + (r.lo - 1), sizeof(double) * r.stride,
                                      L.d_mirror + ((size_t)iv * T + ind) * gspan + (r.lo - L.gmin), sizeof(double) * r.stride,
                                      sizeof(double) * r.n, r.count, cudaMemcpyDeviceToHost, G.s_out));
        }
      }
    return RGPU_OK;
  };
  int rc;
  rc = h2d(nsl - 1); if (rc) return rc;
  for (int sl = 0; sl < nsl - 1; sl++) { rc = h2d(sl); if (rc) return rc; }
  rc = gather(nsl - 1); if (rc) return rc;
  rc = gather(0); if (rc) return rc;
  for (int sl = 0; sl < nsl; sl++) {
    if (sl + 1 < nsl - 1) { rc = gather(sl + 1); if (rc) return rc; }
    rc = sweep_out(sl); if (rc) return rc;
  }
  L.unew_valid = true;
  CUDA_OK(cudaStreamSynchronize(G.s_out));
  CUDA_OK(cudaStreamSynchronize(G.stream));
  return RGPU_OK;
}

int rgpu_upload_state(int ilevel, const double* uold) {
  if (G.amr) {   // AMR mode: the whole uold array (all levels) is mirrored; ilevel is ignored
    if (!G.d_uold || !uold) return fail(RGPU_EINVAL, "AMR mode: bind the tree first / null uold");
    CUDA_OK(cudaMemcpyAsync(G.d_uold, uold, sizeof(double) * G.nvs * G.ncell, cudaMemcpyHostToDevice, G.stream));
    CUDA_OK(cudaStreamSynchronize(G.stream));
    return RGPU_OK;
  }
  Level* L; int rc = check_level(ilevel, &L); if (rc) return rc;
  if (!uold) return fail(RGPU_EINVAL, "null uold");
  rc = upload_into(*L, uold, L->d_u[L->cur]); if (rc) return rc;
  L->unew_valid = false;
  L->pfix_ready = false;
  return RGPU_OK;
}
int rgpu_download_state(int ilevel, double* uold) {
  if (G.amr) {
    if (!G.d_uold || !uold) return fail(RGPU_EINVAL, "AMR mode: bind the tree first / null uold");
    CUDA_OK(cudaMemcpyAsync(uold, G.d_uold, sizeof(double) * G.nvs * G.ncell, cudaMemcpyDeviceToHost, G.stream));
    CUDA_OK(cudaStreamSynchronize(G.stream));
    return RGPU_OK;
  }
  Level* L; int rc = check_level(ilevel, &L); if (rc) return rc;
  if (!uold) return fail(RGPU_EINVAL, "null uold");
  return download_from(*L, uold, L->d_u[L->cur], false);
}

int rgpu_set_unew(int ilevel) {
  if (G.amr) { AmrLevel* A; int rc = check_amr_level(ilevel, &A); if (rc) return rc; return amr_set_unew(*A); }
  Level* L; int rc = check_level(ilevel, &L); if (rc) return rc;
  const size_t n = nplanes_() * (size_t)L->nslot;
  copy_state_kernel<<<(unsigned)((n + 255) / 256), 256, 0, G.stream>>>(L->d_u[L->cur], L->d_u[1 - L->cur], n);
  CUDA_OK(cudaGetLastError());
  L->launches++;
  for (auto& P : L->peers)
    if (P.nrecv) {   // unew = 0 in the reception octs (godunov_fine.f90:93-100)
      zero_octs_kernel<<<(P.nrecv + 127) / 128, 128, 0, G.stream>>>(L->d_u[1 - L->cur], P.d_recv, P.nrecv, L->nslot, (int)nplanes_());
      CUDA_OK(cudaGetLastError());
      L->launches++;
    }
  if (G.p.pressure_fix) {   // divu = 0, enew = e_int of uold on the owned cells (godunov_fine.f90:71-90)
    rc = launch_pfix_pass(*L, PFIX_INIT, 0.0, nullptr); if (rc) return rc;
    L->pfix_ready = true;
  }
  L->unew_valid = true;
  return RGPU_OK;
}

int rgpu_godunov_fine_dev(int ilevel, double dt) {
  if (G.amr) {
    AmrLevel* A; int rc = check_amr_level(ilevel, &A); if (rc) return rc;
    if (!(dt > 0)) return fail(RGPU_EINVAL, "dt=%g", dt);
    return amr_godunov(*A, ilevel, dt);
  }
  Level* L; int rc = check_level(ilevel, &L); if (rc) return rc;
  if (!(dt > 0)) return fail(RGPU_EINVAL, "dt=%g", dt);
  // pressure_fix: the sweep accumulates into divu / enew, so they must hold set_unew's values -- never a previous sweep's
  if (G.p.pressure_fix && !L->pfix_ready) return fail(RGPU_EINVAL, "pressure_fix: rgpu_set_unew has not initialised divu / enew since the last sweep");
  // dt travels by value in the launch arguments (hydro kernels): no copy, no host synchronisation per call.  The MHD passes
  // read it from device memory: asynchronous copy from a buffer that outlives the call
  if (G.p.mhd) {
    L->dt_stage = dt;
    CUDA_OK(cudaMemcpyAsync(L->d_dt, &L->dt_stage, sizeof(double), cudaMemcpyHostToDevice, G.stream));
    CUDA_OK(cudaStreamSynchronize(G.stream));
  } else {
    L->dt_by_value = dt;
  }
  // the fused kernel evaluates unew = uold + dF for the owned cells (== set_unew followed by the flux update)
  rc = launch_sweep(*L);
  L->dt_by_value = 0.0;
  if (rc) return rc;
  L->unew_valid = true;
  L->pfix_ready = false;
  L->dt_last = dt;
  return RGPU_OK;
}

int rgpu_set_uold(int ilevel) {
  if (G.amr) {
    AmrLevel* A; int rc = check_amr_level(ilevel, &A); if (rc) return rc;
    return amr_set_uold(*A, ilevel, nullptr);
  }
  Level* L; int rc = check_level(ilevel, &L); if (rc) return rc;
  if (!L->unew_valid) return fail(RGPU_EINVAL, "set_uold before set_unew/godunov_fine");
  if (G.p.poisson) {   // add_gravity_source_terms on the owned cells of unew (godunov_fine.f90:159-161)
    if (!(L->dt_last > 0)) return fail(RGPU_EINVAL, "set_uold with poisson before godunov_fine (dtnew(ilevel) unknown)");
    rc = need_force(*L); if (rc) return rc;
    long long n = L->g.ox1 - L->g.ox0;
    if (G.p.ndim > 1) n *= L->g.oy1 - L->g.oy0;
    if (G.p.ndim > 2) n *= L->g.oz1 - L->g.oz0;
    const unsigned nb = (unsigned)((n + 127) / 128);
    const double* uo = L->d_u[L->cur];
    double* un = L->d_u[1 - L->cur];
    if (G.p.ndim == 1) dense_gravity_src_kernel<1><<<nb, 128, 0, G.stream>>>(uo, un, L->d_f, L->g, G.p.smallr, L->dt_last);
    else if (G.p.ndim == 2) dense_gravity_src_kernel<2><<<nb, 128, 0, G.stream>>>(uo, un, L->d_f, L->g, G.p.smallr, L->dt_last);
    else dense_gravity_src_kernel<3><<<nb, 128, 0, G.stream>>>(uo, un, L->d_f, L->g, G.p.smallr, L->dt_last);
    CUDA_OK(cudaGetLastError());
    L->launches++;
  }
  if (G.p.pressure_fix) {   // add_pdv_source_terms on enew from uold (godunov_fine.f90:164-168)
    if (!(L->dt_last > 0)) return fail(RGPU_EINVAL, "set_uold with pressure_fix before godunov_fine (dtnew(ilevel) unknown)");
    rc = launch_pfix_pass(*L, PFIX_PDV, L->dt_last, nullptr); if (rc) return rc;
  }
  // uold <- unew on the active cells (godunov_fine.f90:193-197); shells keep their uold values
  rc = carry_shells(*L, L->d_u[L->cur], L->d_u[1 - L->cur]); if (rc) return rc;
  L->cur = 1 - L->cur;
  L->unew_valid = false;
  L->pfix_ready = false;
  if (G.p.pressure_fix) { rc = launch_pfix_pass(*L, PFIX_SWITCH, L->dt_last, nullptr); if (rc) return rc; }   // :203-227
  return RGPU_OK;
}

int rgpu_courant_fine(int ilevel, double* dt_io, double sums[3]) {
  if (G.amr) {
    AmrLevel* A; int rc = check_amr_level(ilevel, &A); if (rc) return rc;
    if (!dt_io) return fail(RGPU_EINVAL, "null dt");
    const int nb = reduce_blocks();
    rc = amr_courant_launch(*A); if (rc) return rc;
    const double vol = std::pow(A->dx, G.p.ndim), dt0 = G.p.courant_factor * A->dx / G.p.smallc;
    courant_reduce_kernel<<<1, 1024, 0, G.stream>>>(A->d_part, nb, *dt_io, dt0, vol, A->d_out, A->d_dt, nullptr);
    CUDA_OK(cudaGetLastError());
    A->launches += 2;
    if (G.comm && G.nranks > 1) {   // MPI_ALLREDUCE MIN(1) + SUM(3), courant_fine.f90:138-141
      NCCL_OK(ncclAllReduce(A->d_out, A->d_out, 1, ncclDouble, ncclMin, G.comm, G.stream));
      NCCL_OK(ncclAllReduce(A->d_out + 1, A->d_out + 1, 3, ncclDouble, ncclSum, G.comm, G.stream));
    }
    double out[4];
    CUDA_OK(cudaMemcpyAsync(out, A->d_out, sizeof(out), cudaMemcpyDeviceToHost, G.stream));
    CUDA_OK(cudaStreamSynchronize(G.stream));
    *dt_io = std::min(*dt_io, out[0]);
    if (sums) { sums[0] += out[1]; sums[1] += out[2]; sums[2] += out[3]; }
    return RGPU_OK;
  }
  Level* L; int rc = check_level(ilevel, &L); if (rc) return rc;
  if (!dt_io) return fail(RGPU_EINVAL, "null dt");
  rc = launch_courant(*L, *dt_io, nullptr); if (rc) return rc;
  double out[5];
  CUDA_OK(cudaMemcpyAsync(out, L->d_out, sizeof(out), cudaMemcpyDeviceToHost, G.stream));
  CUDA_OK(cudaStreamSynchronize(G.stream));
  if (G.comm && G.nranks > 1) {
    // MPI_ALLREDUCE SUM(3 or 4) + MIN(1) of courant_fine.f90:138-141, carried by NCCL
    double* d = L->d_out;
    NCCL_OK(ncclAllReduce(d, d, 1, ncclDouble, ncclMin, G.comm, G.stream));
    NCCL_OK(ncclAllReduce(d + 1, d + 1, 4, ncclDouble, ncclSum, G.comm, G.stream));
    CUDA_OK(cudaMemcpyAsync(out, L->d_out, sizeof(out), cudaMemcpyDeviceToHost, G.stream));
    CUDA_OK(cudaStreamSynchronize(G.stream));
  }
  *dt_io = std::min(*dt_io, out[0]);
  if (sums) { sums[0] += out[1]; sums[1] += out[2]; sums[2] += out[3]; if (G.p.mhd) sums[3] += out[4]; }
  return RGPU_OK;
}

int rgpu_make_boundary_hydro(int ilevel) {
  if (G.amr) { AmrLevel* A; int rc = check_amr_level(ilevel, &A); if (rc) return rc; return amr_boundaries(*A); }
  Level* L; int rc = check_level(ilevel, &L); if (rc) return rc;
  return launch_boundaries(*L, L->d_u[L->cur]);
}

int rgpu_make_virtual_fine(int ilevel) {
  if (G.amr) { AmrLevel* A; int rc = check_amr_level(ilevel, &A); if (rc) return rc; return amr_exchange(*A, G.d_uold, false); }
  Level* L; int rc = check_level(ilevel, &L); if (rc) return rc;
  return exchange_ghosts(*L, L->d_u[L->cur], false);
}
int rgpu_make_virtual_reverse(int ilevel) {
  if (G.amr) { AmrLevel* A; int rc = check_amr_level(ilevel, &A); if (rc) return rc; return amr_exchange(*A, G.d_unew, true); }
  Level* L; int rc = check_level(ilevel, &L); if (rc) return rc;
  if (!L->unew_valid) return fail(RGPU_EINVAL, "make_virtual_reverse before godunov_fine");
  return exchange_ghosts(*L, L->d_u[1 - L->cur], true);
}

int rgpu_godunov_fine(int ilevel, double dt, const double* uold, double* unew) {
  if (G.amr) {   // Level-0 in AMR mode: uold and unew (it carries the refluxes of finer levels) both travel
    AmrLevel* A; int rc = check_amr_level(ilevel, &A); if (rc) return rc;
    if (!uold || !unew) return fail(RGPU_EINVAL, "null state array");
    if (!(dt > 0)) return fail(RGPU_EINVAL, "dt=%g", dt);
    if (G.p.pressure_fix) return fail(RGPU_EUNSUPPORTED, "pressure_fix: divu / enew live on the device; use the device-resident calls (rgpu_set_unew ... rgpu_set_uold)");
    const size_t bytes = sizeof(double) * G.nvs * G.ncell;
    CUDA_OK(cudaMemcpyAsync(G.d_uold, uold, bytes, cudaMemcpyHostToDevice, G.stream));
    CUDA_OK(cudaMemcpyAsync(G.d_unew, unew, bytes, cudaMemcpyHostToDevice, G.stream));
    rc = amr_godunov(*A, ilevel, dt); if (rc) return rc;
    CUDA_OK(cudaMemcpyAsync(unew, G.d_unew, bytes, cudaMemcpyDeviceToHost, G.stream));
    CUDA_OK(cudaStreamSynchronize(G.stream));
    return RGPU_OK;
  }
  Level* L; int rc = check_level(ilevel, &L); if (rc) return rc;
  if (!uold || !unew) return fail(RGPU_EINVAL, "null state array");
  if (!(dt > 0)) return fail(RGPU_EINVAL, "dt=%g", dt);
  if (G.p.pressure_fix) return fail(RGPU_EUNSUPPORTED, "pressure_fix: divu / enew live on the device; use the device-resident calls (rgpu_set_unew ... rgpu_set_uold)");
  rc = need_force(*L); if (rc) return rc;
  CUDA_OK(cudaMemcpyAsync(L->d_dt, &dt, sizeof(double), cudaMemcpyHostToDevice, G.stream));
  L->dt_last = dt;   // poisson: unew = uold + dF with the gravity predictor; the host's set_uold adds the source term
  if (!L->slabs.empty() && G.pipeline && !G.timing) return godunov_fine_pipelined(*L, uold, unew);
  rc = upload_into(*L, uold, L->d_u[L->cur]); if (rc) return rc;
  rc = launch_sweep(*L); if (rc) return rc;
  L->unew_valid = true;
  return download_from(*L, unew, L->d_u[1 - L->cur], true);
}

int rgpu_level_steps(int ilevel, int nstep, double* dt_hist, double sums_last[3]) {
  if (G.amr) return fail(RGPU_EUNSUPPORTED, "rgpu_level_steps is the levelmin=levelmax fast path; in AMR mode call the per-level routines in amr_step order");
  Level* L; int rc = check_level(ilevel, &L); if (rc) return rc;
  if (nstep < 1) return fail(RGPU_EINVAL, "nstep=%d", nstep);
  if (L->hist_cap < nstep + 1) {
    cudaFree(L->d_hist);
    CUDA_OK(cudaMalloc(&L->d_hist, sizeof(double) * (nstep + 1)));
    L->hist_cap = nstep + 1;
  }
  const double dt_cap = G.p.boxlen / G.p.smallc;   // pm/newdt_fine.f90:47-51
  const bool multi = G.comm && G.nranks > 1 && !L->peers.empty();
  const bool fused = multi && L->d_emit_off != nullptr;
  const bool ovl = fused && L->overlap && G.comm_x != nullptr && !G.timing;   // per-kernel timing runs keep one sweep launch
  const bool pfix = G.p.pressure_fix != 0;
  CUDA_OK(cudaEventRecord(G.ev2, G.stream));
  // amr_step order.  Ghost shells of uold are current on entry (upload / previous step).
  if (fused) rc = exchange_ghosts_fused(*L, L->d_u[L->cur], G.stream, G.comm); else rc = exchange_ghosts(*L, L->d_u[L->cur], false);
  if (rc) return rc;
  rc = launch_boundaries(*L, L->d_u[L->cur]); if (rc) return rc;
  rc = launch_courant(*L, dt_cap, L->d_hist); if (rc) return rc;                    // courant_fine  amr_step.f90:326
  if (ovl) {   // unused columns of the shared partial array stay neutral (min: huge, sums: 0)
    const size_t stride = 2 * (size_t)L->nblocks;
    CUDA_OK(cudaMemsetAsync(L->d_part, 0x7f, sizeof(double) * stride, G.stream));
    CUDA_OK(cudaMemsetAsync(L->d_part + stride, 0, sizeof(double) * 3 * stride, G.stream));
    CUDA_OK(cudaEventRecord(L->ev_x, G.stream));
  }
  for (int s = 0; s < nstep; s++) {
    if (G.comm && G.nranks > 1) {
      NCCL_OK(ncclAllReduce(L->d_dt, L->d_dt, 1, ncclDouble, ncclMin, G.comm, G.stream));
      if (s < nstep) CUDA_OK(cudaMemcpyAsync(L->d_hist + s, L->d_dt, sizeof(double), cudaMemcpyDeviceToDevice, G.stream));
    }
    // pressure_fix: set_unew's divu / enew (owned cells of uold only), the sweep, then set_uold's pdV source (it reads the ghost
    // and boundary shells of uold) and, after the swap, the energy switch.  The sweep's fused Courant partials would describe the
    // state before the switch: dt and the sums of the next step come from a Courant scan of the switched state instead.
    if (pfix) { rc = launch_pfix_pass(*L, PFIX_INIT, 0.0, nullptr); if (rc) return rc; }   // set_unew :333
    if (ovl) {
      // interior tiles read owned cells only: they run while the exchange of the previous step (stream s_x) fills the ghost
      // shells; the frame (outer tile ring + plane caps) waits for it.  Same kernel, same arithmetic, two launches.
      rc = launch_sweep(*L, -1, -1, 1, true); if (rc) return rc;
      CUDA_OK(cudaStreamWaitEvent(G.stream, L->ev_x, 0));
      rc = launch_sweep(*L, -1, -1, 2, true); if (rc) return rc;
      if (pfix) {   // after the frame launch: the ghost shells of uold are the ones the previous step's exchange sent
        rc = launch_pfix_pass(*L, PFIX_PDV, 0.0, L->d_dt); if (rc) return rc;
      } else {
        rc = launch_reduce(*L, 2 * L->nblocks, dt_cap, L->d_hist + s + 1); if (rc) return rc;
      }
      rc = carry_shells(*L, L->d_u[L->cur], L->d_u[1 - L->cur], false); if (rc) return rc;
      L->cur = 1 - L->cur;
      if (pfix) {   // the exchange below packs the switched state
        rc = launch_pfix_pass(*L, PFIX_SWITCH, 0.0, L->d_dt); if (rc) return rc;
        rc = launch_courant(*L, dt_cap, L->d_hist + s + 1); if (rc) return rc;
      }
      CUDA_OK(cudaEventRecord(L->ev_s, G.stream));
      CUDA_OK(cudaStreamWaitEvent(G.s_x, L->ev_s, 0));
      rc = exchange_ghosts_fused(*L, L->d_u[L->cur], G.s_x, G.comm_x); if (rc) return rc;   // make_virtual_fine :505
      {   // make_boundary_hydro :514 on the exchange stream (it reads the fresh ghost octs at box corners)
        cudaStream_t keep = G.stream; G.stream = G.s_x;
        rc = launch_boundaries(*L, L->d_u[L->cur]);
        G.stream = keep;
        if (rc) return rc;
      }
      CUDA_OK(cudaEventRecord(L->ev_x, G.s_x));
      continue;
    }
    rc = launch_sweep(*L, -1, -1, 0, true); if (rc) return rc;                       // set_unew + godunov_fine + set_uold  :333,:388,:423
    if (pfix) { rc = launch_pfix_pass(*L, PFIX_PDV, 0.0, L->d_dt); if (rc) return rc; }
    else { rc = launch_reduce(*L, L->nblocks, dt_cap, L->d_hist + s + 1); if (rc) return rc; }  // courant_fine of the next step
    rc = carry_shells(*L, L->d_u[L->cur], L->d_u[1 - L->cur], !fused); if (rc) return rc;
    L->cur = 1 - L->cur;
    if (pfix) {
      rc = launch_pfix_pass(*L, PFIX_SWITCH, 0.0, L->d_dt); if (rc) return rc;
      rc = launch_courant(*L, dt_cap, L->d_hist + s + 1); if (rc) return rc;
    }
    if (fused) rc = exchange_ghosts_fused(*L, L->d_u[L->cur], G.stream, G.comm); else rc = exchange_ghosts(*L, L->d_u[L->cur], false);   // make_virtual_fine :505
    if (rc) return rc;
    rc = launch_boundaries(*L, L->d_u[L->cur]); if (rc) return rc;                  // make_boundary_hydro :514
  }
  if (ovl) CUDA_OK(cudaStreamWaitEvent(G.stream, L->ev_x, 0));
  L->unew_valid = false;
  L->pfix_ready = false;
  CUDA_OK(cudaEventRecord(G.ev3, G.stream));
  if (dt_hist) CUDA_OK(cudaMemcpyAsync(dt_hist, L->d_hist, sizeof(double) * nstep, cudaMemcpyDeviceToHost, G.stream));
  double out[5];
  CUDA_OK(cudaMemcpyAsync(out, L->d_out, sizeof(out), cudaMemcpyDeviceToHost, G.stream));
  CUDA_OK(cudaStreamSynchronize(G.stream));
  if (sums_last) { sums_last[0] = out[1]; sums_last[1] = out[2]; sums_last[2] = out[3]; if (G.p.mhd) sums_last[3] = out[4]; }
  { float ms = 0; cudaEventElapsedTime(&ms, G.ev2, G.ev3); L->last_steps_ms = ms; }
  return RGPU_OK;
}

// amr_step(levelmin, 1) x ncoarse with every time step kept on the device: the recursion and the sub-cycling run on the host
// (they only depend on which levels hold octs), but no value travels back -- courant_fine's reduction, the MIN with the coarser
// level's dt/nsubcycle and the dtnew(l-1) = dtold(l) + dtnew(l) synchronisation are tiny kernels on device-resident
// dtnew/dtold, so the ~90 launches of a coarse step queue back to back.  Same arithmetic, same order as the host-driven
// sequence (ramses_b200.hydro.amr_step): bit-identical state and time steps.
// numbtot(1,ilevel) over all ranks (the reference gates amr_step and its recursion on the GLOBAL oct count, amr/amr_step.f90:33,345:
// a rank that owns no oct of a level still takes part in the level's all-reduce and ghost exchanges)
static int refresh_numbtot() {
  for (int l = 0; l <= MAXLEVEL + 1; l++) G.numbtot[l] = (l >= 1 && l <= MAXLEVEL && G.alev[l].bound) ? G.alev[l].nact : 0;
  if (G.comm && G.nranks > 1) {
    if (!G.d_numb) CUDA_OK(cudaMalloc(&G.d_numb, sizeof(int) * (MAXLEVEL + 2)));
    CUDA_OK(cudaMemcpyAsync(G.d_numb, G.numbtot, sizeof(int) * (MAXLEVEL + 2), cudaMemcpyHostToDevice, G.stream));
    NCCL_OK(ncclAllReduce(G.d_numb, G.d_numb, MAXLEVEL + 2, ncclInt, ncclSum, G.comm, G.stream));
    CUDA_OK(cudaMemcpyAsync(G.numbtot, G.d_numb, sizeof(int) * (MAXLEVEL + 2), cudaMemcpyDeviceToHost, G.stream));
    CUDA_OK(cudaStreamSynchronize(G.stream));
  }
  return RGPU_OK;
}

// nsub = nsubcycle(1:nlevelmax) of amr_parameters, passed as the Fortran array: nsub[l-1] = nsubcycle(l)
static int amr_step_dev(int l, int icount, int levelmin, const int* nsub) {
  AmrLevel& A = G.alev[l];
  if (G.numbtot[l] == 0) return RGPU_OK;                                   // amr_step.f90:33
  if (!A.bound) return fail(RGPU_EINVAL, "level %d holds octs on other ranks: bind it on every rank (ngrid_active = 0 is fine)", l);
  const int nlev = G.p.nlevelmax;
  int rc;
  auto op = [&](int o, int lev, double nsc, double nsl, int ic) {
    amr_dt_op_kernel<<<1, 32, 0, G.stream>>>(o, G.d_dtn, G.d_dto, A.d_dt, lev, levelmin, nsc, nsl, ic);
  };
  op(DT_SAVE_OLD, l, 1.0, 1.0, icount);
  {   // courant_fine :326 (newdt_fine: dtnew = boxlen/smallc, then the CFL scan)
    const int nb = reduce_blocks();
    rc = amr_courant_launch(A); if (rc) return rc;
    const double vol = std::pow(A.dx, G.p.ndim), dt0 = G.p.courant_factor * A.dx / G.p.smallc;
    courant_reduce_kernel<<<1, 1024, 0, G.stream>>>(A.d_part, nb, G.p.boxlen / G.p.smallc, dt0, vol, A.d_out, A.d_dt, nullptr);
    CUDA_OK(cudaGetLastError());
    if (G.comm && G.nranks > 1) NCCL_OK(ncclAllReduce(A.d_dt, A.d_dt, 1, ncclDouble, ncclMin, G.comm, G.stream));
    A.launches += 2;
  }
  op(DT_AFTER_COURANT, l, l > levelmin ? (double)nsub[l - 2] : 1.0, 1.0, icount);
  rc = amr_set_unew(A); if (rc) return rc;                            // set_unew :333
  if (l < nlev && G.numbtot[l + 1] > 0) {                               // :345-361
    rc = amr_step_dev(l + 1, 1, levelmin, nsub); if (rc) return rc;
    if (nsub[l - 1] == 2) { rc = amr_step_dev(l + 1, 2, levelmin, nsub); if (rc) return rc; }
  } else if (l < nlev) {
    op(DT_NO_FINER, l, 1.0, (double)nsub[l - 1], icount);
  }
  rc = amr_godunov(A, l, 0.0, G.d_dtn + l); if (rc) return rc;         // :388
  if (G.comm && G.nranks > 1) { rc = amr_exchange(A, G.d_unew, true); if (rc) return rc; }     // :397
  rc = amr_set_uold(A, l, G.d_dtn + l); if (rc) return rc;            // set_uold :423 (source terms, scalar floor fix, energy switch)
  if (l < nlev && A.nact > 0 && G.p.mhd) { rc = mhd_amr_upload(A); if (rc) return rc; }
  else if (l < nlev && A.nact > 0) {                                    // upload_fine :441
    const int n = A.nact * T_();
    amr_upload_kernel<<<(n + 127) / 128, 128, 0, G.stream>>>(G.d_uold, G.d_son - 1, A.d_active, A.nact, G.ncoarse, G.ngridmax, G.ncell, T_(), G.p.nvar, G.p.smallr, G.interpol_var, G.p.ndim);
    CUDA_OK(cudaGetLastError());
    A.launches++;
  }
  if (G.comm && G.nranks > 1) { rc = amr_exchange(A, G.d_uold, false); if (rc) return rc; }    // :505
  rc = amr_boundaries(A); if (rc) return rc;                           // :514
  if (l > levelmin) op(DT_SYNC_COARSE, l, (double)nsub[l - 2], 1.0, icount);   // :567-577
  A.launches += 4;
  return RGPU_OK;
}

int rgpu_amr_steps(int levelmin, const int* nsubcycle, int ncoarse_steps, double* dt_hist) {
  if (!G.init || !G.amr) return fail(RGPU_EINVAL, "rgpu_amr_steps needs AMR mode (rgpu_set_amr)");
  if (levelmin < 1 || levelmin > G.p.nlevelmax || !nsubcycle || ncoarse_steps < 1) return fail(RGPU_EINVAL, "bad argument");
  for (int l = levelmin; l <= G.p.nlevelmax; l++)
    if (nsubcycle[l - 1] != 1 && nsubcycle[l - 1] != 2) return fail(RGPU_EINVAL, "nsubcycle(%d)=%d (1 or 2)", l, nsubcycle[l - 1]);   // amr/read_params.f90:441
  { const int rc0 = refresh_numbtot(); if (rc0) return rc0; }
  if (!G.d_dtn) {
    CUDA_OK(cudaMalloc(&G.d_dtn, sizeof(double) * (MAXLEVEL + 2)));
    CUDA_OK(cudaMalloc(&G.d_dto, sizeof(double) * (MAXLEVEL + 2)));
    CUDA_OK(cudaMemset(G.d_dtn, 0, sizeof(double) * (MAXLEVEL + 2)));
    CUDA_OK(cudaMemset(G.d_dto, 0, sizeof(double) * (MAXLEVEL + 2)));
  }
  std::vector<double> hist(ncoarse_steps);
  double* d_hist = nullptr;
  CUDA_OK(cudaMalloc(&d_hist, sizeof(double) * ncoarse_steps));
  CUDA_OK(cudaEventRecord(G.ev2, G.stream));
  // Graph replay: single rank, no timing instrumentation; the first step of a call always runs eagerly (it also performs the
  // one-time cudaFuncSetAttribute calls), the second is captured, the rest replay.  RGPU_AMR_GRAPH=0 disables.
  static int graph_env = -1;
  if (graph_env < 0) { const char* e = getenv("RGPU_AMR_GRAPH"); graph_env = e ? atoi(e) : 1; }
  const bool graph_ok = graph_env != 0 && !(G.comm && G.nranks > 1) && !G.timing;
  if (G.amr_graph) {   // captured for another levelmin / nsubcycle?
    bool same = G.amr_graph_levelmin == levelmin;
    for (int l = levelmin; l <= G.p.nlevelmax && same; l++) same = G.amr_graph_nsub[l] == nsubcycle[l - 1];
    if (!same) drop_amr_graph();
  }
  for (int s = 0; s < ncoarse_steps; s++) {
    if (graph_ok && s > 0 && !G.amr_graph) {
      long long before[MAXLEVEL + 1];
      for (int l = 0; l <= MAXLEVEL; l++) before[l] = G.alev[l].launches;
      cudaGraph_t g = nullptr;
      CUDA_OK(cudaStreamBeginCapture(G.stream, cudaStreamCaptureModeThreadLocal));
      const int rc = amr_step_dev(levelmin, 1, levelmin, nsubcycle);
      const cudaError_t ce = cudaStreamEndCapture(G.stream, &g);
      if (rc || ce != cudaSuccess) { if (g) cudaGraphDestroy(g); cudaFree(d_hist); return rc ? rc : fail(RGPU_ECUDA, "graph capture of the coarse step: %s", cudaGetErrorString(ce)); }
      const cudaError_t ie = cudaGraphInstantiate(&G.amr_graph, g, 0);
      cudaGraphDestroy(g);
      if (ie != cudaSuccess) { G.amr_graph = nullptr; cudaFree(d_hist); return fail(RGPU_ECUDA, "graph instantiation: %s", cudaGetErrorString(ie)); }
      for (int l = 0; l <= MAXLEVEL; l++) { G.amr_graph_launches[l] = G.alev[l].launches - before[l]; G.alev[l].launches = before[l]; }
      G.amr_graph_levelmin = levelmin;
      for (int l = levelmin; l <= G.p.nlevelmax; l++) G.amr_graph_nsub[l] = nsubcycle[l - 1];
    }
    if (graph_ok && s > 0 && G.amr_graph) {
      CUDA_OK(cudaGraphLaunch(G.amr_graph, G.stream));
      for (int l = 0; l <= MAXLEVEL; l++) G.alev[l].launches += G.amr_graph_launches[l];
    } else {
      const int rc = amr_step_dev(levelmin, 1, levelmin, nsubcycle);
      if (rc) { cudaFree(d_hist); return rc; }
    }
    CUDA_OK(cudaMemcpyAsync(d_hist + s, G.d_dtn + levelmin, sizeof(double), cudaMemcpyDeviceToDevice, G.stream));
  }
  CUDA_OK(cudaEventRecord(G.ev3, G.stream));
  CUDA_OK(cudaMemcpyAsync(hist.data(), d_hist, sizeof(double) * ncoarse_steps, cudaMemcpyDeviceToHost, G.stream));
  CUDA_OK(cudaStreamSynchronize(G.stream));
  cudaFree(d_hist);
  if (dt_hist) memcpy(dt_hist, hist.data(), sizeof(double) * ncoarse_steps);
  { float ms = 0; cudaEventElapsedTime(&ms, G.ev2, G.ev3); G.alev[levelmin].last_steps_ms = ms; }
  return RGPU_OK;
}

int rgpu_level_totals(int nlevelmax, int* numbtot) {
  if (!G.init || !numbtot || nlevelmax < 1 || nlevelmax > MAXLEVEL) return fail(RGPU_EINVAL, "bad argument");
  if (G.amr) { const int rc = refresh_numbtot(); if (rc) return rc; }
  else for (int l = 1; l <= nlevelmax; l++) G.numbtot[l] = 0;
  for (int l = 1; l <= nlevelmax; l++) numbtot[l - 1] = G.numbtot[l];
  return RGPU_OK;
}

int rgpu_hydro_flag(int ilevel, const double err_grad[3], const double floor[3], int* flag1) {
  if (!G.init || !G.amr) return fail(RGPU_EINVAL, "rgpu_hydro_flag needs AMR mode (rgpu_set_amr)");
  AmrLevel* A; int rc = check_amr_level(ilevel, &A); if (rc) return rc;
  if (!err_grad || !floor || !flag1) return fail(RGPU_EINVAL, "null argument");
  if (G.p.nvar != G.p.ndim + 2) return fail(RGPU_EUNSUPPORTED, "hydro_flag: nvar = ndim+2 only");
  if (ilevel >= G.p.nlevelmax || A->nact == 0) return RGPU_OK;                                   // hydro_flag.f90:31-32
  if (err_grad[0] == -1.0 && err_grad[1] == -1.0 && err_grad[2] == -1.0) return RGPU_OK;          // :56-66
  const int T = T_(), n = A->nact * T;
  int* d_out = nullptr;
  CUDA_OK(cudaMalloc(&d_out, sizeof(int) * n));
  const int nb = (n + 127) / 128;
#define HF(ND) amr_hydro_flag_kernel<ND><<<nb, 128, 0, G.stream>>>(amr_tree(), G.d_uold, A->d_active, A->nact, ilevel, G.p.gamma, G.p.smallr, \
                 err_grad[0], err_grad[1], err_grad[2], floor[0], floor[1], floor[2], d_out)
  if (G.p.ndim == 1) HF(1); else if (G.p.ndim == 2) HF(2); else HF(3);
#undef HF
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { cudaFree(d_out); return fail(RGPU_ECUDA, "hydro_flag launch: %s", cudaGetErrorString(e)); }
  A->launches++;
  std::vector<int> out(n), act(A->nact);
  CUDA_OK(cudaMemcpyAsync(out.data(), d_out, sizeof(int) * n, cudaMemcpyDeviceToHost, G.stream));
  CUDA_OK(cudaMemcpyAsync(act.data(), A->d_active, sizeof(int) * A->nact, cudaMemcpyDeviceToHost, G.stream));
  CUDA_OK(cudaStreamSynchronize(G.stream));
  cudaFree(d_out);
  for (int o = 0; o < A->nact; o++)
    for (int ind = 0; ind < T; ind++)
      if (out[(size_t)o * T + ind]) flag1[(size_t)G.ncoarse + (size_t)ind * G.ngridmax + act[o] - 1] = 1;   // flag1(ind_cell) = 1 :193
  return RGPU_OK;
}

int rgpu_set_interpol_mag(int interpol_mag_type) {
  if (!G.init) return fail(RGPU_EINVAL, "rgpu_init has not been called");
  if (interpol_mag_type < -1 || interpol_mag_type > 3) return fail(RGPU_EINVAL, "interpol_mag_type=%d (-1 = interpol_type, 0..3)", interpol_mag_type);
  drop_amr_graph();
  G.interpol_mag_type = interpol_mag_type;
  return RGPU_OK;
}
int rgpu_set_boundary_var(int ibound, const double* var) {
  if (!G.init) return fail(RGPU_EINVAL, "rgpu_init has not been called");
  if (ibound < 1 || ibound > 64 || !var) return fail(RGPU_EINVAL, "ibound=%d (1..64) / null var", ibound);
  if (G.p.mhd) return fail(RGPU_EUNSUPPORTED, "MHD build: imposed boundaries not supported");
  drop_amr_graph();
  for (int iv = 0; iv < G.p.nvar && iv < 8; iv++) G.bvar[ibound - 1][iv] = var[iv];
  G.bvar_set[ibound - 1] = true;
  return RGPU_OK;
}
int rgpu_upload_force(const double* f) {
  if (!G.init) return fail(RGPU_EINVAL, "rgpu_init has not been called");
  if (!G.p.poisson) return fail(RGPU_EINVAL, "rgpu_upload_force: rgpu_params.poisson is 0");
  if (!f) return fail(RGPU_EINVAL, "null f");
  if (!G.amr) {   // levelmin=levelmax: gather f(1:ncell,1:ndim) into the f store of every bound dense level (no full-size mirror)
    int n = 0;
    for (int l = 1; l <= MAXLEVEL; l++) {
      Level& L = G.lev[l];
      if (!L.bound || !L.dense || !L.d_f) continue;
      const int rc = upload_into(L, f, L.d_f, G.p.ndim); if (rc) return rc;
      L.f_valid = true;
      n++;
    }
    if (n == 0) return fail(RGPU_EINVAL, "rgpu_upload_force: bind a level first");
    CUDA_OK(cudaStreamSynchronize(G.stream));
    return RGPU_OK;
  }
  if (!G.d_force) return fail(RGPU_EINVAL, "bind the tree first");
  CUDA_OK(cudaMemcpyAsync(G.d_force, f, sizeof(double) * G.p.ndim * G.ncell, cudaMemcpyHostToDevice, G.stream));
  CUDA_OK(cudaStreamSynchronize(G.stream));
  return RGPU_OK;
}
int rgpu_download_pressure_fix(double* divu, double* enew) {
  if (!G.init || !G.p.pressure_fix) return fail(RGPU_EINVAL, "rgpu_download_pressure_fix needs rgpu_params.pressure_fix");
  if (!G.amr) {   // every bound dense level: divu / enew of its active cells; every other entry keeps the caller's value
    const int T = T_();
    std::vector<double> h;
    for (int l = 1; l <= MAXLEVEL; l++) {
      const Level& L = G.lev[l];
      if (!L.bound || !L.dense || !L.d_pfix) continue;
      const size_t vs = (size_t)T * L.nslot;
      h.resize(2 * vs);
      CUDA_OK(cudaMemcpyAsync(h.data(), L.d_pfix, sizeof(double) * 2 * vs, cudaMemcpyDeviceToHost, G.stream));
      CUDA_OK(cudaStreamSynchronize(G.stream));
      const DenseGeom& g = L.g;
      for (long long s = 0; s < L.nslot; s++) {
        const int ig = L.slot_igrid[s];
        const int ox = (int)(s % g.nox), oy = (int)((s / g.nox) % g.noy), oz = (int)(s / ((long long)g.nox * g.noy));
        if (ig <= 0 || 2 * ox < g.ox0 || 2 * ox >= g.ox1) continue;
        if (G.p.ndim > 1 && (2 * oy < g.oy0 || 2 * oy >= g.oy1)) continue;
        if (G.p.ndim > 2 && (2 * oz < g.oz0 || 2 * oz >= g.oz1)) continue;
        for (int ind = 0; ind < T; ind++) {
          const size_t c = (size_t)G.ncoarse + (size_t)ind * G.ngridmax + ig - 1;
          if (divu) divu[c] = h[(size_t)ind * L.nslot + s];
          if (enew) enew[c] = h[vs + (size_t)ind * L.nslot + s];
        }
      }
    }
    return RGPU_OK;
  }
  if (!G.d_unew) return fail(RGPU_EINVAL, "bind the tree first");
  if (divu) CUDA_OK(cudaMemcpyAsync(divu, d_divu(), sizeof(double) * G.ncell, cudaMemcpyDeviceToHost, G.stream));
  if (enew) CUDA_OK(cudaMemcpyAsync(enew, d_enew(), sizeof(double) * G.ncell, cudaMemcpyDeviceToHost, G.stream));
  CUDA_OK(cudaStreamSynchronize(G.stream));
  return RGPU_OK;
}

int rgpu_upload_fine(int ilevel) {
  if (!G.amr) return RGPU_OK;   // a dense (levelmin=levelmax) level has no split cells: upload_fine is a no-op
  AmrLevel* A; int rc = check_amr_level(ilevel, &A); if (rc) return rc;
  if (A->nact == 0 || ilevel >= G.p.nlevelmax) return RGPU_OK;
  if (G.p.mhd) return mhd_amr_upload(*A);
  const int n = A->nact * T_();
  amr_upload_kernel<<<(n + 127) / 128, 128, 0, G.stream>>>(G.d_uold, G.d_son - 1, A->d_active, A->nact, G.ncoarse, G.ngridmax, G.ncell, T_(), G.p.nvar, G.p.smallr,
                                                         G.interpol_var, G.p.ndim);
  CUDA_OK(cudaGetLastError());
  A->launches++;
  return RGPU_OK;
}

int rgpu_comm_unique_id(void* unique_id_128) {
  if (!unique_id_128) return fail(RGPU_EINVAL, "null id");
  ncclUniqueId id;
  NCCL_OK(ncclGetUniqueId(&id));
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId size");
  memcpy(unique_id_128, &id, 128);
  return RGPU_OK;
}
int rgpu_comm_init(int nranks, int rank, const void* unique_id_128) {
  if (!G.init) return fail(RGPU_EINVAL, "rgpu_init has not been called");
  if (G.comm) { ncclCommDestroy(G.comm); G.comm = nullptr; }
  ncclUniqueId id;
  memcpy(&id, unique_id_128, 128);
  NCCL_OK(ncclCommInitRank(&G.comm, nranks, id, rank));
  G.nranks = nranks; G.rank = rank;
  if (G.comm_x) { ncclCommDestroy(G.comm_x); G.comm_x = nullptr; }
  // second communicator for the exchange stream: the dt all-reduce (main stream) and the ghost exchange run concurrently
  NCCL_OK(ncclCommSplit(G.comm, 0, rank, &G.comm_x, nullptr));
  return RGPU_OK;
}

int rgpu_get_level_info(int ilevel, rgpu_level_info* o) {
  if (G.init && G.amr && o && ilevel >= 1 && ilevel <= MAXLEVEL && G.alev[ilevel].bound) {
    const AmrLevel& A = G.alev[ilevel];
    memset(o, 0, sizeof(*o));
    o->nslot = A.nact; o->kernel_launches = A.launches; o->last_steps_ms = A.last_steps_ms;
    if (A.dense_sweep) {   // the dense kernel's AMR variant sweeps the level (base box or refined patch): report its box
      const DenseGeom& g = G.lev[ilevel].g;
      o->dense = 1;
      o->ncell_box[0] = g.ncx; o->ncell_box[1] = g.ncy; o->ncell_box[2] = g.ncz;
      o->own_lo[0] = g.ox0; o->own_lo[1] = g.oy0; o->own_lo[2] = g.oz0;
      o->own_hi[0] = g.ox1; o->own_hi[1] = g.oy1; o->own_hi[2] = g.oz1;
      o->wrap[0] = g.wrapx; o->wrap[1] = g.wrapy; o->wrap[2] = g.wrapz;
    }
    return RGPU_OK;
  }
  if (!G.init || ilevel < 1 || ilevel > MAXLEVEL || !G.lev[ilevel].bound || !o) return fail(RGPU_EINVAL, "level %d not bound", ilevel);
  Level& L = G.lev[ilevel];
  o->dense = L.dense;
  o->ncell_box[0] = L.g.ncx; o->ncell_box[1] = L.g.ncy; o->ncell_box[2] = L.g.ncz;
  o->own_lo[0] = L.g.ox0; o->own_lo[1] = L.g.oy0; o->own_lo[2] = L.g.oz0;
  o->own_hi[0] = L.g.ox1; o->own_hi[1] = L.g.oy1; o->own_hi[2] = L.g.oz1;
  o->wrap[0] = L.g.wrapx; o->wrap[1] = L.g.wrapy; o->wrap[2] = L.g.wrapz;
  o->nslot = L.nslot; o->kernel_launches = L.launches; o->last_sweep_ms = L.last_sweep_ms; o->last_steps_ms = L.last_steps_ms;
  o->pipeline_slabs = (int)L.slabs.size(); o->sweep_variant = L.variant;
  return RGPU_OK;
}
int rgpu_selftest_div(long long npairs, unsigned long long seed, long long* mismatches) {
  if (!G.init) return fail(RGPU_EINVAL, "rgpu_init has not been called");
  unsigned long long* d;
  CUDA_OK(cudaMalloc(&d, 8));
  CUDA_OK(cudaMemset(d, 0, 8));
  const int nb = reduce_blocks(), nt = 256;
  const long long per = (npairs + (long long)nb * nt - 1) / ((long long)nb * nt);
  selftest_div_kernel<<<nb, nt, 0, G.stream>>>(per, seed, d);
  CUDA_OK(cudaGetLastError());
  unsigned long long h = 0;
  CUDA_OK(cudaMemcpyAsync(&h, d, 8, cudaMemcpyDeviceToHost, G.stream));
  CUDA_OK(cudaStreamSynchronize(G.stream));
  cudaFree(d);
  *mismatches = (long long)h;
  return RGPU_OK;
}
int rgpu_set_timing(int enable) { G.timing = enable != 0; return RGPU_OK; }
int rgpu_set_pipeline(int enable) { G.pipeline = enable != 0; return RGPU_OK; }
int rgpu_device_synchronize(void) {
  if (!G.init) return fail(RGPU_EINVAL, "rgpu_init has not been called");
  CUDA_OK(cudaStreamSynchronize(G.stream));
  return RGPU_OK;
}

}  // extern "C"

namespace {
// make_virtual_fine_dp / make_virtual_reverse_dp (amr/virtual_boundaries.f90:373,693) for ALL variables at once:
// one packed message per peer inside a single NCCL group (ncclSend/ncclRecv over NVLink) instead of nvar
// MPI_ISEND/IRECV rounds.  forward: emission octs -> peer's reception octs (copy); reverse: reception octs ->
// owner's emission octs (accumulate, in peer order like :852-863).
// forward exchange (make_virtual_fine_dp for all variables and ALL peers): one pack kernel, one NCCL group, one unpack kernel
int exchange_ghosts_fused(Level& L, double* u, cudaStream_t st, ncclComm_t comm) {
  if (L.peers.empty()) return RGPU_OK;
  if (!comm) return fail(RGPU_EINVAL, "ghost exchange needs rgpu_comm_init");
  const long long np = (long long)nplanes_();
  const int nseg = (int)L.peers.size();
  const long long ne = L.emit_off.back(), nr = L.recv_off.back();
  if (ne) {
    pack_all_kernel<<<(unsigned)((ne * np + 255) / 256), 256, 0, st>>>(u, L.d_emit_all, ne, L.nslot, (int)np, L.d_sbuf_all, L.d_emit_off, nseg);
    CUDA_OK(cudaGetLastError());
    L.launches++;
  }
  NCCL_OK(ncclGroupStart());
  for (int c = 0; c < nseg; c++) {
    const long long es = L.emit_off[c + 1] - L.emit_off[c], rs = L.recv_off[c + 1] - L.recv_off[c];
    if (es) NCCL_OK(ncclSend(L.d_sbuf_all + L.emit_off[c] * np, (size_t)(es * np), ncclDouble, c, comm, st));
    if (rs) NCCL_OK(ncclRecv(L.d_rbuf_all + L.recv_off[c] * np, (size_t)(rs * np), ncclDouble, c, comm, st));
  }
  NCCL_OK(ncclGroupEnd());
  if (nr) {
    unpack_all_kernel<<<(unsigned)((nr * np + 255) / 256), 256, 0, st>>>(u, L.d_recv_all, nr, L.nslot, (int)np, L.d_rbuf_all, L.d_recv_off, nseg);
    CUDA_OK(cudaGetLastError());
    L.launches++;
  }
  return RGPU_OK;
}

int exchange_ghosts(Level& L, double* u, bool reverse) {
  if (L.peers.empty()) return RGPU_OK;
  if (!G.comm) return fail(RGPU_EINVAL, "ghost exchange needs rgpu_comm_init");
  const long long np = (long long)nplanes_();
  for (auto& P : L.peers) {
    const int n = reverse ? P.nrecv : P.nemit;
    const int* sl = reverse ? P.d_recv : P.d_emit;
    double* buf = reverse ? P.d_rbuf : P.d_sbuf;
    if (n) {
      pack_kernel<<<(unsigned)(((long long)n * np + 255) / 256), 256, 0, G.stream>>>(u, sl, n, L.nslot, (int)np, buf);
      CUDA_OK(cudaGetLastError());
      L.launches++;
    }
  }
  NCCL_OK(ncclGroupStart());
  for (int c = 0; c < (int)L.peers.size(); c++) {
    PeerList& P = L.peers[c];
    const int nsend = reverse ? P.nrecv : P.nemit, nrecv = reverse ? P.nemit : P.nrecv;
    double* sb = reverse ? P.d_rbuf : P.d_sbuf;
    double* rb = reverse ? P.d_sbuf : P.d_rbuf;
    if (nsend) NCCL_OK(ncclSend(sb, (size_t)nsend * np, ncclDouble, c, G.comm, G.stream));
    if (nrecv) NCCL_OK(ncclRecv(rb, (size_t)nrecv * np, ncclDouble, c, G.comm, G.stream));
  }
  NCCL_OK(ncclGroupEnd());
  for (auto& P : L.peers) {
    const int n = reverse ? P.nemit : P.nrecv;
    const int* sl = reverse ? P.d_emit : P.d_recv;
    const double* buf = reverse ? P.d_sbuf : P.d_rbuf;
    if (n) {
      unpack_kernel<<<(unsigned)(((long long)n * np + 255) / 256), 256, 0, G.stream>>>(u, sl, n, L.nslot, (int)np, buf, reverse ? 1 : 0);
      CUDA_OK(cudaGetLastError());
      L.launches++;
    }
  }
  return RGPU_OK;
}
}  // namespace
