// sweep_dense.cuh -- fused per-level Godunov sweep over a dense box of octs (sm_90a).
//
// One persistent kernel = set_unew + godunov_fine (ctoprim -> uslope -> trace ->
// cmpflxm/riemann -> conservative update) + set_uold + the Courant scan of the NEW
// state, for a level whose octs fill a Cartesian box (levelmin=levelmax runs, and the
// owned sub-box + ghost shell of one rank in multi-GPU runs).
//
// Reference semantics: hydro/godunov_fine.f90:5-35,486-911 (godfine1),
// hydro/umuscl.f90:22-171 (unsplit).  The reference gathers a private 6^ndim patch
// per oct (ctoprim 27x, slopes/trace 8x, Riemann 1.5x per cell); here a CTA owns a
// (BX-2)x(BY-2) column of cells and marches along z, so every primitive state, slope,
// traced state and face flux is evaluated once (plus a one-cell halo ring) --
// bit-identical because each value is a deterministic function of the same inputs
// evaluated in the same operation order.
//
// Execution model:
//  * grid = one CTA per SM; the (column tile, z plane) space is cut into equal
//    contiguous shares, so every SM does the same work (no wave tail);
//  * a warp is one row of 32 cells along x: x-neighbour exchange (left face state,
//    right face flux) by warp shuffles; y exchange through shared memory; the z
//    exchange is a carry from the previous plane;
//  * the raw conserved state of plane k+2 is staged into shared memory with cp.async
//    while plane k is computed; ctoprim runs from the staging buffer into a 3-plane
//    ring of primitive variables (+1/rho);
//  * divisions that share a divisor use one correctly rounded reciprocal and a
//    3-instruction FMA correction per quotient (div_rn below) -- same bits as IEEE
//    division at a fraction of the FP64 issue slots.
//
// Data layout in HBM (the oct-tree layout, octs renumbered in lattice order):
//   u[(ivar*2^ndim + ind)*nslot + slot],  ind = ix+2*iy+4*iz cell-in-oct,
//   slot = ox + nox*(oy + noy*oz).
#pragma once
#include "hydro_device.cuh"

namespace rgpu {

struct DenseGeom {
  int ncx, ncy, ncz;          // box extent in cells (incl. ghost / boundary shell)
  int nox, noy, noz;          // box extent in octs
  int ox0, ox1, oy0, oy1, oz0, oz1;  // owned (active) cell range [o0,o1) per dim
  int wrapx, wrapy, wrapz;    // periodic wrap inside the box (no ghost shell in that dim)
  long long nslot;            // number of oct slots (stride between (ivar,ind) planes)
};

// Which (column tile, plane) pairs a launch covers.  mode 0: every tile x every owned plane.  Multi-GPU level steps split the
// sweep so that the ghost-oct exchange of step s overlaps the part of sweep s+1 that does not read ghost cells:
// mode 1 = interior (tiles [ix0,ix1) x [iy0,iy1), planes [iz0,iz1): every cell they read is an owned cell), mode 2 = the frame
// (the complement: outer tile ring over all planes + the bottom / top plane caps of the interior columns).  3-D only.
struct SweepWork {
  int mode;
  int ix0, ix1, iy0, iy1;
  int iz0, iz1;
};

struct SweepArgs {
  const double* uin;          // state at t^n   (uold)
  double* uout;               // state at t^n+1 (unew after set_uold)
  DenseGeom g;
  Phys P;
  const double* dt_dev;       // time step, device resident (written by the Courant reduce); NULL: use dt_val
  double dt_val;              // time step passed by value (host-driven per-level calls)
  double dx, inv_dx;
  int dx_pow2;                // dx is a power of two: x/dx == x*inv_dx exactly
  int ntx, nty;               // column tiles of the owned range
  long long nwork;            // ntx*nty*(owned planes): plane-tiles to distribute
  double* part;               // per-CTA partials [4][part_stride]: min dt, mass, etot, eint of the new state
  int part_stride, part_off;  // columns of `part` and the first column of this launch (0, 0: gridDim.x columns from column 0)
  SweepWork wk;
  // AMR variant (fully refined level inside an AMR run, godfine1 hydro/godunov_fine.f90:661-666,720-747,751-792):
  const unsigned char* refined;  // [2^ndim][nslot] son(cell)>0: fluxes through faces of refined cells are reset to zero
                                 // and the update ACCUMULATES into uout (= unew, which already holds the refluxes of the
                                 // finer level) instead of starting from uin
  // poisson (GRAV instantiation): the acceleration f of poisson_commons in the level-store layout [ndim][2^ndim][nslot]
  // (addressed like uin); every converted cell gets the gravity predictor (hydro/umuscl.f90:932-938)
  const double* force;
  int gsrc;                   // 1: set_uold's add_gravity_source_terms is fused into the update and the Courant scan of the
                              // new state uses sum|f| (rgpu_level_steps: f stays fixed over the steps of the call)
  // pressure_fix (PFIX instantiation): divu and enew in the level-store layout [2][2^ndim][nslot] (addressed like uout).  On
  // entry they hold set_unew's values (AMR variant: plus the finer level's refluxes); the sweep accumulates the face velocity
  // tmp1 and the internal-energy flux tmp2 into them like two more variables (hydro/godunov_fine.f90:735-745,775-786)
  double* pfix;
};

__device__ __forceinline__ int wrap_or_clamp(int c, int n, int wrap) {
  if (wrap) { c %= n; if (c < 0) c += n; }
  else { c = c < 0 ? 0 : (c >= n ? n - 1 : c); }
  return c;
}

template <int NDIM>
__device__ __forceinline__ long long cell_offset(const DenseGeom& g, int x, int y, int z) {
  int ind = (x & 1);
  long long slot = (x >> 1);
  if (NDIM > 1) { ind |= (y & 1) << 1; slot += (long long)g.nox * (y >> 1); }
  if (NDIM > 2) { ind |= (z & 1) << 2; slot += (long long)g.nox * g.noy * (z >> 1); }
  return (long long)ind * g.nslot + slot;
}

// decode work item w of a launch into (tile, first plane, number of consecutive planes before `wend` or the column end)
__device__ __forceinline__ void sweep_work_decode(const SweepArgs& a, long long w, long long wend, int& tix, int& tiy, int& z0, int& zn) {
  const DenseGeom& g = a.g;
  const SweepWork& k = a.wk;
  const int nzo = g.oz1 - g.oz0;
  if (k.mode == 0) {
    const long long col = w / nzo;
    const int zs = (int)(w - col * nzo);
    zn = (int)min((long long)(nzo - zs), wend - w);
    tix = (int)(col % a.ntx); tiy = (int)(col / a.ntx);
    z0 = g.oz0 + zs;
    return;
  }
  const int nxi = k.ix1 - k.ix0, nyi = k.iy1 - k.iy0;
  if (k.mode == 1) {
    const int nzi = k.iz1 - k.iz0;
    const long long col = w / nzi;
    const int zs = (int)(w - col * nzi);
    zn = (int)min((long long)(nzi - zs), wend - w);
    tix = k.ix0 + (int)(col % nxi); tiy = k.iy0 + (int)(col / nxi);
    z0 = k.iz0 + zs;
    return;
  }
  const long long ncolA = (long long)a.ntx * a.nty - (long long)nxi * nyi;
  const long long WA = ncolA * nzo;
  if (w < WA) {                                 // frame tiles, all planes
    long long c = w / nzo;
    const int zs = (int)(w - c * nzo);
    zn = (int)min((long long)(nzo - zs), wend - w);
    z0 = g.oz0 + zs;
    const long long nbot = (long long)a.ntx * k.iy0, ntop = (long long)a.ntx * (a.nty - k.iy1);
    if (c < nbot) { tiy = (int)(c / a.ntx); tix = (int)(c % a.ntx); return; }
    c -= nbot;
    if (c < ntop) { tiy = k.iy1 + (int)(c / a.ntx); tix = (int)(c % a.ntx); return; }
    c -= ntop;
    const int nside = k.ix0 + (a.ntx - k.ix1);
    const int r = (int)(c / nside), q = (int)(c % nside);
    tiy = k.iy0 + r;
    tix = q < k.ix0 ? q : k.ix1 + (q - k.ix0);
    return;
  }
  const long long wc = w - WA;                  // interior columns: bottom cap [oz0, iz0), then top cap [iz1, oz1)
  const int nlo = k.iz0 - g.oz0, nhi = g.oz1 - k.iz1, ncap = nlo + nhi;
  const long long col = wc / ncap;
  const int r = (int)(wc - col * ncap);
  tix = k.ix0 + (int)(col % nxi); tiy = k.iy0 + (int)(col / nxi);
  if (r < nlo) { z0 = g.oz0 + r; zn = (int)min((long long)(nlo - r), wend - w); }
  else { z0 = k.iz1 + (r - nlo); zn = (int)min((long long)(nhi - (r - nlo)), wend - w); }
}

__device__ __forceinline__ double warp_min(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { double t = __shfl_xor_sync(0xffffffffu, v, o); v = t < v ? t : v; }
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// flux scaling of unsplit: flux = fx*dt/dx (hydro/umuscl.f90:106,129,153).  dx a power of two: x/dx == x*(1/dx)
// exactly; otherwise the shared-reciprocal quotient (inv_dx = correctly rounded 1/dx).
template <int NV>
__device__ __forceinline__ void scale_fluxes(double* f, double dt, double dx, double inv_dx, int pow2) {
  if (pow2) {
#pragma unroll
    for (int n = 0; n < NV; n++) f[n] = (f[n] * dt) * inv_dx;
  } else {
#pragma unroll
    for (int n = 0; n < NV; n++) f[n] = div_rn(f[n] * dt, dx, inv_dx);
  }
}

#ifdef RGPU_HOST_NUMERICS   // tests/host_numerics (g++, no CUDA): a plain copy
inline void cp_async8(double* smem_dst, const double* gsrc) { *smem_dst = *gsrc; }
inline void cp_async_wait_all() {}
#else
__device__ __forceinline__ void cp_async8(double* smem_dst, const double* gsrc) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"(d), "l"(gsrc));
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;\n" ::: "memory"); }
#endif

template <int NDIM, int BX, int BY, bool GRAV = false, bool PFIX = false>
struct SweepSmem {
  static constexpr int NV = NDIM + 2;
  static constexpr int HY = (NDIM > 1) ? 1 : 0;
  static constexpr int HZ = (NDIM > 2) ? 1 : 0;
  static constexpr int QX = BX + 2, QY = HY ? BY + 2 : 1;
  static constexpr int NQ = NV + 1;                       // primitive variables + 1/rho
  static constexpr int NRING = HZ ? 3 : 1;
  static constexpr int NT = BX * BY;
  static constexpr size_t ring = (size_t)NRING * NQ * QY * QX;
  static constexpr size_t stage = HZ ? (size_t)NV * QY * QX : 0;
  static constexpr size_t fstage = (HZ && GRAV) ? (size_t)NDIM * QY * QX : 0;   // f of the staged plane
  static constexpr size_t exq = HY ? (size_t)NV * NT : 0;  // qm_y
  static constexpr size_t exf = HY ? (size_t)NV * NT : 0;  // Fy
  static constexpr size_t carry = HZ ? (size_t)3 * NV * NT : 0;
  static constexpr size_t exft = (PFIX && HY) ? (size_t)2 * NT : 0;    // tmp1, tmp2 of the y faces
  static constexpr size_t carryt = (PFIX && HZ) ? (size_t)4 * NT : 0;  // tmp1, tmp2 of the previous z face, partial divu / enew update
  static constexpr size_t doubles = ring + stage + fstage + exq + exf + carry + exft + carryt;
};

// LATE (experimental, not dispatched by the product yet; exercised by tests/host_numerics): the x/y part of the update of plane k
// is finished after the FIRST barrier of plane k+1 instead of after a third barrier of its own -- the y fluxes of the row above
// are complete by then -- so the plane loop has two CTA barriers instead of three.  Same arithmetic in the same order.
// GRAV (poisson): the gravity predictor with f = a.force in ctoprim of every converted cell and, when a.gsrc is set, set_uold's
// add_gravity_source_terms in the update plus the gravity term of the fused Courant scan.
// PFIX (pressure_fix; the 3-D AMR variant, and the plain form without GRAV in 1-D, 2-D and 3-D): every face also yields tmp1 =
// half*(ql(ln)+qr(ln)) and tmp2 = the internal-energy flux of the solver (hydro/umuscl.f90:844-850), scaled and masked like the
// fluxes; the update accumulates them into divu / enew (a.pfix, initialised by set_unew) in the same x, y, z order.  They travel
// like the fluxes: x by shuffle, y through shared memory, z in the carry.  The plain form starts the state from uin as usual.
template <int NDIM, int RIEMANN, int SLOPE, int BX, int BY, bool AMRV = false, bool LATE = false, bool GRAV = false, bool PFIX = false>
__global__ void __launch_bounds__(BX * BY, 1) sweep_dense_kernel(const SweepArgs a) {
  static_assert(!(LATE && AMRV), "the late-update variant exists for the plain dense sweep only");
  static_assert(!(LATE && GRAV), "the late-update variant exists for the plain dense sweep only");
  static_assert(!PFIX || (AMRV && NDIM == 3) || (!AMRV && !GRAV), "pressure_fix: the 3-D AMR variant, or the plain form without poisson");
  static_assert(!(LATE && PFIX), "the late-update variant exists for the plain dense sweep only");
  using S = SweepSmem<NDIM, BX, BY, GRAV, PFIX>;
  constexpr int NV = S::NV, HY = S::HY, HZ = S::HZ, QX = S::QX, QY = S::QY, NQ = S::NQ, NT = S::NT;
  constexpr int TXO = BX - 2;                 // owned cells per tile in x
  constexpr int TYO = HY ? BY - 2 : 1;
  constexpr int TWOTONDIM = 1 << NDIM;
  constexpr int PL = QY * QX;                 // one variable of one q plane
  static_assert(BX == 32, "a warp must be one x-row of the tile");
#ifdef RGPU_HOST_NUMERICS
  double* smem = rgpu_host_dyn_smem;           // dynamic shared memory of the emulated launch (tests/host_numerics)
#else
  extern __shared__ double smem[];
#endif
  double* qring = smem;                        // [NRING][NQ][QY][QX]
  double* stage = qring + S::ring;             // [NV][QY][QX] raw conserved state of the next plane
  double* fstg = stage + S::stage;             // GRAV: [NDIM][QY][QX] f of the next plane
  double* exq = fstg + S::fstage;              // [NV][NT] qm_y
  double* exf = exq + S::exq;                  // [NV][NT] Fy
  double* carry = exf + S::exf;                // [3][NV][NT]: qm_z, Fz, partial update of the previous plane
  double* exft = carry + S::carry;             // PFIX: [2][NT] tmp1, tmp2 of the y faces
  double* carryt = exft + S::exft;             // PFIX: [4][NT] tmp1, tmp2 of the z face below, partial divu / enew update
  constexpr int NPF = PFIX ? 2 : 1;            // tmp1, tmp2
  __shared__ double red[4][NT / 32];
  __shared__ unsigned char exm[AMRV ? NT : 1];   // AMRV: refined flag of every thread's cell (y exchange)

  const DenseGeom& g = a.g;
  const Phys& P = a.P;
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int tid = ty * BX + tx;
  const double dt = a.dt_dev ? *a.dt_dev : a.dt_val;
  const double dtdx = dt / a.dx;               // trace3d: dtdx = dt/dx (hydro/umuscl.f90:516)
  const size_t vstride = (size_t)TWOTONDIM * g.nslot;
  const int nzo = HZ ? g.oz1 - g.oz0 : 1;

  double my_dt = 1e300, my_mass = 0.0, my_etot = 0.0, my_eint = 0.0;

  // equal contiguous shares of the (column tile, plane) space
  long long w0 = a.nwork * blockIdx.x / gridDim.x;
  const long long w1 = a.nwork * (blockIdx.x + 1) / gridDim.x;
  while (w0 < w1) {
    int tix, tiy, z0, zn;
    if (HZ) sweep_work_decode(a, w0, w1, tix, tiy, z0, zn);
    else { const long long col = w0; zn = 1; z0 = 0; tix = (int)(col % a.ntx); tiy = (int)(col / a.ntx); }
    w0 += zn;
    const int x0 = g.ox0 + tix * TXO;
    const int y0 = HY ? g.oy0 + tiy * TYO : 0;
    const int z1 = HZ ? z0 + zn : 1;
    const int cx = x0 - 1 + tx;
    const int cy = HY ? y0 - 1 + ty : 0;

    const bool col_own = (tx >= 1) && (tx <= BX - 2) && (cx < g.ox1);
    const bool row_own = HY ? ((ty >= 1) && (ty <= BY - 2) && (cy < g.oy1)) : true;
    const bool own = col_own && row_own;
    const bool need_tr = (cx <= g.ox1) && (HY ? (cy <= g.oy1) : true);
    const bool need_fx = (tx >= 1) && row_own && (cx <= g.ox1);
    const bool need_fy = HY && (ty >= 1) && col_own && (cy <= g.oy1);

    // each thread owns the q-tile cells i = tid, tid+NT, ...; their global offsets without the z part are
    // plane independent and computed once per segment
    constexpr int NOWN = (PL + NT - 1) / NT;
    long long offxy[NOWN];
#pragma unroll
    for (int j = 0; j < NOWN; j++) {
      const int i = tid + j * NT;
      const int qx_ = i % QX, qy_ = i / QX;
      const int xc = wrap_or_clamp(x0 - 2 + qx_, g.ncx, g.wrapx);
      const int yc = HY ? wrap_or_clamp(y0 - 2 + qy_, g.ncy, g.wrapy) : 0;
      offxy[j] = cell_offset<NDIM>(g, xc, yc, 0);
    }
    auto zoff = [&](int z) -> long long {     // z part of cell_offset
      if (!HZ) return 0;
      const int zc = wrap_or_clamp(z, g.ncz, g.wrapz);
      return (long long)((zc & 1) << 2) * g.nslot + (long long)g.nox * g.noy * (zc >> 1);
    };
    // ctoprim (hydro/umuscl.f90:861) of one cell into ring slot `slot`; fg: GRAV: the cell's f
    auto to_ring = [&](const double* u, const double* fg, int slot, int i) {
      double q[NV];
      const double r = fmx(u[0], P.smallr);
      const double oneoverrho = rcp_rn(r);
      q[0] = r;
      double eken;
      q[1] = u[1] * oneoverrho;
      eken = 0.5 * q[1] * q[1];
      if (NDIM > 1) { q[2] = u[2] * oneoverrho; eken = eken + 0.5 * q[2] * q[2]; }
      if (NDIM > 2) { q[3] = u[3] * oneoverrho; eken = eken + 0.5 * q[3] * q[3]; }
      const double eint = fmx(u[NDIM + 1] * oneoverrho - eken - 0.0, P.smalle);
      q[NDIM + 1] = (P.gamma - 1.0) * r * eint;
      if (GRAV) {                              // gravity predictor (:932-938)
        const double dtxhalf = dt * 0.5;
        q[1] = q[1] + fg[0] * dtxhalf;
        if (NDIM > 1) q[2] = q[2] + fg[1 % NDIM] * dtxhalf;
        if (NDIM > 2) q[3] = q[3] + fg[2 % NDIM] * dtxhalf;
      } else {
        q[1] = q[1] + 0.0;                     // gravity predictor with gloc = 0 (:932-938): -0 -> +0
        if (NDIM > 1) q[2] = q[2] + 0.0;
        if (NDIM > 2) q[3] = q[3] + 0.0;
      }
      double* qs = qring + (size_t)slot * NQ * PL + i;
#pragma unroll
      for (int n = 0; n < NV; n++) qs[n * PL] = q[n];
      qs[NV * PL] = oneoverrho;
    };
    auto load_plane_direct = [&](int z, int slot) {
      const long long zo = zoff(z);
#pragma unroll
      for (int j = 0; j < NOWN; j++) {
        const int i = tid + j * NT;
        if (i >= PL) break;
        const long long off = offxy[j] + zo;
        double u[NV], fg[NDIM];
#pragma unroll
        for (int n = 0; n < NV; n++) u[n] = __ldg(a.uin + n * vstride + off);
        if (GRAV) {
#pragma unroll
          for (int d = 0; d < NDIM; d++) fg[d] = __ldg(a.force + d * vstride + off);
        }
        to_ring(u, fg, slot, i);
      }
    };
    auto stage_plane_async = [&](int z) {     // raw u (and f) of plane z -> staging buffer (cp.async, no registers)
      const long long zo = zoff(z);
#pragma unroll
      for (int j = 0; j < NOWN; j++) {
        const int i = tid + j * NT;
        if (i >= PL) break;
        const long long off = offxy[j] + zo;
#pragma unroll
        for (int n = 0; n < NV; n++) cp_async8(stage + n * PL + i, a.uin + n * vstride + off);
        if (GRAV) {
#pragma unroll
          for (int d = 0; d < NDIM; d++) cp_async8(fstg + d * PL + i, a.force + d * vstride + off);
        }
      }
    };
    auto stage_to_ring = [&](int slot) {       // each thread converts the cells it staged itself
      cp_async_wait_all();
      for (int i = tid; i < PL; i += NT) {
        double u[NV], fg[NDIM];
#pragma unroll
        for (int n = 0; n < NV; n++) u[n] = stage[n * PL + i];
        if (GRAV) {
#pragma unroll
          for (int d = 0; d < NDIM; d++) fg[d] = fstg[d * PL + i];
        }
        to_ring(u, fg, slot, i);
      }
    };

    __syncthreads();                           // previous segment done with shared memory
    if (HZ) {
      load_plane_direct(z0 - 2, 0);
      load_plane_direct(z0 - 1, 1);
      stage_plane_async(z0);
    }
    const int kbeg = HZ ? z0 - 1 : 0, kend = HZ ? z1 : 0;
    int mprev = 0;                             // AMRV: refined flag of my cell in the previous plane
    // LATE: uold + (Fx - Fx') and my own y flux of the pending plane.  3-D: both live in per-thread shared-memory slots (the
    // partial-update slot of `carry`, and NV*NT doubles behind `carry`: the launch must add them to the dynamic shared memory);
    // 1-D / 2-D: the single plane keeps them in registers
    double late_p1[(LATE && !HZ) ? NV : 1], late_fy[(LATE && !HZ) ? NV : 1];
    double* late_fys = carry + S::carry;
    bool late_pend = false;
    for (int k = kbeg; k <= kend; k++) {
      const int c = k - kbeg;
      const int sm1 = HZ ? c % 3 : 0, sc = HZ ? (c + 1) % 3 : 0, sp1 = HZ ? (c + 2) % 3 : 0;
      if (HZ) stage_to_ring(sp1); else load_plane_direct(0, 0);
      __syncthreads();
      if (HZ && k < kend) stage_plane_async(k + 2);
      if (LATE && HZ && late_pend) {           // y part of the update of plane k-1: every warp has written its Fy(k-1) by now
#pragma unroll
        for (int n = 0; n < NV; n++) {
          double u = carry[(2 * NV + n) * NT + tid];
          if (HY) u = u + (late_fys[n * NT + tid] - exf[n * NT + tid + BX]);
          carry[(2 * NV + n) * NT + tid] = u;
        }
        late_pend = false;
      }

      const int qx = tx + 1, qy = HY ? ty + 1 : 0;
      const double* qc = qring + (size_t)sc * NQ * PL + qy * QX + qx;   // + n*PL
      double q[NV], dq[NDIM][NV], t0[NV];
      const bool plane_flux = HZ ? (k >= z0 && k < z1) : true;          // x/y fluxes + update of this plane
      double qmx[NV];                                                   // left state of the +x face (to lane+1)
#pragma unroll
      for (int n = 0; n < NV; n++) { qmx[n] = 0.0; q[n] = 1.0; t0[n] = 0.0; }
      if (need_tr) {
#pragma unroll
        for (int n = 0; n < NV; n++) q[n] = qc[n * PL];
        const double rinv = qc[NV * PL];
        // ---- uslope (hydro/umuscl.f90:970) ----
        if (SLOPE < 0 && P.slope_type == 3 && NDIM > 1) {
          // positivity preserving unsplit slope :1101-1144 (2-D), :1328-1391 (3-D)
#pragma unroll
          for (int n = 0; n < NV; n++) {
            const double* qn = qc + n * PL;
            double vmin = 0, vmax = 0;
            bool first = true;
            for (int cc = (HZ ? -1 : 0); cc <= (HZ ? 1 : 0); cc++) {
              const double* qz = qring + (size_t)(HZ ? (cc < 0 ? sm1 : (cc > 0 ? sp1 : sc)) : 0) * NQ * PL + n * PL + qy * QX + qx;
              for (int aa = -1; aa <= 1; aa++)
                for (int bb = -1; bb <= 1; bb++) {
                  const double d = qz[bb * QX + aa] - q[n];
                  if (first) { vmin = d; vmax = d; first = false; }
                  else { vmin = fmn(vmin, d); vmax = fmx(vmax, d); }
                }
            }
            const double dfx = 0.5 * (qn[1] - qn[-1]);
            const double dfy = 0.5 * (qn[QX] - qn[-QX]);
            double dfz = 0, dff;
            if (HZ) {
              dfz = 0.5 * (qring[(size_t)sp1 * NQ * PL + n * PL + qy * QX + qx] - qring[(size_t)sm1 * NQ * PL + n * PL + qy * QX + qx]);
              dff = 0.5 * (fabs(dfx) + fabs(dfy) + fabs(dfz));
            } else dff = 0.5 * (fabs(dfx) + fabs(dfy));
            double slop;
            if (dff > 0.0) slop = fmn(1.0, fdiv(fmn(fabs(vmin), fabs(vmax)), dff));
            else slop = 1.0;
            dq[0][n] = slop * dfx;
            dq[HY][n] = slop * dfy;
            if (HZ) dq[NDIM - 1][n] = slop * dfz;
          }
        } else if (SLOPE < 0 && NDIM == 1 && P.slope_type >= 4 && P.slope_type <= 6) {
          // 1-D only limiters :1021-1068
          const double uvel = q[1];
#pragma unroll
          for (int n = 0; n < NV; n++) {
            const double* qn = qc + n * PL;
            const double qL = qn[-1], qC = qn[0], qR = qn[1];
            double r;
            if (P.slope_type == 4) {
              double dcen = uvel * dt / a.dx;
              const double dlft = 2.0 / (1.0 + dcen) * (qC - qL);
              const double drgt = 2.0 / (1.0 - dcen) * (qR - qC);
              const double dsgn = fsign1(dlft);
              double dlim = fmn(fabs(dlft), fabs(drgt));
              if ((dlft * drgt) <= 0.0) dlim = 0.0;
              r = dsgn * dlim;
            } else if (P.slope_type == 5) {
              if (n == 0) {
                const double dcen = uvel * dt / a.dx;
                double dlft, drgt;
                if (dcen >= 0) { dlft = 2.0 / (0.0 + dcen + 1e-10) * (qC - qL); drgt = 2.0 / (1.0 - dcen) * (qR - qC); }
                else { dlft = 2.0 / (1.0 + dcen) * (qC - qL); drgt = 2.0 / (0.0 - dcen + 1e-10) * (qR - qC); }
                const double dsgn = fsign1(dlft);
                double dlim = fmn(fabs(dlft), fabs(drgt));
                if ((dlft * drgt) <= 0.0) dlim = 0.0;
                r = dsgn * dlim;
              } else r = 0;
            } else {
              if (n == 0) { const double dlft = qC - qL, drgt = qR - qC; r = 0.5 * (dlft + drgt); }
              else r = 0;
            }
            dq[0][n] = r;
          }
        } else {
#pragma unroll
          for (int n = 0; n < NV; n++) {
            const double* qn = qc + n * PL;
            dq[0][n] = slope_lcr<NDIM, SLOPE>(qn[-1], q[n], qn[1], P);
            if (HY) dq[HY][n] = slope_lcr<NDIM, SLOPE>(qn[-QX], q[n], qn[QX], P);
            if (HZ) {
              const double qb = qring[(size_t)sm1 * NQ * PL + n * PL + qy * QX + qx];
              const double qf = qring[(size_t)sp1 * NQ * PL + n * PL + qy * QX + qx];
              dq[NDIM - 1][n] = slope_lcr<NDIM, SLOPE>(qb, q[n], qf, P);
            }
          }
        }
        // ---- trace (hydro/umuscl.f90:176/305/483): t0 = s0*dtdx*half ----
        double s0[NV];
        trace_sources<NDIM>(q, dq, rinv, s0, P);
#pragma unroll
        for (int n = 0; n < NV; n++) t0[n] = s0[n] * dtdx * 0.5;
#pragma unroll
        for (int n = 0; n < NV; n++) {
          double qm = q[n] + 0.5 * dq[0][n] + t0[n];
          if (n == 0 && qm < P.smallr) qm = q[0];
          qmx[n] = qm;
        }
        if (HY) {
#pragma unroll
          for (int n = 0; n < NV; n++) {
            double qm = q[n] + 0.5 * dq[HY][n] + t0[n];
            if (n == 0 && qm < P.smallr) qm = q[0];
            exq[n * NT + tid] = qm;
          }
        }
      }
      // left state of my -x face comes from lane-1 (a warp is one x-row)
      double qlx[NV];
#pragma unroll
      for (int n = 0; n < NV; n++) qlx[n] = __shfl_up_sync(0xffffffffu, qmx[n], 1);
      int mc = 0, mlx = 0;                     // AMRV: ok(cell) = son(cell)>0 of my cell / of the cell at lane-1
      if (AMRV) {
        if (need_tr) {
          const long long offm = cell_offset<NDIM>(g, wrap_or_clamp(cx, g.ncx, g.wrapx), HY ? wrap_or_clamp(cy, g.ncy, g.wrapy) : 0,
                                                   HZ ? wrap_or_clamp(k, g.ncz, g.wrapz) : 0);
          mc = a.refined[offm];
        }
        mlx = __shfl_up_sync(0xffffffffu, mc, 1);
        exm[AMRV ? tid : 0] = (unsigned char)mc;
      }
      __syncthreads();

      double fx[NV], fy[NV], fz[NV], ucur[NV];
      double tx[NPF], ty[NPF], tz[NPF], pcur[NPF];   // PFIX: tmp1, tmp2 of my -x, -y, -z faces; divu, enew of my cell
#pragma unroll
      for (int n = 0; n < NV; n++) { fx[n] = 0.0; fy[n] = 0.0; fz[n] = 0.0; ucur[n] = 0.0; }
#pragma unroll
      for (int n = 0; n < NPF; n++) { tx[n] = 0.0; ty[n] = 0.0; tz[n] = 0.0; pcur[n] = 0.0; }
      if (own && plane_flux) {   // set_unew: unew = uold; issued early so the latency hides under the Riemann solves
        const long long off = cell_offset<NDIM>(g, cx, cy, HZ ? k : 0);
        if (AMRV) {              // unew already holds uold + the refluxes of the finer level (godunov_fine.f90:751-792 adds to it)
#pragma unroll
          for (int n = 0; n < NV; n++) ucur[n] = a.uout[n * vstride + off];
          if (PFIX) {
#pragma unroll
            for (int n = 0; n < NPF; n++) pcur[n] = a.pfix[n * vstride + off];
          }
        } else {
#pragma unroll
          for (int n = 0; n < NV; n++) ucur[n] = __ldg(a.uin + n * vstride + off);
          if (PFIX) {            // set_unew's divu = 0, enew = e_int of uold
#pragma unroll
            for (int n = 0; n < NPF; n++) pcur[n] = a.pfix[n * vstride + off];
          }
        }
      }
      // PFIX: tmp1 = half*(qleft(ln)+qright(ln)), tmp2 = fgdnv(nvar+1) (hydro/umuscl.f90:844-850), scaled like the fluxes (:111-112)
      auto pfix_face = [&](const double* ql, const double* qr, double fe, double* t) {
        t[0] = 0.5 * (ql[1] + qr[1]);
        t[NPF - 1] = fe;
        scale_fluxes<NPF>(t, dt, a.dx, a.inv_dx, a.dx_pow2);
      };
      // ---- X faces: cmpflxm(...,2,3,4) hydro/umuscl.f90:97 ----
      if (need_fx && plane_flux) {
        double ql[NV], qr[NV], fg[NV];
        ql[0] = qlx[0]; ql[1] = qlx[1]; ql[2] = qlx[NDIM + 1];
        if (NDIM > 1) ql[3] = qlx[2];
        if (NDIM > 2) ql[4] = qlx[3];
        double qp[NV];
#pragma unroll
        for (int n = 0; n < NV; n++) qp[n] = q[n] - 0.5 * dq[0][n] + t0[n];
        if (qp[0] < P.smallr) qp[0] = q[0];
        qr[0] = qp[0]; qr[1] = qp[1]; qr[2] = qp[NDIM + 1];
        if (NDIM > 1) qr[3] = qp[2];
        if (NDIM > 2) qr[4] = qp[3];
        double fe = 0.0;
        riemann<NDIM, RIEMANN>(ql, qr, fg, P, PFIX ? &fe : nullptr);
        fx[0] = fg[0]; fx[1] = fg[1]; fx[NDIM + 1] = fg[2];
        if (NDIM > 1) fx[2] = fg[3];
        if (NDIM > 2) fx[3] = fg[4];
        scale_fluxes<NV>(fx, dt, a.dx, a.inv_dx, a.dx_pow2);
        if (PFIX) pfix_face(ql, qr, fe, tx);
        if (AMRV && (mlx | mc)) {   // reset flux along direction at refined interface :720-747
#pragma unroll
          for (int n = 0; n < NV; n++) fx[n] = 0.0;
#pragma unroll
          for (int n = 0; n < NPF; n++) tx[n] = 0.0;
        }
      }
      // ---- Y faces: cmpflxm(...,3,2,4) hydro/umuscl.f90:120 ----
      if (HY && need_fy && plane_flux) {
        double ql[NV], qr[NV], fg[NV];
        const double* e = exq + tid - BX;        // row ty-1
        ql[0] = e[0 * NT]; ql[1] = e[2 * NT]; ql[2] = e[(NDIM + 1) * NT]; ql[3] = e[1 * NT];
        if (NDIM > 2) ql[4] = e[3 * NT];
        double qp[NV];
#pragma unroll
        for (int n = 0; n < NV; n++) qp[n] = q[n] - 0.5 * dq[HY][n] + t0[n];
        if (qp[0] < P.smallr) qp[0] = q[0];
        qr[0] = qp[0]; qr[1] = qp[2]; qr[2] = qp[NDIM + 1]; qr[3] = qp[1];
        if (NDIM > 2) qr[4] = qp[3];
        double fe = 0.0;
        riemann<NDIM, RIEMANN>(ql, qr, fg, P, PFIX ? &fe : nullptr);
        fy[0] = fg[0]; fy[2] = fg[1]; fy[NDIM + 1] = fg[2]; fy[1] = fg[3];
        if (NDIM > 2) fy[3] = fg[4];
        scale_fluxes<NV>(fy, dt, a.dx, a.inv_dx, a.dx_pow2);
        if (PFIX) pfix_face(ql, qr, fe, ty);
        if (AMRV && (exm[AMRV ? tid - BX : 0] | mc)) {
#pragma unroll
          for (int n = 0; n < NV; n++) fy[n] = 0.0;
#pragma unroll
          for (int n = 0; n < NPF; n++) ty[n] = 0.0;
        }
#pragma unroll
        for (int n = 0; n < NV; n++) exf[n * NT + tid] = fy[n];
        if (PFIX) {
#pragma unroll
          for (int n = 0; n < NPF; n++) exft[n * NT + tid] = ty[n];
        }
      }
      // ---- Z faces: cmpflxm(...,4,2,3) hydro/umuscl.f90:144; left state carried from the previous plane ----
      if (HZ && own && k >= z0) {
        double ql[NV], qr[NV], fg[NV];
        const double* cq = carry + tid;          // qm_z of plane k-1
        ql[0] = cq[0 * NT]; ql[1] = cq[3 * NT]; ql[2] = cq[(NDIM + 1) * NT]; ql[3] = cq[1 * NT]; ql[4 % NV] = cq[2 * NT];
        double qp[NV];
#pragma unroll
        for (int n = 0; n < NV; n++) qp[n] = q[n] - 0.5 * dq[NDIM - 1][n] + t0[n];
        if (qp[0] < P.smallr) qp[0] = q[0];
        qr[0] = qp[0]; qr[1] = qp[3 % NV]; qr[2] = qp[NDIM + 1]; qr[3] = qp[1]; qr[4 % NV] = qp[2];
        double fe = 0.0;
        riemann<NDIM, RIEMANN>(ql, qr, fg, P, PFIX ? &fe : nullptr);
        fz[0] = fg[0]; fz[3 % NV] = fg[1]; fz[NDIM + 1] = fg[2]; fz[1] = fg[3]; fz[2] = fg[4 % NV];
        scale_fluxes<NV>(fz, dt, a.dx, a.inv_dx, a.dx_pow2);
        if (PFIX) pfix_face(ql, qr, fe, tz);
        if (AMRV && (mprev | mc)) {
#pragma unroll
          for (int n = 0; n < NV; n++) fz[n] = 0.0;
#pragma unroll
          for (int n = 0; n < NPF; n++) tz[n] = 0.0;
        }
      }
      mprev = mc;
      if (HZ && own) {
#pragma unroll
        for (int n = 0; n < NV; n++) {
          double qm = q[n] + 0.5 * dq[NDIM - 1][n] + t0[n];
          if (n == 0 && qm < P.smallr) qm = q[0];
          carry[n * NT + tid] = qm;
        }
      }
      // flux through my +x face comes from lane+1
      double fxr[NV];
#pragma unroll
      for (int n = 0; n < NV; n++) fxr[n] = __shfl_down_sync(0xffffffffu, fx[n], 1);
      double txr[NPF];
      if (PFIX) {
#pragma unroll
        for (int n = 0; n < NPF; n++) txr[n] = __shfl_down_sync(0xffffffffu, tx[n], 1);
      }
      if (!LATE) __syncthreads();

      // ---- conservative update (godfine1, hydro/godunov_fine.f90:751-792): x, then y, then z ----
      // PFIX: divu, enew accumulate tmp1, tmp2 in the same order (:775-786)
      if (own) {
        double unew_[NV], pnew[NPF];
        bool have = false;
        if (HZ) {
          if (k > z0) {   // finish plane k-1 with the z fluxes
#pragma unroll
            for (int n = 0; n < NV; n++) unew_[n] = carry[(2 * NV + n) * NT + tid] + (carry[(NV + n) * NT + tid] - fz[n]);
            if (PFIX) {
#pragma unroll
              for (int n = 0; n < NPF; n++) pnew[n] = carryt[(2 + n) * NT + tid] + (carryt[n * NT + tid] - tz[n]);
            }
            have = true;
          }
          if (k >= z0) {
#pragma unroll
            for (int n = 0; n < NV; n++) carry[(NV + n) * NT + tid] = fz[n];
            if (PFIX) {
#pragma unroll
              for (int n = 0; n < NPF; n++) carryt[n * NT + tid] = tz[n];
            }
          }
        }
        if (plane_flux && LATE) {
#pragma unroll
          for (int n = 0; n < NV; n++) {
            double u = ucur[n];
            u = u + (fx[n] - fxr[n]);
            if (HZ) { carry[(2 * NV + n) * NT + tid] = u; late_fys[n * NT + tid] = fy[n]; }
            else { late_p1[(LATE && !HZ) ? n : 0] = u; late_fy[(LATE && !HZ) ? n : 0] = fy[n]; }
          }
          late_pend = true;
        }
        if (plane_flux && !LATE) {
#pragma unroll
          for (int n = 0; n < NV; n++) {
            double u = ucur[n];
            u = u + (fx[n] - fxr[n]);
            if (HY) u = u + (fy[n] - exf[n * NT + tid + BX]);
            if (HZ) carry[(2 * NV + n) * NT + tid] = u; else unew_[n] = u;
          }
          if (PFIX) {
#pragma unroll
            for (int n = 0; n < NPF; n++) {
              double p = pcur[n];
              p = p + (tx[n] - txr[n]);
              if (HY) p = p + (ty[n] - exft[n * NT + tid + BX]);
              if (HZ) carryt[(2 + n) * NT + tid] = p; else pnew[n] = p;
            }
          }
          if (!HZ) have = true;
        }
        if (have) {
          const long long off = cell_offset<NDIM>(g, cx, cy, HZ ? k - 1 : 0);
          double gsum = -1.0;                  // no gravity term in the Courant scan
          if (GRAV && a.gsrc) {                // set_uold: add_gravity_source_terms (godunov_fine.f90:159-161); courant gg = f
            // d_old = MAX(uold(rho), smallr): the q[0] that ctoprim put into the ring for this cell, re-read from uold
            double fc[NDIM];
#pragma unroll
            for (int d = 0; d < NDIM; d++) fc[d] = __ldg(a.force + d * vstride + off);
            const double d_old = fmx(__ldg(a.uin + off), P.smallr);
            gravity_src_cell(unew_[0], unew_[1], unew_[1 + 1 % NDIM], unew_[1 + 2 % NDIM], unew_[NDIM + 1], d_old, fc[0],
                             fc[1 % NDIM], fc[2 % NDIM], NDIM, P.smallr, dt);
            gsum = 0.0;
#pragma unroll
            for (int d = 0; d < NDIM; d++) gsum = gsum + fabs(fc[d]);
          }
#pragma unroll
          for (int n = 0; n < NV; n++) a.uout[n * vstride + off] = unew_[n];   // set_uold: uold = unew
          if (PFIX) {
#pragma unroll
            for (int n = 0; n < NPF; n++) a.pfix[n * vstride + off] = pnew[n];
          }
          // fused courant_fine of the new state (hydro/courant_fine.f90:96-123)
          double ei;
          const double dtc = cmpdt_cell<NDIM>(unew_, a.dx, P, ei, gsum);
          my_dt = dtc < my_dt ? dtc : my_dt;
          my_mass += unew_[0];
          my_etot += unew_[NDIM + 1];
          my_eint += ei;
        }
      }
    }
    if (LATE && !HZ) {                         // 1-D / 2-D: the only plane is finished after one more barrier
      __syncthreads();
      if (own && late_pend) {
        double unew_[NV];
#pragma unroll
        for (int n = 0; n < NV; n++) {
          double u = late_p1[(LATE && !HZ) ? n : 0];
          if (HY) u = u + (late_fy[(LATE && !HZ) ? n : 0] - exf[n * NT + tid + BX]);
          unew_[n] = u;
        }
        const long long off = cell_offset<NDIM>(g, cx, cy, 0);
#pragma unroll
        for (int n = 0; n < NV; n++) a.uout[n * vstride + off] = unew_[n];
        double ei;
        const double dtc = cmpdt_cell<NDIM>(unew_, a.dx, P, ei);
        my_dt = dtc < my_dt ? dtc : my_dt;
        my_mass += unew_[0];
        my_etot += unew_[NDIM + 1];
        my_eint += ei;
      }
    }
  }

  // ---- warp-shuffle + shared reduction of the Courant scan partials ----
  my_dt = warp_min(my_dt);
  my_mass = warp_sum(my_mass); my_etot = warp_sum(my_etot); my_eint = warp_sum(my_eint);
  const int w = tid >> 5, l = tid & 31;
  __syncthreads();
  if (l == 0) { red[0][w] = my_dt; red[1][w] = my_mass; red[2][w] = my_etot; red[3][w] = my_eint; }
  __syncthreads();
  if (w == 0) {
    double v0 = 1e300, v1 = 0, v2 = 0, v3 = 0;
    for (int i = l; i < NT / 32; i += 32) { v0 = red[0][i] < v0 ? red[0][i] : v0; v1 += red[1][i]; v2 += red[2][i]; v3 += red[3][i]; }
    v0 = warp_min(v0); v1 = warp_sum(v1); v2 = warp_sum(v2); v3 = warp_sum(v3);
    if (l == 0 && a.part) {
      const size_t nb = a.part_stride ? (size_t)a.part_stride : (size_t)gridDim.x, c0 = (size_t)a.part_off + blockIdx.x;
      a.part[0 * nb + c0] = v0; a.part[1 * nb + c0] = v1;
      a.part[2 * nb + c0] = v2; a.part[3 * nb + c0] = v3;
    }
  }
}

// ---- pressure_fix passes of set_unew / set_uold on a dense level store: one thread per owned cell, divu / enew in the
// PFIX store [2][2^ndim][nslot].  The per-cell arithmetic is the one of the AMR list kernels (hydro_device.cuh).  dt_dev != NULL:
// the time step is read from device memory (rgpu_level_steps), otherwise dt is used.
template <int NDIM>
__device__ __forceinline__ bool dense_owned_cell(const DenseGeom& g, long long i, long long& off) {
  const long long nx = g.ox1 - g.ox0, ny = NDIM > 1 ? g.oy1 - g.oy0 : 1, nz = NDIM > 2 ? g.oz1 - g.oz0 : 1;
  if (i >= nx * ny * nz) return false;
  const int x = g.ox0 + (int)(i % nx), y = NDIM > 1 ? g.oy0 + (int)((i / nx) % ny) : 0, z = NDIM > 2 ? g.oz0 + (int)(i / (nx * ny)) : 0;
  off = cell_offset<NDIM>(g, x, y, z);
  return true;
}
// set_unew (hydro/godunov_fine.f90:71-90): divu = 0, enew = E - e_kin of uold
template <int NDIM>
__global__ void dense_pfix_init_kernel(const double* __restrict__ uold, double* __restrict__ pfix, DenseGeom g, double smallr) {
  long long off;
  if (!dense_owned_cell<NDIM>(g, blockIdx.x * (long long)blockDim.x + threadIdx.x, off)) return;
  const size_t vs = (size_t)(1 << NDIM) * g.nslot;
  pfix_init_cell(uold + off, vs, pfix + off, pfix + vs + off, NDIM, smallr);
}
// add_pdv_source_terms (:294-437): enew -= (gamma-1) e_old div(u) dt from the face neighbours in uold.  On a full level every face
// neighbour of an owned cell is a cell of the box at distance dx -- owned, a ghost or boundary oct of the shell, or the periodic
// image -- so the reference's fallback to the father cell at 1.5 dx never applies (rgpu_bind_level refuses a shell with a hole)
template <int NDIM>
__global__ void dense_pdv_kernel(const double* __restrict__ uold, double* __restrict__ pfix, DenseGeom g, double gamma, double smallr,
                                 double dx, double dt, const double* __restrict__ dt_dev) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  long long off;
  if (!dense_owned_cell<NDIM>(g, i, off)) return;
  const long long nx = g.ox1 - g.ox0, ny = NDIM > 1 ? g.oy1 - g.oy0 : 1;
  const int c[3] = {g.ox0 + (int)(i % nx), NDIM > 1 ? g.oy0 + (int)((i / nx) % ny) : 0, NDIM > 2 ? g.oz0 + (int)(i / (nx * ny)) : 0};
  const int n[3] = {g.ncx, g.ncy, g.ncz}, w[3] = {g.wrapx, g.wrapy, g.wrapz};
  const size_t vs = (size_t)(1 << NDIM) * g.nslot;
  auto uo = [&](long long o, int k) -> double { return uold[k * vs + o]; };
  double divu_loc = 0.0;
#pragma unroll
  for (int d = 0; d < NDIM; d++) {
    int l[3] = {c[0], c[1], c[2]}, r[3] = {c[0], c[1], c[2]};
    l[d] = wrap_or_clamp(c[d] - 1, n[d], w[d]);
    r[d] = wrap_or_clamp(c[d] + 1, n[d], w[d]);
    const long long ol = cell_offset<NDIM>(g, l[0], l[1], l[2]), orr = cell_offset<NDIM>(g, r[0], r[1], r[2]);
    divu_loc = pdv_face_term(divu_loc, uo, ol, orr, d, dx, dx, smallr);
  }
  pfix[vs + off] = pdv_cell(pfix[vs + off], divu_loc, uo, off, NDIM, gamma, smallr, dt_dev ? *dt_dev : dt);
}
// set_uold's energy switch (:203-227) on the new state, in place
template <int NDIM>
__global__ void dense_pfix_switch_kernel(double* __restrict__ uold, const double* __restrict__ pfix, DenseGeom g, double smallr,
                                         double beta_fix, double dx, double dt, const double* __restrict__ dt_dev) {
  long long off;
  if (!dense_owned_cell<NDIM>(g, blockIdx.x * (long long)blockDim.x + threadIdx.x, off)) return;
  const size_t vs = (size_t)(1 << NDIM) * g.nslot;
  pfix_switch_cell(uold + off, vs, pfix + off, pfix + vs + off, NDIM, smallr, beta_fix, dx, dt_dev ? *dt_dev : dt);
}

// tile shapes (a warp = one x-row of 32 cells): BX = 32, BY = tile height in rows (threads = 32*BY).
// 3-D default: 12 rows (384 threads, one CTA per SM); not re-tuned on H100: RGPU_BY3=8|12|16 overrides at bind time
// (profiles/tune_sweep.py times the choices).
__host__ __device__ constexpr int tile_by_default(int ndim, int riemann) {
  return ndim == 1 ? 1 : ndim == 2 ? 8 : 12;   // the same for every solver (riemann unused)
}

#ifndef RGPU_HOST_NUMERICS   // kernel launches: product build only
template <int NDIM, int RIEMANN, int SLOPE, int BY>
cudaError_t launch_sweep_dense_sb(const SweepArgs& a, int nblocks, cudaStream_t st) {
  constexpr int BX = 32;
  constexpr size_t smem = sizeof(double) * SweepSmem<NDIM, BX, BY>::doubles;
  auto kern = sweep_dense_kernel<NDIM, RIEMANN, SLOPE, BX, BY>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  kern<<<nblocks, dim3(BX, BY, 1), smem, st>>>(a);
  return cudaGetLastError();
}
template <int NDIM, int RIEMANN, int SLOPE>
cudaError_t launch_sweep_dense_s(const SweepArgs& a, int nblocks, cudaStream_t st, int by) {
  if (NDIM == 1) return launch_sweep_dense_sb<NDIM, RIEMANN, SLOPE, 1>(a, nblocks, st);
  if (NDIM == 2) return launch_sweep_dense_sb<NDIM, RIEMANN, SLOPE, (NDIM == 2 ? 8 : 1)>(a, nblocks, st);
  if (by == 8) return launch_sweep_dense_sb<NDIM, RIEMANN, SLOPE, (NDIM == 3 ? 8 : 1)>(a, nblocks, st);
  if (by == 16) return launch_sweep_dense_sb<NDIM, RIEMANN, SLOPE, (NDIM == 3 ? 16 : 1)>(a, nblocks, st);
  return launch_sweep_dense_sb<NDIM, RIEMANN, SLOPE, (NDIM == 3 ? 12 : 1)>(a, nblocks, st);
}
// slope_type 1 (minmod) and 2 (moncen) are compiled in; every other limiter goes through the runtime switch
// AMR variant: one instantiation per solver (runtime slope switch, 12-row tiles), 3-D only
template <int NDIM, int RIEMANN>
cudaError_t launch_sweep_dense_amr(const SweepArgs& a, int nblocks, cudaStream_t st) {
  constexpr int BX = 32, BY = (NDIM == 3 ? 12 : (NDIM == 2 ? 8 : 1));
  constexpr size_t smem = sizeof(double) * SweepSmem<NDIM, BX, BY>::doubles;
  auto kern = sweep_dense_kernel<NDIM, RIEMANN, -1, BX, BY, true>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  kern<<<nblocks, dim3(BX, BY, 1), smem, st>>>(a);
  return cudaGetLastError();
}
template <int NDIM, int RIEMANN>
cudaError_t launch_sweep_dense(const SweepArgs& a, int nblocks, cudaStream_t st, int by) {
  if (a.P.slope_type == 1) return launch_sweep_dense_s<NDIM, RIEMANN, 1>(a, nblocks, st, by);
  if (a.P.slope_type == 2) return launch_sweep_dense_s<NDIM, RIEMANN, 2>(a, nblocks, st, by);
  return launch_sweep_dense_s<NDIM, RIEMANN, -1>(a, nblocks, st, by);
}
// poisson (GRAV): one instantiation per dimension and solver with the runtime slope switch and the default tile height, plus
// the 3-D AMR variant (sweep_grav_inst_*.cu)
template <int NDIM, int RIEMANN, bool AMRV>
cudaError_t launch_sweep_dense_grav(const SweepArgs& a, int nblocks, cudaStream_t st) {
  static_assert(!AMRV || NDIM == 3, "the AMR variant is 3-D only");
  constexpr int BX = 32, BY = tile_by_default(NDIM, RIEMANN);
  constexpr size_t smem = sizeof(double) * SweepSmem<NDIM, BX, BY, true>::doubles;
  auto kern = sweep_dense_kernel<NDIM, RIEMANN, -1, BX, BY, AMRV, false, true>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  kern<<<nblocks, dim3(BX, BY, 1), smem, st>>>(a);
  return cudaGetLastError();
}
// pressure_fix (PFIX): the 3-D AMR variant, one instantiation per solver without and with poisson (sweep_pfix_inst_3d_*.cu),
// runtime slope switch and 12-row tiles
template <int RIEMANN, bool GRAV>
cudaError_t launch_sweep_dense_pfix(const SweepArgs& a, int nblocks, cudaStream_t st) {
  constexpr int BX = 32, BY = tile_by_default(3, RIEMANN);
  constexpr size_t smem = sizeof(double) * SweepSmem<3, BX, BY, GRAV, true>::doubles;
  auto kern = sweep_dense_kernel<3, RIEMANN, -1, BX, BY, true, false, GRAV, true>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  kern<<<nblocks, dim3(BX, BY, 1), smem, st>>>(a);
  return cudaGetLastError();
}
// pressure_fix (PFIX) outside AMR mode: the plain form without poisson, one instantiation per dimension and solver with the
// runtime slope switch and the default tile height (sweep_pfix_inst_plain_*.cu)
template <int NDIM, int RIEMANN>
cudaError_t launch_sweep_dense_pfix_plain(const SweepArgs& a, int nblocks, cudaStream_t st) {
  constexpr int BX = 32, BY = tile_by_default(NDIM, RIEMANN);
  constexpr size_t smem = sizeof(double) * SweepSmem<NDIM, BX, BY, false, true>::doubles;
  auto kern = sweep_dense_kernel<NDIM, RIEMANN, -1, BX, BY, false, false, false, true>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  kern<<<nblocks, dim3(BX, BY, 1), smem, st>>>(a);
  return cudaGetLastError();
}
#endif

}  // namespace rgpu
