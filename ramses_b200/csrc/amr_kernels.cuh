// amr_kernels.cuh -- oct-batch kernels for levels that are NOT dense boxes (levelmin < levelmax runs).
//
// In AMR mode the device mirrors the reference's own arrays: son(1:ncell), father(1:ngridmax),
// nbor(1:ngridmax,1:2*ndim) (amr/amr_commons.f90:68-79) and uold/unew(1:ncell,1:nvar) in the Fortran
// layout (hydro/hydro_commons.f90:4), so every index below is the reference's cell / oct index
// (icell = ncoarse + (ind-1)*ngridmax + igrid).  One group of 64 threads reproduces godfine1
// (hydro/godunov_fine.f90:486-911) for one oct:
//   get3cubefather (amr/nbors_utils.f90:5) -> 6^ndim patch gather, with interpol_hydro
//   (hydro/interpol_hydro.f90:268) prolongation of missing neighbour octs from the coarser level ->
//   ctoprim / uslope / trace / cmpflxm+Riemann on the patch (same device functions as the dense sweep) ->
//   flux masking at refined faces (:720-747) -> update of the oct's own cells (:751-792); the fluxes through
//   the oct's outer faces are stored, and a second kernel refluxes them into the coarser level (:798-908) in the
//   reference's accumulation order (deterministic, no atomics).
#pragma once
#include "hydro_device.cuh"

namespace rgpu {

struct AmrTree {
  const int* son;      // 1-based: son[icell]
  const int* father;   // 1-based: father[igrid]
  const int* nbor;     // nbor[(j-1)*ngridmax + igrid-1], j = 1..2*ndim
  int ncoarse, ngridmax, nx, ny, nz;
  long long ncell;
};

__device__ __forceinline__ int amr_nbor(const AmrTree& t, int igrid, int j) { return t.nbor[(size_t)(j - 1) * t.ngridmax + igrid - 1]; }
__device__ __forceinline__ int amr_cell(const AmrTree& t, int ind0, int igrid) { return t.ncoarse + ind0 * t.ngridmax + igrid; }

// getnborfather (amr/nbors_utils.f90:404-525) for one cell of level ilevel-1
template <int NDIM>
__device__ void amr_getnborfather(const AmrTree& t, int ind_cell, int ilevel, int* fa) {
  fa[0] = ind_cell;
  if (ilevel == 1) {
    const int nn[3] = {t.nx, t.ny, t.nz};
    const int s1[3] = {1, t.nx, t.nx * t.ny};
    int ix[3];
    ix[2] = (ind_cell - 1) / (t.nx * t.ny);
    ix[1] = (ind_cell - 1 - ix[2] * t.nx * t.ny) / t.nx;
    ix[0] = ind_cell - 1 - ix[1] * t.nx - ix[2] * t.nx * t.ny;
#pragma unroll
    for (int d = 0; d < NDIM; d++) {
      fa[2 * d + 1] = ix[d] > 0 ? ind_cell - s1[d] : ind_cell + (nn[d] - 1) * s1[d];
      fa[2 * d + 2] = ix[d] < nn[d] - 1 ? ind_cell + s1[d] : ind_cell - (nn[d] - 1) * s1[d];
    }
    return;
  }
  const int pos = (ind_cell - t.ncoarse - 1) / t.ngridmax;
  const int gf = ind_cell - t.ncoarse - pos * t.ngridmax;
#pragma unroll
  for (int d = 0; d < NDIM; d++)
#pragma unroll
    for (int s = 0; s < 2; s++) {
      const int j = 2 * d + s + 1;
      const int bit = (pos >> d) & 1, pos2 = pos ^ (1 << d);
      const int nb = amr_nbor(t, gf, j);
      const int g = (bit != s) ? gf : t.son[nb];
      fa[j] = g > 0 ? amr_cell(t, pos2, g) : nb;
    }
}

// interpol_hydro (hydro/interpol_hydro.f90:268-444, interpol_var = 0) for ONE variable: a[0..2*ndim] -> u2[2^ndim]
template <int NDIM>
__device__ void amr_interpol_var(const double* a, int interpol_type, double* u2) {
  constexpr int T = 1 << NDIM, TW = 2 * NDIM;
  double w[3] = {0, 0, 0};
  if (interpol_type == 1) {            // compute_limiter_minmod :449
#pragma unroll
    for (int d = 0; d < NDIM; d++) {
      const double dl = 0.5 * (a[2 * d + 2] - a[0]), dr = 0.5 * (a[0] - a[2 * d + 1]);
      double mm;
      if (dl * dr <= 0.0) mm = 0; else mm = fmn(fabs(dl), fabs(dr)) * dl / fabs(dl);
      w[d] = mm;
    }
  } else if (interpol_type == 2) {     // compute_limiter_central :481
    double ac[T];
#pragma unroll
    for (int d = 0; d < NDIM; d++) w[d] = 0.25 * (a[2 * d + 2] - a[2 * d + 1]);
#pragma unroll
    for (int i = 0; i < T; i++) ac[i] = a[0];
#pragma unroll
    for (int d = 0; d < NDIM; d++)
#pragma unroll
      for (int i = 0; i < T; i++) ac[i] = ac[i] + 2.0 * w[d] * ((double)((i >> d) & 1) - 0.5);
    double corner = ac[0], kernel = a[1];
#pragma unroll
    for (int j = 1; j < T; j++) corner = fmx(corner, ac[j]);
#pragma unroll
    for (int j = 2; j <= TW; j++) kernel = fmx(kernel, a[j]);
    double dk = a[0] - kernel, dc = a[0] - corner, maxl = 0.0, minl = 0.0;
    if (dk * dc > 0.0) maxl = fmn(1.0, dk / dc);
    corner = ac[0]; kernel = a[1];
#pragma unroll
    for (int j = 1; j < T; j++) corner = fmn(corner, ac[j]);
#pragma unroll
    for (int j = 2; j <= TW; j++) kernel = fmn(kernel, a[j]);
    dk = a[0] - kernel; dc = a[0] - corner;
    if (dk * dc > 0.0) minl = fmn(1.0, dk / dc);
    const double lim = fmn(minl, maxl);
#pragma unroll
    for (int d = 0; d < NDIM; d++) w[d] = w[d] * lim;
  } else if (interpol_type == 3) {     // compute_central :618
#pragma unroll
    for (int d = 0; d < NDIM; d++) w[d] = 0.25 * (a[2 * d + 2] - a[2 * d + 1]);
  }
#pragma unroll
  for (int i = 0; i < T; i++) {
    double v = a[0];
#pragma unroll
    for (int d = 0; d < NDIM; d++) v = v + w[d] * ((double)((i >> d) & 1) - 0.5);
    u2[i] = v;
  }
}

// interpol_hydro (hydro/interpol_hydro.f90:268-444) for ONE father cell and ALL variables: u1[(2*ndim+1)][nvar] (cell, then its
// 2*ndim neighbours) -> u2[2^ndim][nvar].  interpol_var 0: conservative variables (rho, rho u, E); 1: (rho, rho u, rho eps)
// :318-345; 2: (rho, u, rho eps) with the momentum correction :393-415.  interpol_type 0..3 as amr_interpol_var; 4 = type 3 for
// the velocities and type 2 for everything else (:357-366; only meaningful with interpol_var = 2).  NVX = nvar (compile time).
template <int NDIM, int NVX>
__device__ void amr_interpol_hydro(double (*u1)[NVX], int interpol_type, int interpol_var, double smallr, double (*u2)[NVX]) {
  constexpr int T = 1 << NDIM, TW = 2 * NDIM;
  const double oneover_twotondim = 1.0 / (double)T;
  if (interpol_var == 1 || interpol_var == 2) {
    for (int j = 0; j <= TW; j++) {
      double ekin = 0.0;
#pragma unroll
      for (int d = 1; d <= NDIM; d++) ekin = ekin + 0.5 * (u1[j][d] * u1[j][d]) / fmx(u1[j][0], smallr);
      u1[j][NDIM + 1] = u1[j][NDIM + 1] - ekin - 0.0;
      if (interpol_var == 2) {
#pragma unroll
        for (int d = 1; d <= NDIM; d++) u1[j][d] = u1[j][d] / fmx(u1[j][0], smallr);
      }
    }
  }
#pragma unroll 1
  for (int iv = 0; iv < NVX; iv++) {
    double a[7], v2[T];
    for (int j = 0; j <= TW; j++) a[j] = u1[j][iv];
    int tt = interpol_type;
    if (interpol_type == 4) tt = (iv >= 1 && iv <= NDIM) ? 3 : 2;
    amr_interpol_var<NDIM>(a, tt, v2);
#pragma unroll
    for (int is = 0; is < T; is++) u2[is][iv] = v2[is];
  }
  if (interpol_var == 1 || interpol_var == 2) {
    if (interpol_var == 2) {
      for (int is = 0; is < T; is++)
#pragma unroll
        for (int d = 1; d <= NDIM; d++) u2[is][d] = u2[is][d] * u2[is][0];
#pragma unroll
      for (int d = 1; d <= NDIM; d++) {
        double mom = 0.0;
        for (int is = 0; is < T; is++) mom = mom + u2[is][d] * oneover_twotondim;
        mom = mom - u1[0][d] * u1[0][0];
        for (int is = 0; is < T; is++) u2[is][d] = u2[is][d] - mom;
      }
    }
    for (int is = 0; is < T; is++) {
      double ekin = 0.0;
#pragma unroll
      for (int d = 1; d <= NDIM; d++) ekin = ekin + 0.5 * (u2[is][d] * u2[is][d]) / fmx(u2[is][0], smallr);
      u2[is][NDIM + 1] = u2[is][NDIM + 1] + ekin + 0.0;
    }
  }
}

// get3cubefather (amr/nbors_utils.f90:5-194, get3cubepos :199): the 3^ndim father cells around the father cell of an oct
template <int NDIM>
__device__ __forceinline__ void amr_get3cubefather(const AmrTree& t, int igrid, int ilevel, int* nfc /*[3^ndim]*/, int* ng /*[8]*/) {
  constexpr int N3 = (NDIM == 1) ? 3 : (NDIM == 2 ? 9 : 27);
  constexpr int HY = NDIM > 1, HZ = NDIM > 2;

    const int fc = t.father[igrid];
    if (ilevel == 1) {
      const int nxny = t.nx * t.ny;
      const int iz = (fc - 1) / nxny, iy = (fc - 1 - iz * nxny) / t.nx, ix = fc - 1 - iy * t.nx - iz * nxny;
      for (int j = 0; j < N3; j++) {
        int o[3] = {j % 3 - 1, (j / 3) % 3 - 1, (j / 9) % 3 - 1};
        int iix = ix + o[0], iiy = iy, iiz = iz;
        if (iix < 0) iix = t.nx - 1; if (iix > t.nx - 1) iix = 0;
        if (NDIM > 1) { iiy = iy + o[1]; if (iiy < 0) iiy = t.ny - 1; if (iiy > t.ny - 1) iiy = 0; }
        if (NDIM > 2) { iiz = iz + o[2]; if (iiz < 0) iiz = t.nz - 1; if (iiz > t.nz - 1) iiz = 0; }
        nfc[j] = 1 + iix + iiy * t.nx + iiz * nxny;
      }
    } else {
      const int pos = (fc - t.ncoarse - 1) / t.ngridmax;
      const int gf = fc - t.ncoarse - pos * t.ngridmax;
      const int dirx = (pos & 1) ? 2 : 1, diry = ((pos >> 1) & 1) ? 4 : 3, dirz = ((pos >> 2) & 1) ? 6 : 5;
      for (int kk = 0; kk <= HZ; kk++) {
        int g1 = gf;
        if (kk > 0 && gf > 0) g1 = t.son[amr_nbor(t, gf, dirz)];
        for (int jj = 0; jj <= HY; jj++) {
          int g2 = g1;
          if (jj > 0 && g1 > 0) g2 = t.son[amr_nbor(t, g1, diry)];
          for (int ii = 0; ii <= 1; ii++) {
            int g3 = g2;
            if (ii > 0 && g2 > 0) g3 = t.son[amr_nbor(t, g2, dirx)];
            ng[ii + 2 * jj + 4 * kk] = g3;
          }
        }
      }
      const int c[3] = {pos & 1, (pos >> 1) & 1, (pos >> 2) & 1};
      for (int j = 0; j < N3; j++) {
        const int o[3] = {j % 3 - 1, (j / 3) % 3 - 1, (j / 9) % 3 - 1};
        int gi = 0, cp = 0;
        for (int d = 0; d < NDIM; d++) {
          const int tt = c[d] + o[d];
          gi += ((tt < 0 || tt > 1) ? 1 : 0) << d;
          cp += (tt & 1) << d;
        }
        const int g = ng[gi];
        nfc[j] = g > 0 ? amr_cell(t, cp, g) : 0;
      }
    }
}

struct AmrSweepArgs {
  AmrTree t;
  const int* active;      // active(ilevel)%igrid
  int nact, ilevel;
  const double* uold;     // [nvar][ncell]
  double* unew;
  double* rflux;          // [nact][2*ndim sides][2^(ndim-1) faces][nvar]: scaled, masked fluxes through the oct's outer faces
  Phys P;
  double dt, dx, inv_dx;
  int dx_pow2, interpol_type, interpol_var;
  double difmag;          // hydro_parameters.f90:81
  int nps;                // passive scalars: nvar - (ndim+2)
  // patch mode: the level's own cells are updated by the dense kernel; this launch only evaluates the scaled, masked fluxes
  // through the outer faces of the octs at the surface of the patch (coarse refluxing)
  int flux_only;
  const int* rflux_index; // list position -> oct index of rflux (NULL: identity)
  const double* dt_dev;   // device-resident dtnew(ilevel) (rgpu_amr_steps); NULL: use dt
  // source terms (SRC instantiation): poisson -- f[ndim][ncell], the acceleration of poisson_commons (NULL: none);
  // pressure_fix -- divu and enew are columns nvar and nvar+1 of unew (rgpu_api.cu), their face "fluxes" tmp(:,1:2) ride
  // behind the nvar conservative fluxes in rflux, so the update, the coarse reflux and the reverse exchange treat them like
  // two more variables (hydro/godunov_fine.f90:737-745,:773-786,:830-851,:882-903)
  const double* force;
  int pfix;
  int nvr;                // entries per face in rflux: nvar (+2 with pressure_fix)
};

constexpr int AMR_TPO = 64;   // threads per oct
constexpr int AMR_OPB = 1;    // octs per block (26 KB of static shared memory per oct in 3-D)

// DIF: artificial diffusion difmag>0 (cmpdivu hydro/uplmde.f90:702 + consup :769, called from unsplit hydro/umuscl.f90:160-168)
// NPS: passive scalars (NVAR = NDIM+2+NPS): q = u/rho in ctoprim (umuscl.f90:948-961), advected in trace (:680-704), carried
// through cmpflxm like the transverse velocities (:781-789,:835-842), every solver upwinds them with the mass flux
// SRC: gravity predictor (gloc gather :637-647, ctoprim umuscl.f90:932-938) and/or pressure_fix (tmp1 = face velocity,
// tmp2 = internal-energy flux, cmpflxm umuscl.f90:844-850) -- selected at run time by a.force / a.pfix
template <int NDIM, int RIEMANN, bool DIF, int NPS = 0, bool SRC = false>
__global__ void __launch_bounds__(AMR_TPO* AMR_OPB) amr_godfine_kernel(const AmrSweepArgs a) {
  constexpr int NV = NDIM + 2 + NPS, NH = NDIM + 2, T = 1 << NDIM, TW = 2 * NDIM;
  constexpr int N3 = (NDIM == 1) ? 3 : (NDIM == 2 ? 9 : 27);
  constexpr int HY = NDIM > 1, HZ = NDIM > 2;
  constexpr int PJ = HY ? 6 : 1, PK = HZ ? 6 : 1;          // patch extents (i: 6)
  constexpr int NP = 6 * PJ * PK;                          // patch cells
  constexpr int TJ = HY ? 4 : 1, TK = HZ ? 4 : 1;          // trace region 0..3
  constexpr int NTR = 4 * TJ * TK;
  constexpr int FJ = HY ? 2 : 1, FK = HZ ? 2 : 1;          // faces per direction: 3 * 2^(ndim-1)
  constexpr int NF = 3 * FJ * FK;
  constexpr int NSF = FJ * FK;                             // faces per side
  struct Sm {
    double q[NV][NP];           // uloc, then primitive variables
    unsigned char ok[NP];
    double qm[NDIM][NV][NTR], qp[NDIM][NV][NTR];
    double flux[NDIM][NV][NF];
    int nfc[27], gnb[27], ng[8];
    double uc[DIF ? NV : 1][DIF ? NP : 1];   // conservative patch (consup needs uin next to the primitives)
    double div[DIF ? 27 : 1];                // velocity divergence on the 3^ndim vertex lattice if1:if2 x jf1:jf2 x kf1:kf2
    double g[SRC ? NDIM : 1][SRC ? NP : 1];  // gloc
    double tmp[SRC ? NDIM : 1][2][SRC ? NF : 1];
  };
  __shared__ Sm sm_[AMR_OPB];
  const int grp = threadIdx.x / AMR_TPO, tl = threadIdx.x % AMR_TPO;
  const int io = blockIdx.x * AMR_OPB + grp;
  const bool live = io < a.nact;
  Sm& s = sm_[grp];
  const AmrTree& t = a.t;
  const Phys& P = a.P;
  const size_t NC = (size_t)t.ncell;
  const int igrid = live ? a.active[io] : 0;
  auto UO = [&](int icell, int iv) -> double { return a.uold[(size_t)iv * NC + icell - 1]; };

  // ---- get3cubefather (amr/nbors_utils.f90:5-194, get3cubepos :199) ----
  if (live && tl == 0) {
    amr_get3cubefather<NDIM>(t, igrid, a.ilevel, s.nfc, s.ng);
    for (int j = 0; j < N3; j++) s.gnb[j] = s.nfc[j] > 0 ? t.son[s.nfc[j]] : 0;
  }
  __syncthreads();

  // ---- gather the 6^ndim patch (hydro/godunov_fine.f90:562-675) ----
  if (live) {
    // existing neighbour octs: straight copy
    for (int e = tl; e < N3 * T; e += AMR_TPO) {
      const int jf = e / T, is = e % T;
      const int g = s.gnb[jf];
      if (g <= 0) continue;
      const int i1 = jf % 3, j1 = (jf / 3) % 3, k1 = jf / 9;
      const int i3 = 1 + 2 * (i1 - 1) + (is & 1), j3 = HY ? 1 + 2 * (j1 - 1) + ((is >> 1) & 1) : 1, k3 = HZ ? 1 + 2 * (k1 - 1) + ((is >> 2) & 1) : 1;
      const int pc = (i3 + 1) + 6 * ((HY ? j3 + 1 : 0) + PJ * (HZ ? k3 + 1 : 0));
      const int ic = amr_cell(t, is, g);
#pragma unroll
      for (int n = 0; n < NV; n++) s.q[n][pc] = UO(ic, n);
      s.ok[pc] = t.son[ic] > 0;
      if (SRC) {
#pragma unroll
        for (int d = 0; d < NDIM; d++) s.g[SRC ? d : 0][SRC ? pc : 0] = a.force ? a.force[(size_t)d * NC + ic - 1] : 0.0;
      }
    }
    if (SRC)   // buffer cells: straight injection of the father cell's acceleration (:642-646)
      for (int e = tl; e < N3 * T; e += AMR_TPO) {
        const int jf = e / T, is = e % T;
        if (s.gnb[jf] > 0) continue;
        const int i1 = jf % 3, j1 = (jf / 3) % 3, k1 = jf / 9;
        const int i3 = 1 + 2 * (i1 - 1) + (is & 1), j3 = HY ? 1 + 2 * (j1 - 1) + ((is >> 1) & 1) : 1, k3 = HZ ? 1 + 2 * (k1 - 1) + ((is >> 2) & 1) : 1;
        const int pc = (i3 + 1) + 6 * ((HY ? j3 + 1 : 0) + PJ * (HZ ? k3 + 1 : 0));
#pragma unroll
        for (int d = 0; d < NDIM; d++) s.g[SRC ? d : 0][SRC ? pc : 0] = (a.force && s.nfc[jf] > 0) ? a.force[(size_t)d * NC + s.nfc[jf] - 1] : 0.0;
      }
    // missing neighbour octs: interpol_hydro from the coarser level.  interpol_var 1, 2 and interpol_type 4 couple the
    // variables (internal energy / velocities): one thread per father cell interpolates the whole state
    if (a.interpol_var != 0 || a.interpol_type == 4) {
      for (int jf = tl; jf < N3; jf += AMR_TPO) {
        if (s.gnb[jf] > 0) continue;
        int fa[7];
        amr_getnborfather<NDIM>(t, s.nfc[jf], a.ilevel, fa);
        double u1[7][NV], u2[T][NV];
        for (int j = 0; j <= TW; j++)
#pragma unroll
          for (int n = 0; n < NV; n++) u1[j][n] = UO(fa[j], n);
        amr_interpol_hydro<NDIM, NV>(u1, a.interpol_type, a.interpol_var, P.smallr, u2);
        const int i1 = jf % 3, j1 = (jf / 3) % 3, k1 = jf / 9;
        for (int is = 0; is < T; is++) {
          const int i3 = 1 + 2 * (i1 - 1) + (is & 1), j3 = HY ? 1 + 2 * (j1 - 1) + ((is >> 1) & 1) : 1, k3 = HZ ? 1 + 2 * (k1 - 1) + ((is >> 2) & 1) : 1;
          const int pc = (i3 + 1) + 6 * ((HY ? j3 + 1 : 0) + PJ * (HZ ? k3 + 1 : 0));
#pragma unroll
          for (int n = 0; n < NV; n++) s.q[n][pc] = u2[is][n];
          s.ok[pc] = 0;
        }
      }
    } else
    for (int e = tl; e < N3 * NV; e += AMR_TPO) {
      const int jf = e / NV, n = e % NV;
      if (s.gnb[jf] > 0) continue;
      int fa[7];
      amr_getnborfather<NDIM>(t, s.nfc[jf], a.ilevel, fa);
      double av[7], u2[T];
#pragma unroll
      for (int j = 0; j <= TW; j++) av[j] = UO(fa[j], n);
      amr_interpol_var<NDIM>(av, a.interpol_type, u2);
      const int i1 = jf % 3, j1 = (jf / 3) % 3, k1 = jf / 9;
#pragma unroll
      for (int is = 0; is < T; is++) {
        const int i3 = 1 + 2 * (i1 - 1) + (is & 1), j3 = HY ? 1 + 2 * (j1 - 1) + ((is >> 1) & 1) : 1, k3 = HZ ? 1 + 2 * (k1 - 1) + ((is >> 2) & 1) : 1;
        const int pc = (i3 + 1) + 6 * ((HY ? j3 + 1 : 0) + PJ * (HZ ? k3 + 1 : 0));
        s.q[n][pc] = u2[is];
        if (n == 0) s.ok[pc] = 0;
      }
    }
  }
  __syncthreads();
  const double dt_ = a.dt_dev ? *a.dt_dev : a.dt;
  // ---- ctoprim on the whole patch (hydro/umuscl.f90:861) ----
  if (live)
    for (int pc = tl; pc < NP; pc += AMR_TPO) {
      double u[NV], q[NV];
#pragma unroll
      for (int n = 0; n < NV; n++) u[n] = s.q[n][pc];
      if (DIF) {
#pragma unroll
        for (int n = 0; n < NV; n++) s.uc[DIF ? n : 0][DIF ? pc : 0] = u[n];
      }
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
      if (SRC) {   // gravity predictor :932-938
        const double dtxhalf = dt_ * 0.5;
        q[1] = q[1] + s.g[0][SRC ? pc : 0] * dtxhalf;
        if (NDIM > 1) q[2] = q[2] + s.g[SRC ? 1 % NDIM : 0][SRC ? pc : 0] * dtxhalf;
        if (NDIM > 2) q[3] = q[3] + s.g[SRC ? 2 % NDIM : 0][SRC ? pc : 0] * dtxhalf;
      } else {
        q[1] = q[1] + 0.0;
        if (NDIM > 1) q[2] = q[2] + 0.0;
        if (NDIM > 2) q[3] = q[3] + 0.0;
      }
#pragma unroll
      for (int n = NH; n < NV; n++) q[n] = u[n] * oneoverrho;
#pragma unroll
      for (int n = 0; n < NV; n++) s.q[n][pc] = q[n];
    }
  __syncthreads();
  if (DIF && live) {   // cmpdivu :702-764 on the vertices (i,j,k) = low corner of patch cell (i,j,k), i,j,k = 1..3
    constexpr int VJ = HY ? 3 : 1, VK = HZ ? 3 : 1;
    double hp = 1.0;
    for (int d = 1; d < NDIM; d++) hp = hp * 0.5;       // half**(ndim-1)
    const double factorx = hp / a.dx, factory = factorx, factorz = factorx;
    for (int e = tl; e < 3 * VJ * VK; e += AMR_TPO) {
      const int i = 1 + e % 3, j = HY ? 1 + (e / 3) % 3 : 1, k = HZ ? 1 + e / 9 : 1;
      auto Q = [&](int ii, int jj, int kk, int n) -> double { return s.q[n][(ii + 1) + 6 * ((HY ? jj + 1 : 0) + PJ * (HZ ? kk + 1 : 0))]; };
      double ux = 0.0, vy = 0.0, wz = 0.0;
      ux = ux + factorx * (Q(i, j, k, 1) - Q(i - 1, j, k, 1));
      if (NDIM > 1) {
        ux = ux + factorx * (Q(i, j - 1, k, 1) - Q(i - 1, j - 1, k, 1));
        vy = vy + factory * (Q(i, j, k, 2 % NV) - Q(i, j - 1, k, 2 % NV) + Q(i - 1, j, k, 2 % NV) - Q(i - 1, j - 1, k, 2 % NV));
      }
      if (NDIM > 2) {
        ux = ux + factorx * (Q(i, j, k - 1, 1) - Q(i - 1, j, k - 1, 1) + Q(i, j - 1, k - 1, 1) - Q(i - 1, j - 1, k - 1, 1));
        vy = vy + factory * (Q(i, j, k - 1, 2 % NV) - Q(i, j - 1, k - 1, 2 % NV) + Q(i - 1, j, k - 1, 2 % NV) - Q(i - 1, j - 1, k - 1, 2 % NV));
        wz = wz + factorz * (Q(i, j, k, 3 % NV) - Q(i, j, k - 1, 3 % NV) + Q(i, j - 1, k, 3 % NV) - Q(i, j - 1, k - 1, 3 % NV) +
                             Q(i - 1, j, k, 3 % NV) - Q(i - 1, j, k - 1, 3 % NV) + Q(i - 1, j - 1, k, 3 % NV) - Q(i - 1, j - 1, k - 1, 3 % NV));
      }
      s.div[DIF ? e : 0] = ux + vy + wz;
    }
  }
  // ---- uslope + trace on cells 0..3 (hydro/umuscl.f90:970, :176/:305/:483) ----
  const double dtdx = dt_ / a.dx;
  if (live)
    for (int tc = tl; tc < NTR; tc += AMR_TPO) {
      const int i = tc % 4, j = HY ? (tc / 4) % 4 : 1, k = HZ ? tc / 16 : 1;        // patch coordinates 0..3 (1-D/2-D: fixed 1)
      const int pc = (i + 1) + 6 * ((HY ? j + 1 : 0) + PJ * (HZ ? k + 1 : 0));
      constexpr int SJ = 6, SK = 6 * PJ;
      double q[NV], dq[NDIM][NV];
#pragma unroll
      for (int n = 0; n < NV; n++) q[n] = s.q[n][pc];
      if (P.slope_type == 3 && NDIM > 1) {
#pragma unroll
        for (int n = 0; n < NV; n++) {
          const double* qn = &s.q[n][pc];
          double vmin = 0, vmax = 0;
          bool first = true;
          for (int cc = (HZ ? -1 : 0); cc <= (HZ ? 1 : 0); cc++)
            for (int aa = -1; aa <= 1; aa++)
              for (int bb = -1; bb <= 1; bb++) {
                const double d = qn[aa + bb * SJ + cc * SK] - q[n];
                if (first) { vmin = d; vmax = d; first = false; }
                else { vmin = fmn(vmin, d); vmax = fmx(vmax, d); }
              }
          const double dfx = 0.5 * (qn[1] - qn[-1]);
          const double dfy = 0.5 * (qn[SJ] - qn[-SJ]);
          double dfz = 0, dff;
          if (HZ) { dfz = 0.5 * (qn[SK] - qn[-SK]); dff = 0.5 * (fabs(dfx) + fabs(dfy) + fabs(dfz)); }
          else dff = 0.5 * (fabs(dfx) + fabs(dfy));
          double slop;
          if (dff > 0.0) slop = fmn(1.0, fdiv(fmn(fabs(vmin), fabs(vmax)), dff));
          else slop = 1.0;
          dq[0][n] = slop * dfx;
          dq[HY][n] = slop * dfy;
          if (HZ) dq[NDIM - 1][n] = slop * dfz;
        }
      } else if (NDIM == 1 && P.slope_type >= 4 && P.slope_type <= 6) {
        const double uvel = q[1];
#pragma unroll
        for (int n = 0; n < NV; n++) {
          const double qL = s.q[n][pc - 1], qC = q[n], qR = s.q[n][pc + 1];
          double r;
          if (P.slope_type == 4) {
            const double dcen = uvel * dt_ / a.dx;
            const double dlft = 2.0 / (1.0 + dcen) * (qC - qL), drgt = 2.0 / (1.0 - dcen) * (qR - qC);
            double dlim = fmn(fabs(dlft), fabs(drgt));
            if ((dlft * drgt) <= 0.0) dlim = 0.0;
            r = fsign1(dlft) * dlim;
          } else if (P.slope_type == 5) {
            if (n == 0) {
              const double dcen = uvel * dt_ / a.dx;
              double dlft, drgt;
              if (dcen >= 0) { dlft = 2.0 / (0.0 + dcen + 1e-10) * (qC - qL); drgt = 2.0 / (1.0 - dcen) * (qR - qC); }
              else { dlft = 2.0 / (1.0 + dcen) * (qC - qL); drgt = 2.0 / (0.0 - dcen + 1e-10) * (qR - qC); }
              double dlim = fmn(fabs(dlft), fabs(drgt));
              if ((dlft * drgt) <= 0.0) dlim = 0.0;
              r = fsign1(dlft) * dlim;
            } else r = 0;
          } else {
            if (n == 0) r = 0.5 * ((qC - qL) + (qR - qC)); else r = 0;
          }
          dq[0][n] = r;
        }
      } else {
#pragma unroll
        for (int n = 0; n < NV; n++) {
          const double* qn = &s.q[n][pc];
          dq[0][n] = slope_lcr<NDIM, -1>(qn[-1], q[n], qn[1], P);
          if (HY) dq[HY][n] = slope_lcr<NDIM, -1>(qn[-SJ], q[n], qn[SJ], P);
          if (HZ) dq[NDIM - 1][n] = slope_lcr<NDIM, -1>(qn[-SK], q[n], qn[SK], P);
        }
      }
      double s0[NV];
      trace_sources<NDIM, NPS>(q, dq, rcp_rn(q[0]), s0, P);
#pragma unroll
      for (int d = 0; d < NDIM; d++) {
#pragma unroll
        for (int n = 0; n < NV; n++) {
          const double tt = s0[n] * dtdx * 0.5;
          double vp = q[n] - 0.5 * dq[d][n] + tt, vm = q[n] + 0.5 * dq[d][n] + tt;
          if (n == 0) { if (vp < P.smallr) vp = q[0]; if (vm < P.smallr) vm = q[0]; }
          s.qp[d][n][tc] = vp;
          s.qm[d][n][tc] = vm;
        }
      }
    }
  __syncthreads();
  // ---- cmpflxm: 3*2^(ndim-1) faces per direction (hydro/umuscl.f90:97,120,144), flux = fx*dt/dx, masking :720-747 ----
  if (live)
    for (int e = tl; e < NDIM * NF; e += AMR_TPO) {
      const int d = e / NF, f = e % NF;
      // face coordinates: along d: 1..3, transverse: 1..2
      int c3[3] = {1, 1, 1};
      int rem = f;
      for (int dd = 0; dd < NDIM; dd++) {
        const int ext = (dd == d) ? 3 : 2;
        c3[dd] = 1 + rem % ext;
        rem /= ext;
      }
      int cl[3] = {c3[0], c3[1], c3[2]};
      cl[d] -= 1;
      const int tR = c3[0] + 4 * ((HY ? c3[1] : 0) + 4 * (HZ ? c3[2] : 0));
      const int tL = cl[0] + 4 * ((HY ? cl[1] : 0) + 4 * (HZ ? cl[2] : 0));
      const int ln = d + 1, lt1 = (d == 0) ? 2 : 1, lt2 = (d == 2) ? 2 : 3;       // cmpflxm(…,ln,lt1,lt2) as 0-based variable indices
      double ql[NV], qr[NV], fg[NV], fl[NV];
      ql[0] = s.qm[d][0][tL]; ql[1] = s.qm[d][ln][tL]; ql[2] = s.qm[d][NDIM + 1][tL];
      qr[0] = s.qp[d][0][tR]; qr[1] = s.qp[d][ln][tR]; qr[2] = s.qp[d][NDIM + 1][tR];
      if (NDIM > 1) { ql[3] = s.qm[d][lt1 % NV][tL]; qr[3] = s.qp[d][lt1 % NV][tR]; }
      if (NDIM > 2) { ql[4 % NV] = s.qm[d][lt2 % NV][tL]; qr[4 % NV] = s.qp[d][lt2 % NV][tR]; }
#pragma unroll
      for (int n = NH; n < NV; n++) { ql[n] = s.qm[d][n][tL]; qr[n] = s.qp[d][n][tR]; }
      double fe = 0.0;
      riemann<NDIM, RIEMANN, NPS>(ql, qr, fg, P, (SRC && a.pfix) ? &fe : nullptr);
      fl[0] = fg[0]; fl[ln] = fg[1]; fl[NDIM + 1] = fg[2];
      if (NDIM > 1) fl[lt1 % NV] = fg[3];
      if (NDIM > 2) fl[lt2 % NV] = fg[4 % NV];
#pragma unroll
      for (int n = NH; n < NV; n++) fl[n] = fg[n];
      const int pR = (c3[0] + 1) + 6 * ((HY ? c3[1] + 1 : 0) + PJ * (HZ ? c3[2] + 1 : 0));
      const int pL = (cl[0] + 1) + 6 * ((HY ? cl[1] + 1 : 0) + PJ * (HZ ? cl[2] + 1 : 0));
      const bool masked = s.ok[pL] || s.ok[pR];
      double div1 = 0.0;
      if (DIF) {   // consup :769-869: vertices of the face, difmag*min(0, mean divergence)
        constexpr int VJ = HY ? 3 : 1;
        auto DV = [&](int ii, int jj, int kk) -> double { return s.div[DIF ? (ii - 1) + 3 * ((HY ? jj - 1 : 0) + VJ * (HZ ? kk - 1 : 0)) : 0]; };
        double hp = 1.0;
        for (int dd = 1; dd < NDIM; dd++) hp = hp * 0.5;
        const double factor = hp;
        const int i = c3[0], j = c3[1], k = c3[2];
        if (d == 0) {
          div1 = factor * DV(i, j, k);
          if (NDIM > 1) div1 = div1 + factor * DV(i, j + 1, k);
          if (NDIM > 2) div1 = div1 + factor * (DV(i, j, k + 1) + DV(i, j + 1, k + 1));
        } else if (d == 1) {
          div1 = 0.0;
          div1 = div1 + factor * (DV(i, j, k) + DV(i + 1, j, k));
          if (NDIM > 2) div1 = div1 + factor * (DV(i, j, k + 1) + DV(i + 1, j, k + 1));
        } else {
          div1 = factor * (DV(i, j, k) + DV(i + 1, j, k) + DV(i, j + 1, k) + DV(i + 1, j + 1, k));
        }
        div1 = a.difmag * ((div1 < 0.0) ? div1 : 0.0);
      }
#pragma unroll
      for (int n = 0; n < NV; n++) {
        double v = a.dx_pow2 ? (fl[n] * dt_) * a.inv_dx : div_rn(fl[n] * dt_, a.dx, a.inv_dx);
        if (DIF) v = v + dt_ * div1 * (s.uc[DIF ? n : 0][DIF ? pR : 0] - s.uc[DIF ? n : 0][DIF ? pL : 0]);
        if (masked) v = 0.0;
        s.flux[d][n][f] = v;
      }
      if (SRC && a.pfix) {   // tmp1 = half*(qleft(ln)+qright(ln)), tmp2 = fgdnv(nvar+1) (umuscl.f90:844-850), scaled :111-112
        const double t1 = 0.5 * (ql[1] + qr[1]);
        double v1 = a.dx_pow2 ? (t1 * dt_) * a.inv_dx : div_rn(t1 * dt_, a.dx, a.inv_dx);
        double v2 = a.dx_pow2 ? (fe * dt_) * a.inv_dx : div_rn(fe * dt_, a.dx, a.inv_dx);
        if (masked) { v1 = 0.0; v2 = 0.0; }
        s.tmp[SRC ? d : 0][0][SRC ? f : 0] = v1;
        s.tmp[SRC ? d : 0][1][SRC ? f : 0] = v2;
      }
    }
  __syncthreads();
  // ---- conservative update of the oct's own cells (:751-792), x then y then z ----
  if (live) {
    const int nvu = NV + ((SRC && a.pfix) ? 2 : 0);     // + divu, enew
    for (int e = tl; e < (a.flux_only ? 0 : T * nvu); e += AMR_TPO) {
      const int is = e % T, n = e / T;
      const int c3[3] = {1 + (is & 1), 1 + ((is >> 1) & 1), 1 + ((is >> 2) & 1)};
      const int ic = amr_cell(t, is, igrid);
      double u = a.unew[(size_t)n * NC + ic - 1];
#pragma unroll
      for (int d = 0; d < NDIM; d++) {
        int fl_ = 0, fr_ = 0, mul = 1;
        for (int dd = 0; dd < NDIM; dd++) {
          const int ext = (dd == d) ? 3 : 2;
          fl_ += (c3[dd] - 1) * mul;
          fr_ += (c3[dd] - 1 + (dd == d ? 1 : 0)) * mul;
          mul *= ext;
        }
        if (SRC && n >= NV) u = u + (s.tmp[SRC ? d : 0][SRC ? n - NV : 0][SRC ? fl_ : 0] - s.tmp[SRC ? d : 0][SRC ? n - NV : 0][SRC ? fr_ : 0]);
        else u = u + (s.flux[d][n < NV ? n : 0][fl_] - s.flux[d][n < NV ? n : 0][fr_]);
      }
      a.unew[(size_t)n * NC + ic - 1] = u;
    }
    // fluxes through the outer faces, for the coarse reflux pass: side = 2*d + (0 left | 1 right)
    const int nvr = (SRC && a.pfix) ? NV + 2 : NV;
    for (int e = tl; e < TW * NSF * nvr; e += AMR_TPO) {
      const int n = e % nvr, fs = (e / nvr) % NSF, side = e / (nvr * NSF);
      const int d = side / 2, right = side % 2;
      int f = 0, mul = 1, rem = fs;
      for (int dd = 0; dd < NDIM; dd++) {
        const int ext = (dd == d) ? 3 : 2;
        int c;
        if (dd == d) c = right ? 2 : 0;
        else { c = rem % 2; rem /= 2; }
        f += c * mul;
        mul *= ext;
      }
      const int ro = a.rflux_index ? a.rflux_index[io] : io;
      a.rflux[(((size_t)ro * TW + side) * NSF + fs) * nvr + n] =
          (SRC && n >= NV) ? s.tmp[SRC ? d : 0][SRC ? n - NV : 0][SRC ? f : 0] : s.flux[d][n < NV ? n : 0][f];
    }
  }
}

// coarse reflux (hydro/godunov_fine.f90:798-908) in the reference's accumulation order: entries are grouped per target
// (cell), each with its contributions (oct, side, face) in the order the reference visits them.
struct RefluxArgs {
  int nent;                 // target cells
  const int* cell;          // [nent] coarse cell index
  const int* start;         // [nent+1]
  const int* src;           // [ncontrib] packed: oct*64 + side*8 + face
  const double* rflux;
  double* unew;
  long long ncell;
  int nvar, nsides, nsf;
  double oneontwotondim;
};
__global__ void amr_reflux_kernel(const RefluxArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.nent * a.nvar) return;
  const int e = i / a.nvar, n = i % a.nvar;
  const size_t idx = (size_t)n * a.ncell + a.cell[e] - 1;
  double u = a.unew[idx];
  for (int k = a.start[e]; k < a.start[e + 1]; k++) {
    const int sr = a.src[k];
    const int oct = sr >> 6, side = (sr >> 3) & 7, face = sr & 7;
    const double f = a.rflux[(((size_t)oct * a.nsides + side) * a.nsf + face) * a.nvar + n] * a.oneontwotondim;
    if (side & 1) u = u + f; else u = u - f;
  }
  a.unew[idx] = u;
}

// list-based passes on the mirrored arrays ------------------------------------------------------------------------------
// set_unew (hydro/godunov_fine.f90:40): unew = uold on the cells of the listed octs
__global__ void amr_copy_octs_kernel(const double* __restrict__ src, double* __restrict__ dst, const int* __restrict__ igrid, int n,
                                     int ncoarse, int ngridmax, long long ncell, int T, int nvar) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)n * T * nvar) return;
  const int o = (int)(i % n), ind = (int)((i / n) % T), iv = (int)(i / ((long long)n * T));
  const size_t c = (size_t)iv * ncell + ncoarse + (size_t)ind * ngridmax + igrid[o] - 1;
  dst[c] = src[c];
}
// set_uold, passive scalars only (hydro/godunov_fine.f90:176-190): cells whose density crosses the floor smallr keep their
// concentration -- inflow into a floored cell / outflow below the floor
__global__ void amr_scalar_floor_kernel(const double* __restrict__ uold, double* __restrict__ unew, const int* __restrict__ igrid, int n,
                                        int ncoarse, int ngridmax, long long ncell, int T, int nhydro, int nvar, double smallr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * T) return;
  const int o = i % n, ind = i / n;
  const size_t c = (size_t)ncoarse + (size_t)ind * ngridmax + igrid[o] - 1;
  const double dold = uold[c], dnew = unew[c];
  if (dold < smallr && dnew > dold) {
    for (int iv = nhydro; iv < nvar; iv++) unew[(size_t)iv * ncell + c] = uold[(size_t)iv * ncell + c] * fmx(dnew, smallr) / smallr;
  } else if (dnew < smallr && dold > dnew) {
    for (int iv = nhydro; iv < nvar; iv++) unew[(size_t)iv * ncell + c] = uold[(size_t)iv * ncell + c] * smallr / fmx(dold, smallr);
  }
}
// ---- source terms of set_unew / set_uold (poisson, pressure_fix) on the mirrored arrays ---------------------------------------
// set_unew, pressure_fix part (hydro/godunov_fine.f90:71-90): divu = 0, enew = internal energy of uold on the active cells
__global__ void amr_pfix_init_kernel(const double* __restrict__ uold, double* __restrict__ divu, double* __restrict__ enew,
                                     const int* __restrict__ igrid, int n, int ncoarse, int ngridmax, long long ncell, int T, int ndim,
                                     double smallr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * T) return;
  const int o = i % n, ind = i / n;
  const size_t c = (size_t)ncoarse + (size_t)ind * ngridmax + igrid[o] - 1;
  pfix_init_cell(uold + c, (size_t)ncell, divu + c, enew + c, ndim, smallr);
}
// add_gravity_source_terms (hydro/godunov_fine.f90:237-289)
__global__ void amr_gravity_src_kernel(const double* __restrict__ uold, double* __restrict__ unew, const double* __restrict__ force,
                                       const int* __restrict__ igrid, int n, int ncoarse, int ngridmax, long long ncell, int T, int ndim,
                                       double smallr, double dt, const double* __restrict__ dt_dev) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * T) return;
  const int o = i % n, ind = i / n;
  const size_t c = (size_t)ncoarse + (size_t)ind * ngridmax + igrid[o] - 1;
  const double dtl = dt_dev ? *dt_dev : dt;
  double mx = 0, my = 0, mz = 0, fx = 0, fy = 0, fz = 0;
  if (ndim > 0) { mx = unew[(size_t)1 * ncell + c]; fx = force[c]; }
  if (ndim > 1) { my = unew[(size_t)2 * ncell + c]; fy = force[(size_t)1 * ncell + c]; }
  if (ndim > 2) { mz = unew[(size_t)3 * ncell + c]; fz = force[(size_t)2 * ncell + c]; }
  double e = unew[(size_t)(ndim + 1) * ncell + c];
  gravity_src_cell(unew[c], mx, my, mz, e, fmx(uold[c], smallr), fx, fy, fz, ndim, smallr, dtl);   // strict_equilibrium = 0
  if (ndim > 0) unew[(size_t)1 * ncell + c] = mx;
  if (ndim > 1) unew[(size_t)2 * ncell + c] = my;
  if (ndim > 2) unew[(size_t)3 * ncell + c] = mz;
  unew[(size_t)(ndim + 1) * ncell + c] = e;
}
// add_pdv_source_terms, pressure_fix part (hydro/godunov_fine.f90:294-437): enew -= (gamma-1) e_old div(u) dt, the velocity
// divergence from the face neighbours in uold (the coarser father cell, 1.5 dx away, where no neighbour oct exists)
__global__ void amr_pdv_kernel(const AmrTree t, const double* __restrict__ uold, double* __restrict__ enew, const int* __restrict__ igrid,
                               int n, int ndim, double gamma, double smallr, double dx_loc, double dt, const double* __restrict__ dt_dev) {
  const int T = 1 << ndim;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * T) return;
  const int o = i % n, ind = i / n;
  const int ig = igrid[o];
  const size_t NC = (size_t)t.ncell;
  const double dtl = dt_dev ? *dt_dev : dt;
  auto UO = [&](int icell, int iv) -> double { return uold[(size_t)iv * NC + icell - 1]; };
  double divu_loc = 0.0;
  for (int d = 0; d < ndim; d++) {
    const int b = (ind >> d) & 1;                       // position of the cell inside its oct along d
    const int other = ind ^ (1 << d);                   // jjj: the cell across the oct's mid-plane / in the neighbour oct
    const int cl_nb = amr_nbor(t, ig, 2 * d + 1), cr_nb = amr_nbor(t, ig, 2 * d + 2);
    // left neighbour: inside the oct for b = 1 (iii = 0), the left neighbour oct for b = 0
    int c1, c2;
    double dx_g, dx_d;
    if (b == 1) { c1 = amr_cell(t, other, ig); dx_g = dx_loc; }
    else { const int g1 = t.son[cl_nb]; c1 = g1 > 0 ? amr_cell(t, other, g1) : cl_nb; dx_g = g1 > 0 ? dx_loc : dx_loc * 1.5; }
    if (b == 0) { c2 = amr_cell(t, other, ig); dx_d = dx_loc; }
    else { const int g2 = t.son[cr_nb]; c2 = g2 > 0 ? amr_cell(t, other, g2) : cr_nb; dx_d = g2 > 0 ? dx_loc : dx_loc * 1.5; }
    divu_loc = pdv_face_term(divu_loc, UO, c1, c2, d, dx_g, dx_d, smallr);
  }
  const int ic = amr_cell(t, ind, ig);
  enew[ic - 1] = pdv_cell(enew[ic - 1], divu_loc, UO, ic, ndim, gamma, smallr, dtl);
}
// set_uold, pressure_fix part (hydro/godunov_fine.f90:203-227), after uold <- unew: total energy = kinetic + enew where the
// conservative internal energy is below the truncation error beta_fix*d*(|div u| dx)^2  (hexp = 0: no cosmology)
__global__ void amr_pfix_switch_kernel(double* __restrict__ uold, const double* __restrict__ divu, const double* __restrict__ enew,
                                       const int* __restrict__ igrid, int n, int ncoarse, int ngridmax, long long ncell, int T, int ndim,
                                       double smallr, double beta_fix, double dx, double dt, const double* __restrict__ dt_dev) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * T) return;
  const int o = i % n, ind = i / n;
  const size_t c = (size_t)ncoarse + (size_t)ind * ngridmax + igrid[o] - 1;
  const double dtl = dt_dev ? *dt_dev : dt;
  pfix_switch_cell(uold + c, (size_t)ncell, divu + c, enew + c, ndim, smallr, beta_fix, dx, dtl);
}
// ghost-oct exchange buffers on the mirrored arrays: all variables and all cells of the listed octs in one message
// (make_virtual_fine_dp / make_virtual_reverse_dp, amr/virtual_boundaries.f90:373,693)
__global__ void amr_pack_kernel(const double* __restrict__ u, const int* __restrict__ igrid, int n, int ncoarse, int ngridmax,
                                long long ncell, int T, int nvar, double* __restrict__ buf) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)n * T * nvar) return;
  const int o = (int)(i % n), ind = (int)((i / n) % T), iv = (int)(i / ((long long)n * T));
  buf[i] = u[(size_t)iv * ncell + ncoarse + (size_t)ind * ngridmax + igrid[o] - 1];
}
__global__ void amr_unpack_kernel(double* __restrict__ u, const int* __restrict__ igrid, int n, int ncoarse, int ngridmax, long long ncell,
                                  int T, int nvar, const double* __restrict__ buf, int mode /*0 copy, 1 accumulate, 2 zero*/) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)n * T * nvar) return;
  const int o = (int)(i % n), ind = (int)((i / n) % T), iv = (int)(i / ((long long)n * T));
  const size_t c = (size_t)iv * ncell + ncoarse + (size_t)ind * ngridmax + igrid[o] - 1;
  if (mode == 0) u[c] = buf[i];
  else if (mode == 1) u[c] = u[c] + buf[i];
  else u[c] = 0.0;
}
// upload_fine (hydro/interpol_hydro.f90:5, upl :73): split cells <- mean of their sons
__global__ void amr_upload_kernel(double* __restrict__ u, const int* __restrict__ son1, const int* __restrict__ igrid, int n, int ncoarse,
                                  int ngridmax, long long ncell, int T, int nvar, double smallr, int interpol_var = 0, int ndim = 3) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * T) return;
  const int o = i % n, ind = i / n;
  const int ic = ncoarse + ind * ngridmax + igrid[o];
  const int gs = son1[ic];
  if (gs <= 0) return;
  double getx = 0.0;
  for (int is = 0; is < T; is++) getx = getx + fmx(u[(size_t)ncoarse + (size_t)is * ngridmax + gs - 1], smallr);
  u[ic - 1] = getx / (double)T;
  for (int iv = 1; iv < nvar; iv++) {
    getx = 0.0;
    for (int is = 0; is < T; is++) getx = getx + u[(size_t)iv * ncell + ncoarse + (size_t)is * ngridmax + gs - 1];
    u[(size_t)iv * ncell + ic - 1] = getx / (double)T;
  }
  if (interpol_var == 1 || interpol_var == 2) {   // average the internal energy instead of the total energy :204-261
    getx = 0.0;
    for (int is = 0; is < T; is++) {
      const size_t cs = (size_t)ncoarse + (size_t)is * ngridmax + gs - 1;
      double ekin = 0.0;
      for (int d = 1; d <= ndim; d++) ekin = ekin + 0.5 * (u[(size_t)d * ncell + cs] * u[(size_t)d * ncell + cs]) / fmx(u[cs], smallr);
      getx = getx + u[(size_t)(ndim + 1) * ncell + cs] - ekin - 0.0;
    }
    double ekin = 0.0;
    for (int d = 1; d <= ndim; d++) ekin = ekin + 0.5 * (u[(size_t)d * ncell + ic - 1] * u[(size_t)d * ncell + ic - 1]) / fmx(u[ic - 1], smallr);
    u[(size_t)(ndim + 1) * ncell + ic - 1] = getx / (double)T + ekin + 0.0;
  }
}
// hydro_refine (hydro/godunov_utils.f90:125-263) for one (left, centre, right) triple of conservative states: relative
// gradients of density, pressure and Mach-scaled velocity against err_grad_d / _u / _p (a negative threshold disables a test)
template <int NDIM>
__device__ bool amr_hydro_refine(const double* ug_, const double* um_, const double* ud_, double gamma, double smallr,
                                 double err_d, double err_u, double err_p, double floor_d, double floor_u, double floor_p) {
  constexpr int IP = NDIM + 1;
  double u[3][NDIM + 2];
  const double* src[3] = {ug_, um_, ud_};
#pragma unroll
  for (int s = 0; s < 3; s++) {
#pragma unroll
    for (int v = 0; v < NDIM + 2; v++) u[s][v] = src[s][v];
    u[s][0] = u[s][0] > smallr ? u[s][0] : smallr;
#pragma unroll
    for (int d = 0; d < NDIM; d++) u[s][d + 1] = u[s][d + 1] / u[s][0];
    double ek = 0.0;
#pragma unroll
    for (int d = 0; d < NDIM; d++) ek = ek + 0.5 * u[s][0] * (u[s][d + 1] * u[s][d + 1]);
    u[s][IP] = (gamma - 1.0) * (u[s][IP] - ek);
  }
  const double *g = u[0], *c = u[1], *d_ = u[2];
  bool ok = false;
  if (err_d >= 0.0) {
    const double a = fabs((d_[0] - c[0]) / (d_[0] + c[0] + floor_d)), b = fabs((c[0] - g[0]) / (c[0] + g[0] + floor_d));
    const double e = 2.0 * (a > b ? a : b);
    ok = ok || e > err_d;
  }
  if (err_p >= 0.0) {
    const double a = fabs((d_[IP] - c[IP]) / (d_[IP] + c[IP] + floor_p)), b = fabs((c[IP] - g[IP]) / (c[IP] + g[IP] + floor_p));
    const double e = 2.0 * (a > b ? a : b);
    ok = ok || e > err_p;
  }
  if (err_u >= 0.0) {
    const double f2 = floor_u * floor_u;
#pragma unroll
    for (int k = 0; k < NDIM; k++) {
      const double vg = g[k + 1], vm = c[k + 1], vd = d_[k + 1];
      const double tg = gamma * g[IP] / g[0], tm = gamma * c[IP] / c[0], td = gamma * d_[IP] / d_[0];
      const double cg = sqrt(tg > f2 ? tg : f2), cm = sqrt(tm > f2 ? tm : f2), cd = sqrt(td > f2 ? td : f2);
      const double a = fabs((vd - vm) / (cd + cm + fabs(vd) + fabs(vm) + floor_u));
      const double b = fabs((vm - vg) / (cm + cg + fabs(vm) + fabs(vg) + floor_u));
      const double e = 2.0 * (a > b ? a : b);
      ok = ok || e > err_u;
    }
  }
  return ok;
}
// hydro_flag (hydro/hydro_flag.f90:1-200) on the device: one thread per active cell; a missing neighbour cell is replaced by its
// father cell (:113-119 -- exactly what amr_getnborfather returns one level down).  out[i*T + ind] = 1 where the cell must be
// flagged (the host ORs it into flag1: the state never leaves the device for a flag_fine pass).
template <int NDIM>
__global__ void amr_hydro_flag_kernel(const AmrTree t, const double* __restrict__ uold, const int* __restrict__ igrid, int n, int ilevel,
                                      double gamma, double smallr, double err_d, double err_u, double err_p, double floor_d,
                                      double floor_u, double floor_p, int* __restrict__ out) {
  constexpr int T = 1 << NDIM, NV = NDIM + 2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * T) return;
  const int o = i / T, ind = i % T;
  const int c = amr_cell(t, ind, igrid[o]);
  int fa[7];
  amr_getnborfather<NDIM>(t, c, ilevel + 1, fa);
  bool ok = false;
  double um[NV];
#pragma unroll
  for (int v = 0; v < NV; v++) um[v] = uold[(size_t)v * t.ncell + c - 1];
#pragma unroll
  for (int d = 0; d < NDIM; d++) {
    double ug[NV], ud[NV];
#pragma unroll
    for (int v = 0; v < NV; v++) {
      ug[v] = uold[(size_t)v * t.ncell + fa[2 * d + 1] - 1];
      ud[v] = uold[(size_t)v * t.ncell + fa[2 * d + 2] - 1];
    }
    ok = ok || amr_hydro_refine<NDIM>(ug, um, ud, gamma, smallr, err_d, err_u, err_p, floor_d, floor_u, floor_p);
  }
  out[i] = ok ? 1 : 0;
}

// make_boundary_hydro (hydro/hydro_boundary.f90:5) on the mirrored arrays
struct AmrBoundArgs {
  int n; const int* igrid; int inbor; int ind_ref[8]; double gs[3]; int kind; int ndim, nvar; double smallr;
  double bvar[8];   // kind 2: boundary_var(ibound, :) (imposed boundary, default boundana)
};
__global__ void amr_boundary_kernel(double* __restrict__ u, const AmrTree t, const AmrBoundArgs b) {
  const int T = 1 << b.ndim;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= b.n * T) return;
  const int o = i / T, ind = i % T;
  const int ig = b.igrid[o];
  const size_t NC = (size_t)t.ncell;
  if (b.kind == 2) {   // hydro_boundary.f90:229-252
    const int ic2 = amr_cell(t, ind, ig);
    for (int iv = 0; iv < b.nvar; iv++) u[(size_t)iv * NC + ic2 - 1] = b.bvar[iv];
    return;
  }
  const int gref = t.son[amr_nbor(t, ig, b.inbor)];
  const int ic = amr_cell(t, ind, ig), icr = amr_cell(t, b.ind_ref[ind] - 1, gref);
  double uu[8];
  for (int iv = 0; iv < b.nvar; iv++) uu[iv] = u[(size_t)iv * NC + icr - 1];
  if (b.kind == 0) {
    for (int iv = 0; iv < b.nvar; iv++) {
      double sw = 1.0;
      if (iv >= 1 && iv <= b.ndim) sw = b.gs[iv - 1];
      u[(size_t)iv * NC + ic - 1] = uu[iv] * sw;
    }
  } else {
    double ekin = 0.0, d = fmx(uu[0], b.smallr);
    for (int idim = 0; idim < b.ndim; idim++) { const double v = uu[idim + 1] / d; ekin = ekin + 0.5 * d * (v * v); }
    uu[b.ndim + 1] = uu[b.ndim + 1] - ekin;
    ekin = 0.0; d = fmx(uu[0], b.smallr);
    for (int idim = 0; idim < b.ndim; idim++) { const double v = uu[idim + 1] / d; ekin = ekin + 0.5 * d * (v * v); }
    uu[b.ndim + 1] = uu[b.ndim + 1] + ekin;
    for (int iv = 0; iv < b.nvar; iv++) u[(size_t)iv * NC + ic - 1] = uu[iv];
  }
}
// courant_fine over the LEAF cells of the listed octs (hydro/courant_fine.f90:61)
template <int NDIM>
__global__ void amr_courant_kernel(const double* __restrict__ u, const AmrTree t, const int* __restrict__ igrid, int n, Phys P, double dx,
                                   double* __restrict__ part, const double* __restrict__ force = nullptr) {
  constexpr int NV = NDIM + 2, T = 1 << NDIM;
  __shared__ double red[4][32];
  double my_dt = 1e300, m0 = 0, m1 = 0, m2 = 0;
  const size_t NC = (size_t)t.ncell;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (long long)n * T; i += (long long)gridDim.x * blockDim.x) {
    const int o = (int)(i % n), ind = (int)(i / n);
    const int ic = amr_cell(t, ind, igrid[o]);
    if (t.son[ic] != 0) continue;
    double uu[NV];
#pragma unroll
    for (int k = 0; k < NV; k++) uu[k] = u[(size_t)k * NC + ic - 1];
    double ei;
    double dtc;
    if (force) {   // gg = f (courant_fine.f90:75-83)
      double gs = 0.0;
#pragma unroll
      for (int d = 0; d < NDIM; d++) gs = gs + fabs(force[(size_t)d * NC + ic - 1]);
      dtc = cmpdt_cell<NDIM>(uu, dx, P, ei, gs);
    } else dtc = cmpdt_cell<NDIM>(uu, dx, P, ei);
    my_dt = dtc < my_dt ? dtc : my_dt;
    m0 += uu[0]; m1 += uu[NDIM + 1]; m2 += ei;
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

// the time-step bookkeeping of amr_step on device-resident dtnew / dtold (amr/amr_step.f90:326-331,:346-361,:567-577)
enum { DT_SAVE_OLD = 0, DT_AFTER_COURANT = 1, DT_NO_FINER = 2, DT_SYNC_COARSE = 3 };
__global__ void amr_dt_op_kernel(int op, double* dtnew, double* dtold, const double* courant_dt, int l, int levelmin, double nsub_coarse,
                                 double nsub_l, int icount) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  if (op == DT_SAVE_OLD) dtold[l] = dtnew[l];
  else if (op == DT_AFTER_COURANT) {
    double dt = *courant_dt;
    if (l > levelmin) { const double c = dtnew[l - 1] / nsub_coarse; dt = (c < dt) ? c : dt; }   // MIN(dtnew(l-1)/nsubcycle(l-1), dtnew(l))
    dtnew[l] = dt;
  } else if (op == DT_NO_FINER) { dtold[l + 1] = dtnew[l] / nsub_l; dtnew[l + 1] = dtnew[l] / nsub_l; }
  else if (op == DT_SYNC_COARSE) {
    if (nsub_coarse == 1.0) dtnew[l - 1] = dtnew[l];
    if (icount == 2) dtnew[l - 1] = dtold[l] + dtnew[l];
  }
}

// ---- patch mode (a refined level whose octs form a Cartesian box): ghost shell of the level store ------------------------
// father cell (level l-1) of every empty shell slot around the box: the neighbours of the surface octs that have no son
__global__ void amr_shell_father_kernel(const AmrTree t, const int* __restrict__ active, const int* __restrict__ act_slot, int nact, int ilevel,
                                        int nox, int noy, long long nslot, int* __restrict__ shell_father) {
  const int io = blockIdx.x * blockDim.x + threadIdx.x;
  if (io >= nact) return;
  int nfc[27], ng[8];
  amr_get3cubefather<3>(t, active[io], ilevel, nfc, ng);
  const long long s0 = act_slot[io];
  for (int j = 0; j < 27; j++) {
    if (nfc[j] <= 0 || t.son[nfc[j]] > 0) continue;
    const long long s = s0 + (j % 3 - 1) + (long long)nox * ((j / 3) % 3 - 1) + (long long)nox * noy * (j / 9 - 1);
    if (s >= 0 && s < nslot) shell_father[s] = nfc[j];     // every writer stores the same value
  }
}
// prolongation of the shell octs from level l-1 (interpol_hydro, hydro/interpol_hydro.f90:268) into the level store
__global__ void amr_fill_shell_kernel(const AmrTree t, const double* __restrict__ uold, double* __restrict__ u, const int* __restrict__ shell_father,
                                      long long nslot, int ilevel, int nvar, int interpol_type) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= nslot * nvar) return;
  const long long s = i % nslot;
  const int n = (int)(i / nslot);
  const int fc = shell_father[s];
  if (fc <= 0) return;
  int fa[7];
  amr_getnborfather<3>(t, fc, ilevel, fa);
  double av[7], u2[8];
#pragma unroll
  for (int j = 0; j < 7; j++) av[j] = uold[(size_t)n * t.ncell + fa[j] - 1];
  amr_interpol_var<3>(av, interpol_type, u2);
#pragma unroll
  for (int is = 0; is < 8; is++) u[((size_t)n * 8 + is) * nslot + s] = u2[is];
}

// the same for interpol_var 1, 2 / interpol_type 4 (coupled variables): one thread per shell slot, nvar = 5
__global__ void amr_fill_shell_coupled_kernel(const AmrTree t, const double* __restrict__ uold, double* __restrict__ u,
                                              const int* __restrict__ shell_father, long long nslot, int ilevel, int interpol_type,
                                              int interpol_var, double smallr) {
  const long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (s >= nslot) return;
  const int fc = shell_father[s];
  if (fc <= 0) return;
  int fa[7];
  amr_getnborfather<3>(t, fc, ilevel, fa);
  double u1[7][5], u2[8][5];
  for (int j = 0; j < 7; j++)
#pragma unroll
    for (int n = 0; n < 5; n++) u1[j][n] = uold[(size_t)n * t.ncell + fa[j] - 1];
  amr_interpol_hydro<3, 5>(u1, interpol_type, interpol_var, smallr, u2);
  for (int is = 0; is < 8; is++)
#pragma unroll
    for (int n = 0; n < 5; n++) u[((size_t)n * 8 + is) * nslot + s] = u2[is][n];
}

// the instantiation of amr_godfine_kernel that runs a (nullptr: none is built for it); launch_amr_godfine launches it, and the
// host harness (tests/host_numerics) runs the same selection
using AmrGodfineKernel = void (*)(const AmrSweepArgs);
template <int NDIM, int RIEMANN>
AmrGodfineKernel amr_godfine_select(const AmrSweepArgs& a) {
  if (a.force || a.pfix) {   // source terms: hydro variables only, no difmag (checked by rgpu_init)
    if (a.nps != 0 || a.difmag > 0.0) return nullptr;
    return amr_godfine_kernel<NDIM, RIEMANN, false, 0, true>;
  }
  if (a.nps == 0) return a.difmag > 0.0 ? amr_godfine_kernel<NDIM, RIEMANN, true> : amr_godfine_kernel<NDIM, RIEMANN, false>;
  // passive scalars: NDIM=3, up to 2, without difmag (checked by rgpu_init)
  if (NDIM == 3 && a.nps == 1) return amr_godfine_kernel<NDIM, RIEMANN, false, (NDIM == 3 ? 1 : 0)>;
  if (NDIM == 3 && a.nps == 2) return amr_godfine_kernel<NDIM, RIEMANN, false, (NDIM == 3 ? 2 : 0)>;
  return nullptr;
}

#ifndef RGPU_HOST_NUMERICS   // (tests/host_numerics compiles the __device__ helpers above with g++: no kernel launches there)
template <int NDIM, int RIEMANN>
cudaError_t launch_amr_godfine(const AmrSweepArgs& a, cudaStream_t st) {
  const AmrGodfineKernel k = amr_godfine_select<NDIM, RIEMANN>(a);
  if (!k) return cudaErrorInvalidValue;
  k<<<(a.nact + AMR_OPB - 1) / AMR_OPB, AMR_TPO * AMR_OPB, 0, st>>>(a);
  return cudaGetLastError();
}
#endif

}  // namespace rgpu
