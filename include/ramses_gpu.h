/*
 * ramses_gpu.h -- C-ABI of the H100 (sm_90a) per-level Godunov sweep for RAMSES.
 *
 * This is the drop-in boundary: a Fortran patch directory (PATCH=..., reference
 * bin/Makefile:19,153) shadows hydro/godunov_fine.f90 with a shim that forwards
 * each routine to the entry point of the same name below through ISO_C_BINDING
 * (see INTEGRATION.md for the interface block).  Plain pointers and sizes only;
 * all arrays are the reference's own Fortran arrays: column-major, 1-based
 * indices stored as 32-bit integers, never freed or reallocated by the callee.
 *
 * Every function returns 0 on success or a negative RGPU_E* code; the last
 * error text is available from rgpu_last_error().  The reference has no error
 * channel besides write(*,*)+stop (hydro/umuscl.f90:801-803, amr/end.f90:26-46),
 * so the shim maps non-zero to `call clean_stop`.
 *
 * There is NO CPU fallback: every entry point fails with RGPU_ECUDA when no
 * CUDA device is usable.
 */
#ifndef RAMSES_GPU_H
#define RAMSES_GPU_H
#include <stddef.h>
#ifdef __cplusplus
extern "C" {
#endif

#define RGPU_ABI_VERSION 4

enum {
  RGPU_OK = 0,
  RGPU_EINVAL = -1,       /* bad argument / call order                        */
  RGPU_ECUDA = -2,        /* CUDA runtime error (no device, OOM, launch)      */
  RGPU_EUNSUPPORTED = -3, /* valid RAMSES configuration not covered yet        */
  RGPU_ENCCL = -4         /* NCCL error                                       */
};

/* riemann / scheme selectors: the strings of &HYDRO_PARAMS
 * (hydro/hydro_parameters.f90:84-85, dispatch hydro/umuscl.f90:791-804)       */
enum { RGPU_RIEMANN_LLF = 0, RGPU_RIEMANN_EXACT = 1, RGPU_RIEMANN_ACOUSTIC = 2,
       RGPU_RIEMANN_HLLC = 3, RGPU_RIEMANN_HLL = 4 };
enum { RGPU_SCHEME_MUSCL = 0, RGPU_SCHEME_PLMDE = 1 };

/* Run parameters: compile-time constants of the reference build (NDIM, NVAR,
 * bin/Makefile:65-84) and the &HYDRO_PARAMS / &AMR_PARAMS namelist values the
 * path reads (hydro/read_hydro_params.f90:43-54).                            */
typedef struct rgpu_params {
  int ndim;            /* NDIM 1,2,3                                          */
  int nvar;            /* NVAR = ndim+2 (+ up to 2 passive scalars: NDIM=3, oct-batch kernel, i.e. after rgpu_set_amr) */
  int nvector;         /* NVECTOR: accepted for interface parity, unused      */
  int slope_type;      /* 0,1,2,3,7,8 (+4,5,6 in 1-D)                          */
  int niter_riemann;   /* Newton iterations of riemann='exact'                */
  int scheme;          /* RGPU_SCHEME_MUSCL only                              */
  int riemann;         /* RGPU_RIEMANN_*                                       */
  int pressure_fix;    /* amr_parameters.f90:197.  1: divu / enew ride along the sweep (godfine1 :737-903), add_pdv_source_terms and
                        * the energy switch of set_uold (:203-227, with beta_fix below).  Oct-batch kernel only (rgpu_set_amr),
                        * nvar = ndim+2, difmag = 0; divu and enew live on the device (rgpu_download_pressure_fix)            */
  double gamma, smallr, smallc, slope_theta, difmag, courant_factor;
                       /* difmag>0 (cmpdivu/consup, hydro/uplmde.f90:702,769): oct-batch kernel only, i.e. after rgpu_set_amr(1,..) */
  double boxlen;
  int nx, ny, nz;      /* coarse grid incl. boundary cells (amr_parameters)   */
  int icoarse_min, icoarse_max, jcoarse_min, jcoarse_max, kcoarse_min, kcoarse_max;
  int nlevelmax;
  /* ideal-MHD build (SOLVER=mhd, bin/Makefile:20; mhd/ shadows hydro/ through VPATH): NDIM=3, nvar=8; the state arrays
   * then hold nvar+3 = 11 variables (left-face B in 6:8, right-face B in nvar+1:nvar+3, mhd/hydro_parameters.f90:15-30). */
  int mhd;             /* 0: hydro build, 1: MHD build                          */
  int riemann2d;       /* RGPU_MHD2D_* (mhd/hydro_parameters.f90:104)           */
  int slope_mag_type;  /* mhd/hydro_parameters.f90:93; -1 = slope_type (hydro/read_hydro_params.f90:528) */
  int fast;            /* 0 (default): STRICT arithmetic -- no FMA contraction, correctly rounded divisions: results bit-identical
                        * to the reference's evaluation order.  1: FAST arithmetic for the 3-D hydro dense sweep (FMA
                        * contraction, reciprocal-multiply quotients, <= 2 ulp reciprocal / sqrt): within 1e-12 relative of
                        * the strict result on the conserved state after N steps (north_star's tolerance), ~15 % fewer FP64
                        * instructions.  Ignored (strict) by every other path.                                              */
  int poisson;         /* amr_parameters.f90 `poisson`.  1: the acceleration f(1:ncell,1:ndim) of poisson_commons is an INPUT
                        * (rgpu_upload_force; the Poisson solver is out of scope): gravity predictor of ctoprim (umuscl.f90:932-938),
                        * gloc gather of godfine1 (:637-647), add_gravity_source_terms in set_uold (:237-289), gravity term of cmpdt
                        * (godunov_utils.f90:99-111).  Oct-batch kernel only (rgpu_set_amr), nvar = ndim+2, difmag = 0              */
  double beta_fix;     /* amr_parameters.f90:167 (pressure_fix truncation-error factor)                                          */
} rgpu_params;
/* `riemann` / `riemann2d` of the MHD build: iriemann, iriemann2d (hydro/read_hydro_params.f90:190-220) */
enum { RGPU_MHD_LLF = 0, RGPU_MHD_ROE = 1, RGPU_MHD_HLL = 2, RGPU_MHD_HLLD = 3, RGPU_MHD_UPWIND = 4, RGPU_MHD_HYDRO = 5 };
enum { RGPU_MHD2D_LLF = 0, RGPU_MHD2D_ROE = 1, RGPU_MHD2D_UPWIND = 2, RGPU_MHD2D_HLL = 3, RGPU_MHD2D_HLLA = 4, RGPU_MHD2D_HLLD = 5 };

/* ---- life cycle -------------------------------------------------------------
 * rgpu_init: once, after read_params (amr/read_params.f90:1).  device<0 picks
 * LOCAL_RANK (or 0).  myid is 1-based like the reference's.                     */
int rgpu_init(const rgpu_params* p, int myid, int ncpu, int device);
int rgpu_finalize(void);
const char* rgpu_last_error(void);
int rgpu_abi_version(void);

/* ---- tree mirror (amr/amr_commons.f90:68-79; re-call after refine/defrag/
 * load_balance, amr/amr_step.f90:92,109-117) ---------------------------------
 * son(1:ncell), father(1:ngridmax), nbor(1:ngridmax,1:2*ndim): pointers to the
 * first element of the Fortran arrays.  They must stay valid until the next
 * rgpu_bind_tree (the library reads them inside rgpu_bind_level only).         */
int rgpu_bind_tree(int ncoarse, int ngridmax, const int* son, const int* father, const int* nbor);

/* AMR mode (levelmin < nlevelmax): call once after rgpu_init and before rgpu_bind_tree.  The device then mirrors
 * son/father/nbor and the whole uold/unew arrays; every level is processed as a list of octs by the oct-batch kernel
 * (godfine1 with interpol_hydro ghost prolongation, flux masking and coarse refluxing, hydro/godunov_fine.f90:486-911).
 * interpol_type / interpol_var: &REFINE_PARAMS (hydro/hydro_parameters.f90:88-89): interpol_var 0 (conservative variables),
 * 1 (internal energy instead of total energy), 2 (velocities + internal energy, total momentum of the oct restored,
 * hydro/interpol_hydro.f90:318-345,393-440; upload_fine then averages the internal energy :204-261); interpol_type 0 (straight
 * injection), 1 (minmod), 2 (MonCen), 3 (central), 4 (central for the velocities, MonCen for the rest; needs interpol_var = 2).
 * In this mode rgpu_upload_state / rgpu_download_state move the WHOLE arrays (ilevel ignored).                       */
int rgpu_set_amr(int on, int interpol_type, int interpol_var);

/* ---- per-level communicator lists (amr/amr_commons.f90:108-119,170-180; built
 * by build_comm, amr/virtual_boundaries.f90:1286) ------------------------------
 * igrid_* are the %igrid arrays (1-based oct indices).  recv/emit are indexed by
 * peer cpu 0..ncpu-1 (entry myid-1 is ignored); pass ncpu=1 and NULLs for a
 * serial run.  bound lists are boundary(ibound,ilevel)%igrid with
 * boundary_type(ibound) as computed in hydro/read_hydro_params.f90:316-420.    */
int rgpu_bind_level(int ilevel, int ngrid_active, const int* igrid_active,
                    int ncpu, const int* ngrid_recv, const int* const* igrid_recv,
                    const int* ngrid_emit, const int* const* igrid_emit,
                    int nboundary, const int* boundary_type,
                    const int* ngrid_bound, const int* const* igrid_bound);

/* Host-only dry run of rgpu_bind_level: computes the level plan (is it a dense box? extents, owned range, periodic
 * wrap, slot numbering) from the tree and communicator lists without any CUDA call and without rgpu_init.
 * slot_igrid_out (may be NULL, capacity slot_cap) receives the igrid of every lattice slot (0 = empty).           */
int rgpu_plan_level(const rgpu_params* p, int myid, int ncoarse, int ngridmax, const int* father,
                    int ilevel, int ngrid_active, const int* igrid_active,
                    int ncpu, const int* ngrid_recv, const int* const* igrid_recv,
                    const int* ngrid_emit, const int* const* igrid_emit,
                    int nboundary, const int* boundary_type,
                    const int* ngrid_bound, const int* const* igrid_bound,
                    struct rgpu_level_info* info, int* slot_igrid_out, long long slot_cap);

/* ---- Level-0 contract: host arrays in, host arrays out ------------------------
 * godunov_fine(ilevel) (hydro/godunov_fine.f90:5) on uold(1:ncell,1:nvar) ->
 * unew(1:ncell,1:nvar): for every active cell of the level
 *   unew = uold + sum_d (F_d^- - F_d^+), order x,y,z (godunov_fine.f90:751-792)
 * (unew == uold on entry, i.e. right after set_unew; true for every
 * levelmin=levelmax run).  dt = dtnew(ilevel).  Includes H2D/D2H copies.       */
int rgpu_godunov_fine(int ilevel, double dt, const double* uold, double* unew);

/* The Level-0 call runs as a three-stream pipeline over z-slabs of the level (H2D of slab s+1 | gather + sweep + scatter of
 * slab s | D2H of slab s-1; PCIe is full duplex) whenever the oct numbering of the level is spatially coherent enough that a
 * slab is a few contiguous igrid ranges (lattice / Morton / Hilbert order).  The reference's creation order (amr/refine_utils.f90:
 * 395-447) scatters a slab over the whole igrid window; the call then keeps the serial order.  rgpu_set_pipeline(0) forces the
 * serial order (measurements); RGPU_E2E_SLABS=<n> at bind time sets the number of slabs (default 64, <3 disables).            */
int rgpu_set_pipeline(int enable);

/* Page-lock / unlock a host array so the copies above run at full PCIe rate.   */
int rgpu_host_register(void* ptr, size_t bytes);
int rgpu_host_unregister(void* ptr);

/* ---- Level-1 contract: device-resident state, same semantics as the F90 routines
 * of the same name -------------------------------------------------------------- */
int rgpu_upload_state(int ilevel, const double* uold);     /* host uold -> device level store */
int rgpu_download_state(int ilevel, double* uold);         /* device level store -> host uold  */
int rgpu_set_unew(int ilevel);                             /* hydro/godunov_fine.f90:40        */
int rgpu_godunov_fine_dev(int ilevel, double dt);          /* hydro/godunov_fine.f90:5         */
int rgpu_set_uold(int ilevel);                             /* hydro/godunov_fine.f90:135       */
/* courant_fine (hydro/courant_fine.f90:1): *dt_io = min(*dt_io, CFL dt over the leaf
 * cells of the level [over all ranks]); sums[3] += (mass, total E, internal E).
 * MHD build (mhd/courant_fine.f90:1): sums must hold 4 values, sums[3] += magnetic E */
int rgpu_courant_fine(int ilevel, double* dt_io, double sums[3]);
int rgpu_make_boundary_hydro(int ilevel);                  /* hydro/hydro_boundary.f90:5       */
/* imposed boundaries (bound_type = 3, boundary_type = 20+direction): var = boundary_var(ibound, 1:nvar), the conservative state
 * hydro/read_hydro_params.f90:440-468 builds from d_bound, u_bound, ...; what the default boundana (hydro/boundana.f90) copies
 * into every cell of the region (hydro_boundary.f90:229-252).  ibound is 1-based like the Fortran index; call once after
 * rgpu_init for every imposed region.  A patched boundana (position-dependent inflow) is not supported.                      */
int rgpu_set_boundary_var(int ibound, const double* var);
int rgpu_make_virtual_fine(int ilevel);                    /* amr/virtual_boundaries.f90:373, all nvar at once */
int rgpu_make_virtual_reverse(int ilevel);                 /* amr/virtual_boundaries.f90:693   */
int rgpu_upload_fine(int ilevel);                          /* hydro/interpol_hydro.f90:5 (restriction of split cells) */

/* hydro_flag (hydro/hydro_flag.f90:1, hydro_refine hydro/godunov_utils.f90:125-263) on the device-resident state (AMR mode):
 * flag1(cell) = 1 for every active cell of the level whose relative gradient of density / velocity / pressure towards a
 * neighbour (a missing neighbour cell is replaced by its father cell) exceeds err_grad = (err_grad_d, err_grad_u, err_grad_p)
 * (-1 disables a test), floor = (floor_d, floor_u, floor_p).  flag1 is the host array flag1(1:ncell) of amr_commons: only the
 * 4-byte flags of the level travel, the state stays on the device for the flag_fine pass.                                  */
int rgpu_hydro_flag(int ilevel, const double err_grad[3], const double floor[3], int* flag1);

/* Source terms (AMR mode).  rgpu_upload_force: the host array f(1:ncell,1:ndim) of poisson_commons (amr/init_poisson.f90) after
 * force_fine / gravana -- call it whenever the host recomputed the acceleration (rgpu_params.poisson = 1).
 * rgpu_download_pressure_fix: the device-resident divu(1:ncell) / enew(1:ncell) of hydro_commons (hydro/init_hydro.f90:40-42)
 * for diagnostics or a host-side pass that needs them (either pointer may be NULL).                                          */
/* MHD build in AMR mode: interpol_mag_type of &HYDRO_PARAMS (limiter of the face-field prolongation, interpol_mag
 * mhd/interpol_hydro.f90:990); -1 (default) = interpol_type (hydro/read_hydro_params.f90:531).                               */
int rgpu_set_interpol_mag(int interpol_mag_type);
int rgpu_upload_force(const double* f);
int rgpu_download_pressure_fix(double* divu, double* enew);

/* ---- fused fast path --------------------------------------------------------------
 * nstep level steps of a levelmin=levelmax run in amr_step order
 * (amr/amr_step.f90:326 courant, :333 set_unew, :388 godunov_fine, :423 set_uold,
 * :505 ghost exchange, :514 boundary), state and dt staying on the device.
 * dt_hist (nstep doubles, may be NULL) receives the dt of every step; sums_last[3]
 * (may be NULL) the courant_fine sums of the final state.                         */
int rgpu_level_steps(int ilevel, int nstep, double* dt_hist, double sums_last[3]);
/* numbtot(1,1:nlevelmax) of amr_commons: octs per level summed over all ranks (NCCL all-reduce of the bound levels' active
 * counts in AMR mode).  The reference gates amr_step and its recursion on this GLOBAL count (amr/amr_step.f90:33,345); a rank
 * that owns no oct of a level must still bind the level (ngrid_active = 0) and take part in its collectives.            */
int rgpu_level_totals(int nlevelmax, int* numbtot);
/* AMR mode: ncoarse_steps calls of amr_step(levelmin, 1) (amr/amr_step.f90: recursion over the levels whose GLOBAL oct count is
 * non-zero, sub-cycling nsubcycle(l) = 1 or 2; `nsubcycle` is the Fortran array nsubcycle(1:nlevelmax) of amr_parameters.f90
 * passed as it is: nsubcycle[l-1] = nsubcycle(l), nlevelmax elements.  :326 courant, :333 set_unew, :388 godunov_fine,
 * :397/:505 ghost exchanges, :423 set_uold, :441 upload_fine, :514 boundaries, :567-577 dt synchronisation) on a frozen mesh,
 * with dtnew/dtold device resident: no host round trip inside a coarse step.  dt_hist (may be NULL) receives dtnew(levelmin)
 * of every coarse step.                                                                                              */
int rgpu_amr_steps(int levelmin, const int* nsubcycle, int ncoarse_steps, double* dt_hist);

/* ---- multi-GPU: NCCL communicator replacing MPI_COMM_WORLD ----------------------
 * unique_id: the 128-byte ncclUniqueId produced by rgpu_comm_unique_id on rank 0 and
 * broadcast by the host program (MPI_Bcast in the Fortran driver).                */
int rgpu_comm_unique_id(void* unique_id_128);
int rgpu_comm_init(int nranks, int rank, const void* unique_id_128);

/* ---- introspection (tests / bench) ---------------------------------------------- */
typedef struct rgpu_level_info {
  int dense;                 /* 1: dense-box fast path (AMR mode: the dense kernel sweeps the level) */
  int ncell_box[3];          /* box extent in cells                                */
  int own_lo[3], own_hi[3];  /* owned cell range                                   */
  int wrap[3];
  long long nslot;
  long long kernel_launches; /* kernels launched on this level since bind          */
  double last_sweep_ms;      /* CUDA-event duration of the last sweep kernel (timing on) */
  double last_steps_ms;      /* CUDA-event duration of the last rgpu_level_steps call, on the launching stream */
  int pipeline_slabs;        /* z-slabs of the Level-0 pipeline (rgpu_godunov_fine); 0: serial H2D -> sweep -> D2H */
  int sweep_variant;         /* 3-D hydro: kernel variant in use (0: round-1 loop, else 100*BY + 10*CTAs/SM + solver form) */
} rgpu_level_info;
int rgpu_get_level_info(int ilevel, rgpu_level_info* out);
/* bitwise check of the shared-reciprocal division (hydro_device.cuh div_rn) against the IEEE `/` on npairs
 * pseudo-random and adversarial operand pairs; *mismatches must come back 0                                  */
int rgpu_selftest_div(long long npairs, unsigned long long seed, long long* mismatches);
/* time the next sweeps with CUDA events on the launching stream (bench)            */
int rgpu_set_timing(int enable);
int rgpu_device_synchronize(void);

#ifdef __cplusplus
}
#endif
#endif /* RAMSES_GPU_H */
