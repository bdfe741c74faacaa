/*
 * ramses_oracle.h -- CPU ORACLE (test infrastructure, NOT product code).
 *
 * A plain-C restatement of the RAMSES per-level Godunov sweep
 * (godunov_fine -> godfine1 -> unsplit -> ctoprim/uslope/trace/cmpflxm ->
 * riemann_*), its Courant scan and the passes either side of it, written in
 * the reference's own shape (per-oct 6^ndim patches, batches of nvector octs,
 * Fortran operation order, no FMA contraction, IEEE division and sqrt).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may load this library.  The product (ramses_b200/)
 * never links or calls it.
 *
 * PARITY PINNING STATUS: see the header of ramses_oracle.c.
 *
 * All citations "file:line" are relative to the reference tree
 * (tatary/ramses), e.g. hydro/umuscl.f90:22.
 */
#ifndef RAMSES_ORACLE_H
#define RAMSES_ORACLE_H

#ifdef __cplusplus
extern "C" {
#endif

/* riemann solver ids (string `riemann` in hydro/hydro_parameters.f90:85) */
enum { ORC_RIEMANN_LLF = 0, ORC_RIEMANN_EXACT = 1, ORC_RIEMANN_ACOUSTIC = 2,
       ORC_RIEMANN_HLLC = 3, ORC_RIEMANN_HLL = 4 };
/* scheme ids (string `scheme` hydro/hydro_parameters.f90:84) */
enum { ORC_SCHEME_MUSCL = 0, ORC_SCHEME_PLMDE = 1 };

#define ORC_MAXBOUND 6

typedef struct {
  int ndim;            /* NDIM (compile-time in the reference, bin/Makefile)  */
  int nvar;            /* NVAR = ndim+2 (+ passive scalars)                    */
  int nvector;         /* NVECTOR batch length (bin/Makefile:11)               */
  int slope_type;      /* hydro_parameters.f90:76                              */
  int niter_riemann;   /* hydro_parameters.f90:75                              */
  int scheme;          /* ORC_SCHEME_*                                         */
  int riemann;         /* ORC_RIEMANN_*                                        */
  int pad_;
  double gamma, smallr, smallc, slope_theta, difmag, courant_factor;
  double boxlen;
} orc_params;

/* The oct tree, mirrored from amr/amr_commons.f90:68-79.  All arrays are
 * 1-based like the Fortran ones: element [0] is unused.                       */
typedef struct {
  int ndim;
  int nx, ny, nz;                 /* coarse grid incl. boundary coarse cells  */
  int icoarse_min, icoarse_max;   /* domain extent in coarse cells (x)        */
  int jcoarse_min, jcoarse_max;
  int kcoarse_min, kcoarse_max;
  int ncoarse, ngridmax, ncell;   /* ncell = ncoarse + 2^ndim * ngridmax      */
  int nlevelmax;
  int nboundary;
  int boundary_type[ORC_MAXBOUND];/* 1..6 reflexive, 11..16 outflow           */
  int *son;                       /* [ncell+1]                                */
  int *father;                    /* [ngridmax+1]                             */
  int *nbor;                      /* [(2*ndim) * (ngridmax+1)]: nbor[(j-1)*(ngridmax+1)+igrid] */
  double *xg;                     /* [ndim * (ngridmax+1)] oct centres        */
  int *cpu_map;                   /* [ncell+1]                                */
  /* per level (index 1..nlevelmax) */
  int *nactive;  int **active;    /* active(ilevel)%igrid (1-based content, 0-based C array) */
  int *nrecv;    int **recv;      /* reception (ghost) octs, all peers merged */
  int *nbound[ORC_MAXBOUND]; int **bound[ORC_MAXBOUND];
  int ngrid_used;
} orc_mesh;

/* ---------------- numerics (hydro/umuscl.f90, hydro/godunov_utils.f90) ---- */
/* 1-D Riemann solvers on vectors: qleft/qright (nvector,nvar), fgdnv (nvector,nvar+1)
 * column-major like Fortran: q[l + nvector*(ivar-1)]                          */
void orc_riemann_llf     (const orc_params*, const double* ql, const double* qr, double* fg, int ngrid);
void orc_riemann_hll     (const orc_params*, const double* ql, const double* qr, double* fg, int ngrid);
void orc_riemann_hllc    (const orc_params*, const double* ql, const double* qr, double* fg, int ngrid);
void orc_riemann_acoustic(const orc_params*, const double* ql, const double* qr, double* fg, int ngrid);
void orc_riemann_approx  (const orc_params*, const double* ql, const double* qr, double* fg, int ngrid);

/* unsplit (hydro/umuscl.f90:22): uin (nvector,6^ndim,nvar) -> flux, tmp       */
typedef struct orc_work orc_work;
orc_work* orc_work_new(const orc_params*);
void      orc_work_free(orc_work*);
void orc_unsplit(const orc_params*, orc_work*, const double* uin, const double* gravin,
                 double* flux, double* tmp, double dx, double dy, double dz, double dt, int ngrid);
/* cmpdt (hydro/godunov_utils.f90:5): uu(nvector,nvar) destroyed, gg(nvector,ndim) */
void orc_cmpdt(const orc_params*, double* uu, const double* gg, double dx, double* dt, int ncell);

/* ---------------- mesh ------------------------------------------------------ */
/* Build a fully refined tree levels 1..levelmax (levelmin=levelmax run).
 * bound_type[2*d+s] (d=0..2, s=0 min / 1 max face): 0 periodic, 1 reflexive,
 * 2 outflow.  order: 0 = reference creation order (children of all parents,
 * cell position outermost: amr/refine_utils.f90 make_grid_fine order),
 * 1 = lattice row-major, 2 = pseudo-random permutation (seed).               */
orc_mesh* orc_mesh_build_uniform(int ndim, int levelmax, const int bound_type[6], int order, unsigned seed);
/* the same on a domain of ndom[0] x ndom[1] x ndom[2] coarse cells (nx, ny, nz of AMR_PARAMS; ndom[d] = 1 for d >= ndim),
 * boundary coarse cells added around it as above; build_uniform is build_box with a single domain cell                */
orc_mesh* orc_mesh_build_box(int ndim, int levelmax, const int ndom[3], const int bound_type[6], int order, unsigned seed);
void      orc_mesh_free(orc_mesh*);
/* integer position of every oct of a level in units of oct size (for tests)   */
void orc_mesh_oct_pos(const orc_mesh*, int ilevel, int igrid, int pos[3]);
/* get3cubefather (amr/nbors_utils.f90:5) for ONE father cell                  */
void orc_get3cubefather(const orc_mesh*, int ind_cell_father, int ilevel, int* nbors_father_cells /*[3^ndim]*/,
                        int* nbors_father_grids /*[2^ndim]*/);
/* the lll/mmm lookup tables of getindices3cube (amr/nbors_utils.f90:305), generated */
void orc_getindices3cube(int ndim, int ind, int lll[27], int mmm[27]);

/* ---------------- per-level passes (state arrays are Fortran layout:
 *                  u[(ivar-1)*ncell + icell-1]) -------------------------------- */
double orc_dx(const orc_params*, const orc_mesh*, int ilevel);
void orc_condinit_regions(const orc_params*, const orc_mesh*, int ilevel, double* uold,
                          int nregion, const int* region_type /*0 square,1 point*/,
                          const double* x_center, const double* y_center, const double* z_center,
                          const double* length_x, const double* length_y, const double* length_z,
                          const double* exp_region,
                          const double* d_region, const double* u_region, const double* v_region,
                          const double* w_region, const double* p_region);
void orc_set_unew(const orc_params*, const orc_mesh*, int ilevel, const double* uold, double* unew);
void orc_set_uold(const orc_params*, const orc_mesh*, int ilevel, double* uold, const double* unew);
void orc_godunov_fine(const orc_params*, const orc_mesh*, int ilevel, double dt, const double* uold, double* unew, int nthreads);
/* returns dt_all = min(dt_in, CFL dt); sums[3] += mass, etot, eint (courant_fine.f90:1) */
double orc_courant_fine(const orc_params*, const orc_mesh*, int ilevel, double dt_in, const double* uold, double sums[3]);
void orc_make_boundary_hydro(const orc_params*, const orc_mesh*, int ilevel, double* uold);
/* bound_type 3 (imposed): conservative boundary_var of region ibound (0-based) */
void orc_set_boundary_var(int ibound, const double* var, int nvar);
void orc_upload_fine(const orc_params*, const orc_mesh*, int ilevel, double* uold);

/* run nstep level steps of a uniform (levelmin=levelmax) run: amr_step order
 * (amr/amr_step.f90:326,333,388,423,514).  dt_hist[nstep] receives the dt used. */
void orc_run_uniform(const orc_params*, const orc_mesh*, int ilevel, int nstep,
                     double* uold, double* unew, double* dt_hist, double* t_io, int nthreads);

/* AMR pieces (hydro/interpol_hydro.f90, amr/nbors_utils.f90:404) */
void orc_set_interpol(int interpol_type, int interpol_var);
void orc_getnborfather(const orc_mesh*, int ind_cell, int ilevel, int* ind_father /*[2*ndim+1]*/);
void orc_interpol_hydro(const orc_params*, const double* u1 /*[2*ndim+1][nvar]*/, double* u2 /*[2^ndim][nvar]*/);
void orc_interpol_cell(const orc_params*, const orc_mesh*, int ind_cell, int ilevel, const double* uold, double* u2);
orc_mesh* orc_mesh_new(int ndim, const int bound_type[6], int ngridmax, int nlevelmax);
orc_mesh* orc_mesh_new_box(int ndim, const int ndom[3], const int bound_type[6], int ngridmax, int nlevelmax);
void orc_mesh_set_list(orc_mesh*, int kind, int b, int ilevel, int n, const int* igrid);

/* pressure_fix: caller-owned divu / enew cell arrays [ncell] (NULL = off) and beta_fix (amr_parameters.f90:167)      */
void orc_set_pressure_fix(double* divu, double* enew, double beta_fix);
/* poisson: caller-owned acceleration f[ndim][ncell] (NULL = off): gravity predictor in ctoprim (umuscl.f90:932-938), gloc gather
 * in godfine1 (godunov_fine.f90:637-647), add_gravity_source_terms in set_uold (:237-289), gravity term of cmpdt            */
void orc_set_gravity(const double* f);
void orc_set_threads(int n);
void orc_set_amr_threads(int n);   /* flux phase of orc_godunov_fine(nthreads=1); results do not depend on it */
int orc_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif
