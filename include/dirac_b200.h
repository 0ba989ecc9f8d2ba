/*
 * dirac_b200 — Hopper (H100, sm_90a) implementation of the Dirac direction-dependent calibration hot
 * path.  C ABI only: plain pointers and sizes, host memory unless a name says otherwise.
 *
 * Two layers:
 *  (1) the reference's own entry points, same names / argument order / meaning / error behaviour,
 *      so that `sagecal_gpu` (src/MS/fullbatch_mode.cpp:371-446) links unchanged;
 *  (2) a thin `dirac_b200_*` layer that exposes the device-resident problem and the individual
 *      E-step passes (cost, gradient, normal equations), used by the parity tests, bench.py and
 *      the multi-GPU driver.
 *
 * Each declaration cites the reference interface it replaces (paths relative to the reference
 * repository root).
 */
#ifndef DIRAC_B200_H
#define DIRAC_B200_H

#ifdef __cplusplus
extern "C" {
#endif

/* ---- ABI-compatible restatement of the reference structs ------------------------------------ */

/* src/lib/Dirac/Dirac_common.h:190-195 */
typedef struct baseline_t_ {
  int sta1, sta2;
  unsigned char flag; /* 0 ok, 1 flagged, 2 excluded from the solution (uv cut) but subtracted */
} baseline_t;

/* src/lib/Dirac/Dirac_common.h:173-187 */
typedef struct clus_source_t_ {
  int N;  /* sources in this cluster */
  int id;
  double *ll, *mm, *nn, *sI, *sQ, *sU, *sV;
  double *ra, *dec;
  unsigned char *stype;
  void **ex;
  int nchunk; /* hybrid time chunks */
  int *p;     /* nchunk offsets into the parameter array */
  double *sI0, *sQ0, *sU0, *sV0, *f0, *spec_idx, *spec_idx1, *spec_idx2;
} clus_source_t;

/* src/lib/Dirac/Dirac_common.h:56-61 */
typedef struct exinfo_gaussian_ {
  double eX, eY, eP;
  double cxi, sxi, cphi, sphi;
  int use_projection;
} exinfo_gaussian;

/* src/lib/Dirac/Dirac_common.h:63-75 (exinfo_ring has the same layout) */
typedef struct exinfo_disk_ {
  double eX;
  double cxi, sxi, cphi, sphi;
  int use_projection;
} exinfo_disk;

/* src/lib/Dirac/Dirac_common.h:77-85 */
typedef struct exinfo_shapelet_ {
  int n0;        /* model order: n0*n0 modes */
  double beta;   /* scale */
  double *modes; /* n0*n0 coefficients */
  double eX, eY, eP;
  double cxi, sxi, cphi, sphi;
  int use_projection;
} exinfo_shapelet;

#define STYPE_POINT 0    /* src/lib/Radio/Dirac_radio.h:71-75 */
#define STYPE_GAUSSIAN 1
#define STYPE_DISK 2
#define STYPE_RING 3
#define STYPE_SHAPELET 4

/* solver_mode, src/lib/Dirac/Dirac.h:1607-1613 */
#define SM_LM_LBFGS 1
#define SM_OSLM_LBFGS 0
#define SM_OSLM_OSRLM_RLBFGS 3
#define SM_RLM_RLBFGS 2
#define SM_RTR_OSLM_LBFGS 4
#define SM_RTR_OSRLM_RLBFGS 5
#define SM_NSD_RLBFGS 6

/* ---- (1) reference entry points --------------------------------------------------------------
 * `coh` is `complex double *` in the reference (C99); it is declared `double *` here (re,im pairs,
 * identical memory) so that the header is valid C++ as well. */

/* replaces sagefit_visibilities, src/lib/Dirac/Dirac.h:1651 (lmfit.c:778-1053).
 * x: data in, residual out (in place).  pp: Jones in/out.  returns 0, or -1 if res_1 > res_0. */
int sagefit_visibilities(double *u, double *v, double *w, double *x, int N, int Nbase, int tilesz,
                         baseline_t *barr, clus_source_t *carr, double *coh, int M, int Mt,
                         double freq0, double fdelta, double *pp, double uvmin, int Nt,
                         int max_emiter, int max_iter, int max_lbfgs, int lbfgs_m, int gpu_threads,
                         int linsolv, int solver_mode, double nulow, double nuhigh, int randomize,
                         double *mean_nu, double *res_0, double *res_1);

/* GPU-build names of the same call, src/lib/Dirac/Dirac.h:1783,1788,1793 (lmfit_cuda.c:575,1102,
 * 1601; call sites src/MS/fullbatch_mode.cpp:442,446).  Aliases of sagefit_visibilities. */
int sagefit_visibilities_dual_pt_flt(double *u, double *v, double *w, double *x, int N, int Nbase,
                                     int tilesz, baseline_t *barr, clus_source_t *carr,
                                     double *coh, int M, int Mt, double freq0, double fdelta,
                                     double *pp, double uvmin, int Nt, int max_emiter,
                                     int max_iter, int max_lbfgs, int lbfgs_m, int gpu_threads,
                                     int linsolv, int solver_mode, double nulow, double nuhigh,
                                     int randomize, double *mean_nu, double *res_0, double *res_1);
int sagefit_visibilities_dual_pt(double *u, double *v, double *w, double *x, int N, int Nbase,
                                 int tilesz, baseline_t *barr, clus_source_t *carr, double *coh,
                                 int M, int Mt, double freq0, double fdelta, double *pp,
                                 double uvmin, int Nt, int max_emiter, int max_iter, int max_lbfgs,
                                 int lbfgs_m, int gpu_threads, int linsolv, int solver_mode,
                                 double nulow, double nuhigh, int randomize, double *mean_nu,
                                 double *res_0, double *res_1);
int sagefit_visibilities_dual_pt_one_gpu(double *u, double *v, double *w, double *x, int N,
                                         int Nbase, int tilesz, baseline_t *barr,
                                         clus_source_t *carr, double *coh, int M, int Mt,
                                         double freq0, double fdelta, double *pp, double uvmin,
                                         int Nt, int max_emiter, int max_iter, int max_lbfgs,
                                         int lbfgs_m, int gpu_threads, int linsolv,
                                         int solver_mode, double nulow, double nuhigh,
                                         int randomize, double *mean_nu, double *res_0,
                                         double *res_1);

/* replaces bfgsfit_visibilities, src/lib/Dirac/Dirac.h:1683 (lmfit.c:1127-1212) and its GPU-build
 * twin bfgsfit_visibilities_gpu, Dirac.h:1690 (lmfit_cuda.c:1375). */
int bfgsfit_visibilities(double *u, double *v, double *w, double *x, int N, int Nbase, int tilesz,
                         baseline_t *barr, clus_source_t *carr, double *coh, int M, int Mt,
                         double freq0, double fdelta, double *pp, double uvmin, int Nt,
                         int max_lbfgs, int lbfgs_m, int gpu_threads, int solver_mode,
                         double mean_nu, double *res_0, double *res_1);
int bfgsfit_visibilities_gpu(double *u, double *v, double *w, double *x, int N, int Nbase,
                             int tilesz, baseline_t *barr, clus_source_t *carr, double *coh, int M,
                             int Mt, double freq0, double fdelta, double *pp, double uvmin, int Nt,
                             int max_lbfgs, int lbfgs_m, int gpu_threads, int solver_mode,
                             double mean_nu, double *res_0, double *res_1);

/* replaces precalculate_coherencies, src/lib/Radio/Dirac_radio.h:209 (predict.c:503-578).
 * x: coherencies out, [row][cluster][4] complex.  Also sets barr[].flag=2 outside [uvmin,uvmax]. */
int precalculate_coherencies(double *u, double *v, double *w, double *x, int N, int Nbase,
                             baseline_t *barr, clus_source_t *carr, int M, double freq0,
                             double fdelta, double tdelta, double dec0, double uvmin, double uvmax,
                             int Nt);

/* replaces predict_visibilities_multifreq, src/lib/Radio/Dirac_radio.h:659 (residual.c:1257-1340) */
int predict_visibilities_multifreq(double *u, double *v, double *w, double *x, int N, int Nbase,
                                   int tilesz, baseline_t *barr, clus_source_t *carr, int M,
                                   double *freqs, int Nchan, double fdelta, double tdelta,
                                   double dec0, int Nt, int add_to_data);

/* replaces calculate_residuals_multifreq, src/lib/Radio/Dirac_radio.h:652 (residual.c:940-1061,
 * residual_threadfn_multifreq :681-938): full-resolution residual, x[chan][row][8] -= sum over the
 * clusters with id >= 0 of J_p C_k(chan) J_q^H with the coherencies re-predicted from the sources at
 * every channel, then the correction of every row by the inverse Jones (J + rho I)^-1 of the cluster
 * whose id is ccid (none if no cluster has that id).  phase_only != 0: the correction uses only the
 * phases of the cluster's jointly diagonalised solutions (manifold_average.c:399-610). */
int calculate_residuals_multifreq(double *u, double *v, double *w, double *p, double *x, int N,
                                  int Nbase, int tilesz, baseline_t *barr, clus_source_t *carr, int M,
                                  double *freqs, int Nchan, double fdelta, double tdelta, double dec0,
                                  int Nt, int ccid, double rho, int phase_only);

/* helpers the driver calls directly: src/lib/Dirac/Dirac.h generate_baselines
 * (baseline_utils.c:469), preset_flags_and_data (baseline_utils.c:239).  Bit-exact index work. */
int generate_baselines(int Nbase, int tilesz, int N, baseline_t *barr, int Nt);
int preset_flags_and_data(int Nbase, double *flag, baseline_t *barr, double *x, int Nt);
/* uv-distance taper of the data (driver option -W; src/lib/Dirac/Dirac.h:841, updatenu.c:339-420):
 * x[8 row ..] *= 1 / (1 + 1.8 exp(-0.05 d)), d = |(u,v)| freq0 <= 400 wavelengths.  Host, bit-exact. */
void whiten_data(int Nbase, double *x, double *u, double *v, double freq0, int Nt);

/* ---- (2) thin device layer ------------------------------------------------------------------- */

typedef struct dirac_b200_problem dirac_b200_problem; /* opaque, device resident */

/* Upload one solve interval.  coh may be NULL when the coherencies are generated on the device
 * (dirac_b200_precalculate).  Replaces the per-call H2D churn of clmfit_fl.c:193-225 /
 * lbfgs_cuda.c:93-131 with one resident copy.  Exits (reference convention) on CUDA failure. */
dirac_b200_problem *dirac_b200_create(int N, int Nbase, int tilesz, const baseline_t *barr,
                                      const clus_source_t *carr, int M, int Mt, const double *coh,
                                      const double *x);
void dirac_b200_destroy(dirac_b200_problem *pr);
/* replace the data vector (8*Nbase*tilesz doubles, API layout) */
void dirac_b200_set_data(dirac_b200_problem *pr, const double *x);
/* device-side precalculate_coherencies (predict.c:345-497) into the resident planar layout;
 * writes the uv-cut flags (value 2) into the resident flag array and, if barr != NULL, into barr. */
void dirac_b200_precalculate(dirac_b200_problem *pr, const double *u, const double *v,
                             const double *w, const clus_source_t *carr, double freq0,
                             double fdelta, double uvmin, double uvmax, baseline_t *barr);
/* copy the resident coherencies back in API layout ([row][cluster][4] complex) */
void dirac_b200_get_coherencies(dirac_b200_problem *pr, double *coh);

/* model / residual / cost over all clusters at Jones pp (minimize_viz_full_pth, lmfit.c:692;
 * cost_func / robust_cost_func, robust_lbfgs.c:674,707).
 * out_mode: 0 none, 1 out = x - V, 2 out = V (8*Nbase*tilesz doubles, API layout; out may be NULL)
 * cost_mode: 0 none, 1 sum e^2, 2 sum log(1+e^2/nu) */
double dirac_b200_predict(dirac_b200_problem *pr, const double *pp, double *out, int out_mode,
                          int cost_mode, double nu);
/* LBFGS gradient in the reference's sign convention (func_grad / func_grad_robust,
 * robust_lbfgs.c:569-669,322-416); g has 8*N*Mt doubles. */
void dirac_b200_grad(dirac_b200_problem *pr, const double *pp, double *g, int robust, double nu);
/* Student's-t cost sum log(1+e^2/nu) over the rows [row0, row0+nrows) alone (rows count baselines
 * times timeslots, the window may cut a timeslot; robust_cost_func_batch,
 * robust_batchmode_lbfgs.c:822-846).  A window with nrows <= 0 is empty: cost 0. */
double dirac_b200_cost_window(dirac_b200_problem *pr, const double *pp, long long row0,
                              long long nrows, double nu);
/* gradient of that cost over the same rows, in the sign of the reference's minibatch gradient
 * (robust_grad_func_batch, robust_batchmode_lbfgs.c:347-600): the NEGATIVE of what
 * dirac_b200_grad(robust=1) returns for those rows; g has 8*N*Mt doubles, 0 for an empty window. */
void dirac_b200_grad_window(dirac_b200_problem *pr, const double *pp, double *g, long long row0,
                            long long nrows, double nu);
/* per-cluster normal equations at pblk (8N doubles) for hybrid chunk `chunk` of cluster `clus`
 * against the hidden data xd (API layout, full interval): JTJ (8N x 8N), JTe (8N), returns
 * ||e||^2.  Equivalent of mylm_jac_single_pth + dgemm/dgemv (lmfit.c:484, clmfit.c:307-315). */
double dirac_b200_normal_eq(dirac_b200_problem *pr, int clus, int chunk, const double *pblk,
                            const double *xd, double *JTJ, double *JTe);

/* the same system with the sqrt-weights of the robust LM applied to the rows of J and to e
 * (robustlm.c:2298-2316); wt has 8 weights per row of the full interval, API layout. */
double dirac_b200_normal_eq_weighted(dirac_b200_problem *pr, int clus, int chunk,
                                     const double *pblk, const double *xd, const double *wt,
                                     double *JTJ, double *JTe);

/* sagefit_visibilities (lmfit.c:778-1053) on an already resident problem: no upload, Jones pp
 * in/out on the host, final residual to x_out (API layout) unless x_out == NULL.  This is what the
 * drop-in sagefit_visibilities calls between dirac_b200_create and dirac_b200_destroy. */
int dirac_b200_sagefit(dirac_b200_problem *pr, double *pp, double *x_out, int max_emiter,
                       int max_iter, int max_lbfgs, int lbfgs_m, int linsolv, int solver_mode,
                       double nulow, double nuhigh, int randomize, double *mean_nu, double *res_0,
                       double *res_1);

/* ---- cluster sharding over the GPUs of one box (one process per GPU) --------------------------
 * The reference splits clusters over GPUs with host pthreads and merges on the host
 * (src/lib/Radio/predict_withbeam_cuda.c:713-794, src/lib/Dirac/lmfit_cuda.c:1801-1950).  Here a
 * rank holds the coherencies of its own contiguous block of clusters only; carr_local[k].p[] are
 * offsets into the GLOBAL Jones vector of npar_global doubles, which is replicated like the data.
 * The host supplies the collective: `allreduce(dev, count, stream, user)` must sum `count` doubles
 * at device address `dev` over all ranks, enqueued on `stream` (an NCCL all-reduce).  Every rank
 * calls dirac_b200_sagefit with identical arguments and gets identical pp / residual back.
 * beta: hidden-data weight of the residual during a sweep (SAGE); <= 0 selects 1/world, the
 * generalisation of the reference's 0.5 for two concurrent clusters (lmfit_cuda.c:1832-1842). */
dirac_b200_problem *dirac_b200_create_shard(int N, int Nbase, int tilesz, const baseline_t *barr,
                                            const clus_source_t *carr_local, int M_local,
                                            int Mt_local, long long npar_global, const double *coh,
                                            const double *x);
void dirac_b200_set_comm(dirac_b200_problem *pr, int rank, int world,
                         void (*allreduce)(void *dev, long long count, void *stream, void *user),
                         void *user, int m_global, int k_global0, double beta);
/* The collective itself: with allreduce == NULL in dirac_b200_set_comm the library calls
 * ncclAllReduce (fp64, sum, in place) on its own stream through a process-wide communicator:
 *   rank 0:     dirac_b200_nccl_unique_id(id)         (128 bytes; the host distributes them: MPI_Bcast,
 *   every rank: dirac_b200_nccl_init(rank, world, id)   a file, a TCP store ...)  [collective call]
 * NCCL is bound at run time (an already loaded libnccl.so.2, $DIRAC_B200_NCCL_LIB, libnccl.so.2).
 * A C host (the reference driver) needs nothing else for the multi-GPU path; the callback remains
 * for hosts that bring their own collective.  All return 0 on success. */
int dirac_b200_nccl_unique_id(char *id128);
int dirac_b200_nccl_init(int rank, int world, const char *id128);
void dirac_b200_nccl_finalize(void);
int dirac_b200_nccl_ready(void);
/* collectives issued since the last reset: calls, bytes, host seconds spent enqueueing them */
void dirac_b200_comm_stats(unsigned long long *calls, unsigned long long *bytes,
                           double *enqueue_seconds, int reset);

/* ---- consensus (ADMM) calibration over frequency subbands, one subband per GPU -------------------
 * (BASELINE.json config 5; src/MPI/sagecal_master.cpp:844-877, sagecal_slave.cpp:831-878,
 * src/lib/Dirac/consensus_poly.c, admm_solve.c).  No master process: the sum over subbands is ONE
 * all-reduce of Npoly*8*N*Mt doubles per ADMM iteration on the library's stream (the communicator of
 * dirac_b200_nccl_init, or the callback of dirac_b200_set_comm), every rank applies the replicated
 * pseudo-inverse and its own basis row itself. */
/* replaces setup_polynomials (consensus_poly.c:38): B[f*Npoly + p], type 0 ordinary, 1 normalised,
 * 2 Bernstein, 3 mixed powers.  Host arithmetic, no GPU needed. */
int dirac_b200_consensus_basis(double *B, int Npoly, int Nf, const double *freqs, double freq0,
                               int type);
/* replaces find_prod_inverse_full (consensus_poly.c:465): Bi[k] = pinv(sum_f rho[k + f*M] B_f B_f^T),
 * Npoly x Npoly per cluster.  Host arithmetic, no GPU needed. */
int dirac_b200_consensus_prod_inverse(const double *B, double *Bi, int Npoly, int Nf, int M,
                                      const double *rho);
/* one exchange for this rank's subband (J, Y, BZ: host vectors laid out like pp; rho[M]; Bf[Npoly] =
 * this subband's basis row; Bi[M][Npoly][Npoly]):  Y += rho J;  z = B_f (x) Y summed over the ranks;
 * BZ = B_f Bi z;  Y -= rho BZ.  *primal = ||J - BZ||, *dual = ||BZ - BZ_old||. */
int dirac_b200_consensus_step(dirac_b200_problem *pr, const double *J, double *Y, double *BZ,
                              const double *rho, const double *Bf, const double *Bi, int Npoly,
                              double *primal, double *dual);
/* the J-update of one ADMM iteration on a resident problem, and its drop-in form: replaces
 * sagefit_visibilities_admm (Dirac.h:1521, admm_solve.c:221) and its GPU-build twin (:1533).  Each
 * cluster's cost carries y^T (p - bz) + rho/2 |p - bz|^2.
 *   dirac_b200_sagefit_admm_rtr: as the reference solves it -- every visit by the robust Riemannian
 *     trust-region solver on the augmented cost (rtr_solve_nocuda_robust_admm, admm_solve.c:331-352);
 *     what sagefit_visibilities_admm runs.
 *   dirac_b200_sagefit_admm: this library's LM on the same cost (Gauss-Newton system with rho/2 on the
 *     diagonal): other iterates, the same ADMM fixed point; dirac_b200_set_option("admm_lm", 1)
 *     makes the drop-in entry point use it. */
int dirac_b200_sagefit_admm_rtr(dirac_b200_problem *pr, double *pp, double *x_out, const double *Y,
                                const double *BZ, const double *admm_rho, int max_emiter,
                                int max_iter, double nulow, double nuhigh, int randomize,
                                double *mean_nu, double *res_0, double *res_1);
int dirac_b200_sagefit_admm(dirac_b200_problem *pr, double *pp, double *x_out, const double *Y,
                            const double *BZ, const double *admm_rho, int max_emiter, int max_iter,
                            int linsolv, int randomize, double *res_0, double *res_1);
int sagefit_visibilities_admm(double *u, double *v, double *w, double *x, int N, int Nbase, int tilesz,
                              baseline_t *barr, clus_source_t *carr, double *coh, int M, int Mt,
                              double freq0, double fdelta, double *pp, double *Y, double *BZ,
                              double uvmin, int Nt, int max_emiter, int max_iter, int max_lbfgs,
                              int lbfgs_m, int gpu_threads, int linsolv, int solver_mode, double nulow,
                              double nuhigh, int randomize, double *admm_rho, double *mean_nu,
                              double *res_0, double *res_1);
int sagefit_visibilities_admm_dual_pt_flt(double *u, double *v, double *w, double *x, int N, int Nbase,
                                          int tilesz, baseline_t *barr, clus_source_t *carr,
                                          double *coh, int M, int Mt, double freq0, double fdelta,
                                          double *pp, double *Y, double *BZ, double uvmin, int Nt,
                                          int max_emiter, int max_iter, int max_lbfgs, int lbfgs_m,
                                          int gpu_threads, int linsolv, int solver_mode, double nulow,
                                          double nuhigh, int randomize, double *admm_rho,
                                          double *mean_nu, double *res_0, double *res_1);

/* run on a caller-supplied CUDA stream (cudaStream_t) instead of a private one; NULL restores the
 * default.  Affects problems created afterwards and the reference entry points. */
void dirac_b200_set_stream(void *stream);

/* test / tuning switches; returns 0, or -1 for an unknown name.
 *   "rtr_nu_unjoined"  robust RTR / NSD (solver_mode 5, 6): update nu as if the reference's worker
 *               threads' partial sums, which it reads before joining the threads
 *               (rtr_solve_robust.c:361-370), were all still zero -- what the threaded reference does
 *               on most runs; default 0: the sums are complete, as the code was meant
 *   "admm_lm"   sagefit_visibilities_admm solves with this library's LM instead of the robust RTR
 *   "cp_rows"   timeslots per CTA of the gradient-carrying cluster pass (0: one wave over the SMs);
 *               the parity tests use it to drive the multi-row TMA ring on small problems */
int dirac_b200_set_option(const char *name, int value);

/* LM accept/reject decisions that were taken at rounding level (|dF| <= 1e-11 ||e||^2) since the last
 * reset: on such runs (typical for the ordered-subsets modes 0 and 3 once trial steps get rejected
 * down to ~1e-15 |p|) the iterates of two correct implementations diverge, the reference's own CPU
 * path included; parity of the solved Jones is defined for runs where this stays 0. */
long dirac_b200_noise_decisions(int reset);

/* extract_phases (manifold_average.c:399-610): unit-modulus diagonal of the N Jones matrices of one
 * (cluster, chunk) after niter rounds of joint diagonalisation by Jacobi rotations; what the
 * phase_only correction of calculate_residuals_multifreq inverts.  Host arithmetic, no GPU needed. */
int dirac_b200_extract_phases(const double *p, double *pout, int N, int niter);

/* ---- station beams (SURVEY.md 8f-4) -------------------------------------------------------------------
 * Dirac_common.h:94-162 */
#define ELEM_LBA 0
#define ELEM_HBA 1
#define STAT_NONE 0
#define STAT_SINGLE 1
#define STAT_TILE 2
#define HBA_TILE_SIZE 16
#define DOBEAM_NONE 0
#define DOBEAM_ARRAY 1
#define DOBEAM_FULL 2
#define DOBEAM_ELEMENT 3
#define DOBEAM_ARRAY_WB 4
#define DOBEAM_FULL_WB 5
#define DOBEAM_ELEMENT_WB 6
typedef struct elementcoff_ {
  int M;      /* model order */
  int Nmodes; /* M (M+1) / 2 */
  int Nf;     /* frequencies of the wide-band tables (1 otherwise) */
  double beta;
  double *pattern_phi;   /* complex, Nmodes*Nf */
  double *pattern_theta; /* complex, Nmodes*Nf */
  double *preamble;      /* Nmodes */
} elementcoeff;
/* Dirac_radio.h:472,485,489 and their GPU-build twins :516,521,525 (predict_withbeam.c:553-723,
 * 1219-1440, 1989-2315): the three coherency / prediction calls with the station beam towards every
 * source folded in.  Array factor (STAT_SINGLE, STAT_TILE) and element beam (the caller's
 * elementcoeff tables, set_elementcoeffs stays in the reference library) per timeslot and channel;
 * doBeam DOBEAM_ARRAY / _FULL / _ELEMENT and their wide-band variants.  The lunar element beam
 * (DOBEAM_ALO, needs CSPICE) is refused. */
int precalculate_coherencies_withbeam(
    double *u, double *v, double *w, double *x, int N, int Nbase, baseline_t *barr,
    clus_source_t *carr, int M, double freq0, double fdelta, double tdelta, double dec0, double uvmin,
    double uvmax, int bf_type, double b_ra0, double b_dec0, double ph_ra0, double ph_dec0,
    double ph_freq0, double *longitude, double *latitude, double *time_utc, int tilesz, int *Nelem,
    double **xx, double **yy, double **zz, elementcoeff *ecoeff, int doBeam, int Nt);
int precalculate_coherencies_withbeam_gpu(
    double *u, double *v, double *w, double *x, int N, int Nbase, baseline_t *barr,
    clus_source_t *carr, int M, double freq0, double fdelta, double tdelta, double dec0, double uvmin,
    double uvmax, int bf_type, double b_ra0, double b_dec0, double ph_ra0, double ph_dec0,
    double ph_freq0, double *longitude, double *latitude, double *time_utc, int tilesz, int *Nelem,
    double **xx, double **yy, double **zz, elementcoeff *ecoeff, int doBeam, int Nt);
/* Dirac_radio.h:221,479,534 (predict.c:745-816): coherencies of Nchan channels,
 * x[chan][row][cluster][4]: the input of bfgsfit_minibatch_*.  Flag 2 for rows shorter than uvmin at
 * the first channel or longer than uvmax at the last. */
int precalculate_coherencies_multifreq(double *u, double *v, double *w, double *x, int N, int Nbase,
                                       baseline_t *barr, clus_source_t *carr, int M, double *freqs,
                                       int Nchan, double fdelta, double tdelta, double dec0,
                                       double uvmin, double uvmax, int Nt);
int precalculate_coherencies_multifreq_withbeam(
    double *u, double *v, double *w, double *x, int N, int Nbase, baseline_t *barr,
    clus_source_t *carr, int M, double *freqs, int Nchan, double fdelta, double tdelta, double dec0,
    double uvmin, double uvmax, int bf_type, double b_ra0, double b_dec0, double ph_ra0,
    double ph_dec0, double ph_freq0, double *longitude, double *latitude, double *time_utc, int tilesz,
    int *Nelem, double **xx, double **yy, double **zz, elementcoeff *ecoeff, int doBeam, int Nt);
int precalculate_coherencies_multifreq_withbeam_gpu(
    double *u, double *v, double *w, double *x, int N, int Nbase, baseline_t *barr,
    clus_source_t *carr, int M, double *freqs, int Nchan, double fdelta, double tdelta, double dec0,
    double uvmin, double uvmax, int bf_type, double b_ra0, double b_dec0, double ph_ra0,
    double ph_dec0, double ph_freq0, double *longitude, double *latitude, double *time_utc, int tilesz,
    int *Nelem, double **xx, double **yy, double **zz, elementcoeff *ecoeff, int doBeam, int Nt);
int predict_visibilities_multifreq_withbeam(
    double *u, double *v, double *w, double *x, int N, int Nbase, int tilesz, baseline_t *barr,
    clus_source_t *carr, int M, double *freqs, int Nchan, double fdelta, double tdelta, double dec0,
    int bf_type, double b_ra0, double b_dec0, double ph_ra0, double ph_dec0, double ph_freq0,
    double *longitude, double *latitude, double *time_utc, int *Nelem, double **xx, double **yy,
    double **zz, elementcoeff *ecoeff, int doBeam, int Nt, int add_to_data);
int predict_visibilities_multifreq_withbeam_gpu(
    double *u, double *v, double *w, double *x, int N, int Nbase, int tilesz, baseline_t *barr,
    clus_source_t *carr, int M, double *freqs, int Nchan, double fdelta, double tdelta, double dec0,
    int bf_type, double b_ra0, double b_dec0, double ph_ra0, double ph_dec0, double ph_freq0,
    double *longitude, double *latitude, double *time_utc, int *Nelem, double **xx, double **yy,
    double **zz, elementcoeff *ecoeff, int doBeam, int Nt, int add_to_data);
int calculate_residuals_multifreq_withbeam(
    double *u, double *v, double *w, double *p, double *x, int N, int Nbase, int tilesz,
    baseline_t *barr, clus_source_t *carr, int M, double *freqs, int Nchan, double fdelta,
    double tdelta, double dec0, int bf_type, double b_ra0, double b_dec0, double ph_ra0,
    double ph_dec0, double ph_freq0, double *longitude, double *latitude, double *time_utc,
    int *Nelem, double **xx, double **yy, double **zz, elementcoeff *ecoeff, int doBeam, int Nt,
    int ccid, double rho, int phase_only);
int calculate_residuals_multifreq_withbeam_gpu(
    double *u, double *v, double *w, double *p, double *x, int N, int Nbase, int tilesz,
    baseline_t *barr, clus_source_t *carr, int M, double *freqs, int Nchan, double fdelta,
    double tdelta, double dec0, int bf_type, double b_ra0, double b_dec0, double ph_ra0,
    double ph_dec0, double ph_freq0, double *longitude, double *latitude, double *time_utc,
    int *Nelem, double **xx, double **yy, double **zz, elementcoeff *ecoeff, int doBeam, int Nt,
    int ccid, double rho, int phase_only);

/* ---- multi-channel minibatch (stochastic) robust LBFGS, SURVEY.md 8f-3 ------------------------------
 * persistent_data_t: the reference declares it twice (Dirac.h:86-110 without HAVE_CUDA, :196-226 with);
 * the two layouts agree up to `Nt`, and this library touches nothing beyond that prefix (the running
 * averages and the iteration count of the on-line variance live behind the curvature pairs in `s`), so
 * a caller compiled against either reference header can pass its own struct. */
typedef struct persistent_data_t_ {
  double *y, *s; /* curvature pairs, lbfgs_m x m each (allocated by lbfgs_persist_init) */
  double *rho;   /* 1 / y^T s */
  int nfilled;   /* pairs in use, 0..lbfgs_m */
  int vacant;    /* next slot, cycles through 0..lbfgs_m-1 */
  int lbfgs_m;
  int m;
  int Nt;
  /* (the reference's further fields differ between its builds and are not used) */
} persistent_data_t;
/* lbfgs.c:954-1045 */
int lbfgs_persist_init(persistent_data_t *pt, int Nminibatch, int m, int n, int lbfgs_m, int Nt);
int lbfgs_persist_clear(persistent_data_t *pt);
int lbfgs_persist_reset(persistent_data_t *pt);
/* Dirac.h:317,343 (robust_batchmode_lbfgs.c:1446-1577): x and coh hold Nf channels
 * ([channel][row][8] and [channel][row][cluster][4] complex), ONE set of Jones p for all of them;
 * Student's-t cost with fixed robust_nu, LBFGS with Armijo backtracking, curvature pairs and the
 * gradient's on-line variance carried from minibatch to minibatch in *indata.  res = cost / n.
 * _consensus adds y^T (p - z) + rho/2 |p - z|^2 per (cluster, chunk) block. */
int bfgsfit_minibatch_visibilities(double *u, double *v, double *w, double *x, int N, int Nbase,
                                   int tilesz, baseline_t *barr, clus_source_t *carr, double *coh,
                                   int M, int Mt, double *freqs, int Nf, double fdelta, double *p,
                                   int Nt, int max_lbfgs, int lbfgs_m, int gpu_threads,
                                   int solver_mode, double robust_nu, double *res_0, double *res_1,
                                   persistent_data_t *indata, int nminibatch, int totalminibatch);
int bfgsfit_minibatch_consensus(double *u, double *v, double *w, double *x, int N, int Nbase,
                                int tilesz, baseline_t *barr, clus_source_t *carr, double *coh, int M,
                                int Mt, double *freqs, int Nf, double fdelta, double *p, double *y,
                                double *z, double *rho, int Nt, int max_lbfgs, int lbfgs_m,
                                int gpu_threads, int solver_mode, double robust_nu, double *res_0,
                                double *res_1, persistent_data_t *indata, int nminibatch,
                                int totalminibatch);
/* The same two calls with the argument list the reference declares under HAVE_CUDA (Dirac.h:315-319,
 * 343-347; call sites minibatch_mode.cpp:438, minibatch_consensus_mode.cpp:536): `short *hbb`
 * (2 shorts per row: stations, or -1 -1 for a flagged row; rearrange_baselines, baseline_utils.c:123-145)
 * and `int *ptoclus` (2 ints per cluster: nchunk and the offset of its first chunk in p, the chunks of a
 * cluster contiguous) in place of barr / carr.  One symbol cannot carry both signatures: a driver
 * compiled with HAVE_CUDA binds these names (INTEGRATION.md section 2). */
int bfgsfit_minibatch_visibilities_hbb(double *u, double *v, double *w, double *x, int N, int Nbase,
                                       int tilesz, short *hbb, int *ptoclus, double *coh, int M, int Mt,
                                       double *freqs, int Nf, double fdelta, double *p, int Nt,
                                       int max_lbfgs, int lbfgs_m, int gpu_threads, int solver_mode,
                                       double robust_nu, double *res_0, double *res_1,
                                       persistent_data_t *indata, int nminibatch, int totalminibatch);
int bfgsfit_minibatch_consensus_hbb(double *u, double *v, double *w, double *x, int N, int Nbase,
                                    int tilesz, short *hbb, int *ptoclus, double *coh, int M, int Mt,
                                    double *freqs, int Nf, double fdelta, double *p, double *y,
                                    double *z, double *rho, int Nt, int max_lbfgs, int lbfgs_m,
                                    int gpu_threads, int solver_mode, double robust_nu, double *res_0,
                                    double *res_1, persistent_data_t *indata, int nminibatch,
                                    int totalminibatch);
/* host helper behind them: baseline_t rows from hbb (stations by position in the canonical order, flag 1
 * where hbb marks the row); -1 if an unflagged row does not carry the canonical pair of its position. */
int dirac_b200_barr_from_hbb(int N, int Nbase, int tilesz, const short *hbb, baseline_t *barr);

/* Device memory freed by dirac_b200_destroy is kept (up to 40 % of the device's memory,
 * $DIRAC_B200_CACHE_GB overrides, 0 disables) and handed out again when a problem of the same shape
 * is created: the driver calls tile after tile with the same sizes, and cudaMalloc / cudaFree of the
 * coherencies alone cost 50-350 ms at 512 stations.  This returns all of it to the driver. */
void dirac_b200_release_cache(void);

/* number of kernels this library launched since load (bench.py's gpu_launches) */
unsigned long long dirac_b200_launch_count(void);
/* per-launch CUDA-event timing of the library's kernels on their launching stream.
 * kind: 0 full predict, 1 LBFGS gradient, 2 k_cluster_pass*, 3 k_coh_gram, 4 assembly, 5 damped solve
 * (k_chol_solve / k_tri_solve / batched potrf), 6 k_weighted_jtj, 7 line setup, 8 k_cluster_pass
 * without gradient (ADD / SUB / cost-only; kind 2 then counts the gradient-carrying INIT / TRIAL passes),
 * 9 k_rtr_stats (row condensation of the RTR / NSD solvers), 10 k_rtr_eval, 13 k_stream_band (cost
 * or residual of every channel of a minibatch band), 14 k_grad_tma_band (its gradient), 15 k_beam_tables
 * (station beam tables), 16 k_sky_predict<0> of a stochastic interval (coherencies into device
 * storage).  enable(1) clears the
 * records; read returns the launch count and sums the elapsed
 * milliseconds and the algorithmic bytes of the recorded launches of that kind. */
unsigned long long dirac_b200_kernel_count(int kind); /* launches of `kind` since load */
void dirac_b200_profile_enable(int on);
int dirac_b200_profile_read(int kind, double *ms, double *bytes);

/* host synchronisations (stream / event waits of the host-side solver logic) since the last reset and
 * the seconds the host spent blocked in them */
void dirac_b200_host_stats(unsigned long long *syncs, double *wait_seconds, int reset);

/* ---- the dense solver of the LM step on its own (diagnostics, tests) ---------------------------
 * (A + mu I) x = b for a symmetric positive definite A (n x n, column-major, only the lower triangle
 * is read; n <= 512) on one thread-block cluster: blocked Cholesky, both substitutions, one kernel
 * (replaces dpotrf + dpotrs of clmfit.c:373-395).  Host buffers.  *info as dpotrf (0, or the index
 * of the first non-positive pivot).  Returns 0, or -1 if the device grants no 8/16-CTA cluster.
 * dirac_b200_tri_solve: L L^T x = b for an existing factor L (column-major lower, ld = n), i.e.
 * dpotrs; reps > 0 additionally times `reps` back-to-back solves (us per solve in *us).
 * dirac_b200_tri_solve_ld: the same for a factor with leading dimension ld >= n (the batched
 * factorisation of the LM leaves its factors at ld = 32*ceil(n/32)). */
int dirac_b200_spd_solve(int n, const double *A, const double *b, double mu, double *x, int *info);
int dirac_b200_tri_solve(int n, const double *L, const double *b, double *x, int reps, double *us);
int dirac_b200_tri_solve_ld(int n, const double *L, int ld, const double *b, double *x, int reps,
                            double *us);
/* the same for systems beyond the cluster kernels (n > 512, a multiple of 64, e.g. 4096 at 512
 * stations): blocked dataflow substitutions over n/64 co-resident CTAs (replaces cusolverDnDpotrs
 * behind cuSOLVER's dpotrf).  Returns -1 when the size is not handled. */
int dirac_b200_bigtri_solve(int n, const double *L, const double *b, double *x, int reps, double *us);

#ifdef __cplusplus
}
#endif

/* simulation with solutions (predict_visibilities_multifreq_withsol and its beam variants) */
#include "dirac_b200_withsol.h"
/* coherencies of the diffuse cluster from a spatial model (recalculate_diffuse_coherencies) */
#include "dirac_b200_diffuse.h"
/* per-channel refinement (calculate_residuals and the channel loop on one resident problem) */
#include "dirac_b200_channels.h"
/* stochastic calibration of a whole solution interval (the minibatch driver's loop in one call) */
#include "dirac_b200_stochastic.h"
/* federated stochastic calibration (the projectback manifold average and the slave's ADMM step) */
#include "dirac_b200_federated.h"
/* influence-function diagnostics (calculate_diagnostics_gpu, driver option -i 1) */
#include "dirac_b200_diagnostics.h"
#endif
