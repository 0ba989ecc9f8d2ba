// Per-cluster Levenberg-Marquardt on the device-resident problem.
//
// Control flow mirrors clevmar_der_single_nocuda (clmfit.c:219-529), oslevmar_der_single_nocuda
// (clmfit.c:1281-1640), rlevmar_der_single_nocuda (robustlm.c:2008-2600) and
// osrlevmar_der_single_nocuda (robustlm.c:2607-3250) decision for decision; what differs is how
// the quantities are produced:
//   e, ||e||^2, J^T e   one streaming pass over (hidden data, coh_k)          k_cluster_pass
//   J^T J               assembled from the per-baseline Gram tensors           k_coh_gram/
//                       (8N > 512: damped, lower triangle, factored in place)  k_assemble_tiles
//                       (weighted, robust LM: one streaming pass)              k_weighted_jtj
//   (J^T J + mu I) dp   linsolv 0: k_chol_solve / k_tri_solve on one thread-block cluster
//                       (kernels_chol.cu; cuSOLVER potrf/potrs when 8N > 512 or no cluster)
//                       (8N > 1024: the sweep's first systems by one blocked batch, bigchol.cu)
//                       linsolv 1, 2: cuSOLVER geqrf+ormqr+trsm | gesvd
// The dense n x 8N Jacobian of the reference (7.2 GB per cluster at N=62, T=120) never exists.
#include <float.h>
#include <math.h>
#include <string.h>
#include <vector>

#include "../../include/dirac_b200.h"
#include "problem.h"

#define CS_CHECK(call)                                                                     \
  do {                                                                                     \
    cusolverStatus_t s__ = (call);                                                         \
    if (s__ != CUSOLVER_STATUS_SUCCESS) {                                                  \
      fprintf(stderr, "dirac_b200: cuSOLVER error %d at %s:%d\n", (int)s__, __FILE__, __LINE__); \
      exit(1);                                                                             \
    }                                                                                      \
  } while (0)
#define CB_CHECK(call)                                                                     \
  do {                                                                                     \
    cublasStatus_t s__ = (call);                                                           \
    if (s__ != CUBLAS_STATUS_SUCCESS) {                                                    \
      fprintf(stderr, "dirac_b200: cuBLAS error %d at %s:%d\n", (int)s__, __FILE__, __LINE__); \
      exit(1);                                                                             \
    }                                                                                      \
  } while (0)

extern "C" {
void db_launch_weighted_jtj(const WeightedJtjArgs *a, int ntile, cudaStream_t st);
void db_launch_sum_abs(const double2 *v, long long R, long long r0, long long r1, double *partials,
                       double *out, unsigned int *counter, cudaStream_t st);
void db_launch_update_weights(const double2 *e, double2 *wt, long long R, long long r0,
                              long long r1, double nu0, double *partials, double *out,
                              unsigned int *counter, cudaStream_t st);
void db_launch_scale_vis(double2 *v, long long R, long long r0, long long r1, double alpha,
                         int set_const, cudaStream_t st);
void db_launch_extract_diag(const double *A, double *dst, int n, cudaStream_t st);
void db_launch_lm_step(const double *p, const double *Dp, const double *jte, double *pnew,
                       double *sc, double *zero, int n, cudaStream_t st);
void db_launch_os_shift(const double2 *e, const double2 *wt, double2 *eps, double2 *wout, long long R,
                        long long row_sub0, long long nrow_sub, long long row_chunk0, long long kl,
                        long long nJ, cudaStream_t st);
}

template <typename T>
static T *dalloc(size_t n) {
  return (T *)db_malloc(n * sizeof(T) + 16);
}

void db_lm_init(dirac_b200_problem *pr) {
  LMWork &w = pr->lm;
  if (w.ready) return;
  DevProblem &d = pr->d;
  const int n8 = 8 * d.N;
  w.n8 = n8;
  w.T = dalloc<double>((size_t)d.Mt * d.Nbase * 16);
  w.T_valid = (unsigned char *)calloc(d.Mt, 1);
  w.Tsub = dalloc<double>((size_t)d.Nbase * 16);
  w.JTJ0 = dalloc<double>((size_t)n8 * n8);
  w.JTJ = dalloc<double>((size_t)n8 * n8);
  w.JTe = d.scal + 64 + n8;       // mailbox, see create_impl
  w.JTe_new = d.scal + 64 + 2 * n8;
  w.Hst = dalloc<double>((size_t)4 * d.N);
  w.Dp = d.scal + 64;
  w.pnew = dalloc<double>(n8);
  w.plast = dalloc<double>(n8);
  w.pold = dalloc<double>(n8);
  w.devinfo = reinterpret_cast<int *>(d.scal + 64 + 3 * n8);
  w.tau = dalloc<double>(n8);
  w.svdS = w.svdU = w.svdVT = nullptr;
  w.wbuf = w.ebuf = nullptr;
  w.os_eps = w.os_w = nullptr;
  w.HP = w.HQ = nullptr;
  w.JB = w.LB = nullptr;
  w.sys_T = w.sys_p = w.sys_H = nullptr;
  w.pref_slot = (int *)malloc(sizeof(int) * d.M);
  for (int k = 0; k < d.M; k++) w.pref_slot[k] = -1;
  w.jtj0_cur = nullptr;
  w.jtj_spec = nullptr;
  {
    // linear-mapped gradient pass: (baseline groups of 256) x (time slices, about one CTA per SM)
    const int nbg = (d.Nbase + 255) / 256;
    const int nsl = db_cp_max_slices(d.Nbase, d.tilesz);
    w.jte_part = dalloc<double>((size_t)nbg * (nsl + 1) * n8);
  }
  DB_CHECK(cudaEventCreateWithFlags(&w.ev_mail, cudaEventDisableTiming));
  DB_CHECK(cudaMallocHost((void **)&w.h_vec, sizeof(double) * (5 * n8 + 4 * d.N + 64)));
  // library handles are process-wide (creating them costs tens of ms; the drop-in entry points
  // build and tear down a problem per call)
  static cusolverDnHandle_t g_cs = nullptr;
  static cublasHandle_t g_cb = nullptr;
  if (!g_cs) {
    CS_CHECK(cusolverDnCreate(&g_cs));
    CB_CHECK(cublasCreate(&g_cb));
  }
  w.cs = g_cs;
  w.cb = g_cb;
  CS_CHECK(cusolverDnSetStream(w.cs, d.stream));
  CB_CHECK(cublasSetStream(w.cb, d.stream));
  int l1 = 0, l2 = 0, l3 = 0;
  CS_CHECK(cusolverDnDpotrf_bufferSize(w.cs, CUBLAS_FILL_MODE_LOWER, n8, w.JTJ, n8, &l1));
  CS_CHECK(cusolverDnDgeqrf_bufferSize(w.cs, n8, n8, w.JTJ, n8, &l2));
  CS_CHECK(cusolverDnDormqr_bufferSize(w.cs, CUBLAS_SIDE_LEFT, CUBLAS_OP_T, n8, 1, n8, w.JTJ, n8,
                                       w.tau, w.Dp, n8, &l3));
  w.lwork = l1 > l2 ? l1 : l2;
  if (l3 > w.lwork) w.lwork = l3;
  int l4 = 0;
  CS_CHECK(cusolverDnDgesvd_bufferSize(w.cs, n8, n8, &l4));
  if (l4 > w.lwork) w.lwork = l4;
  // the cluster Cholesky solver (kernels_chol.cu) shares the workspace
  w.own_chol = n8 <= db_chol_max_n() && db_chol_available() && !getenv("DIRAC_B200_CUSOLVER");
  if (w.own_chol && (size_t)w.lwork < db_chol_ws_doubles(n8)) w.lwork = (int)db_chol_ws_doubles(n8);
  w.cswork = dalloc<double>((size_t)w.lwork);
  w.bc = (!w.own_chol && n8 > 1024) ? db_bigchol_create(n8, BC_BLOCK, BC_INV_PANEL, BC_LOOKAHEAD) : nullptr;
  w.bt_ws = (!w.own_chol && db_bigtri_available(n8)) ? dalloc<double>(db_bigtri_ws_doubles(n8)) : nullptr;
  w.dbuf = dalloc<double2>((size_t)4 * d.R);
  w.ready = true;
}

static void robust_init(dirac_b200_problem *pr) {
  LMWork &w = pr->lm;
  if (w.wbuf) return;
  DevProblem &d = pr->d;
  w.wbuf = dalloc<double2>((size_t)4 * d.R);
  w.ebuf = dalloc<double2>((size_t)4 * d.R);
  w.HP = dalloc<double>((size_t)d.N * 20);
  w.HQ = dalloc<double>((size_t)d.N * 20);
}

static void os_init(dirac_b200_problem *pr) {
  robust_init(pr);
  LMWork &w = pr->lm;
  if (w.os_eps) return;
  w.os_eps = dalloc<double2>((size_t)4 * pr->d.R);
  w.os_w = dalloc<double2>((size_t)4 * pr->d.R);
}

void db_lm_free(dirac_b200_problem *pr) {
  LMWork &w = pr->lm;
  if (!w.ready) return;
  db_free(w.T); db_free(w.Tsub); db_free(w.JTJ0); db_free(w.JTJ);
  db_free(w.Hst); db_free(w.pnew); db_free(w.plast); db_free(w.pold); db_free(w.jte_part);
  db_free(w.tau); db_free(w.cswork); db_free(w.dbuf);
  if (w.bt_ws) db_free(w.bt_ws);
  db_bigchol_destroy(w.bc);
  if (w.svdS) { db_free(w.svdS); db_free(w.svdU); db_free(w.svdVT); }
  if (w.wbuf) { db_free(w.wbuf); db_free(w.ebuf); db_free(w.HP); db_free(w.HQ); }
  if (w.os_eps) { db_free(w.os_eps); db_free(w.os_w); }
  if (w.LB) {
    if (w.JB) db_free(w.JB);
    db_free(w.LB); db_free(w.HB); db_free(w.mu_dev); db_free(w.binfo_dev);
    db_free(w.LBptr_dev); db_free(w.blist_dev); db_free(w.btix_dev); db_free(w.bpoff_dev);
    cudaFreeHost(w.h_mu); cudaFreeHost(w.h_binfo);
  }
  free(w.pref_slot);
  cudaEventDestroy(w.ev_mail);
  cudaFreeHost(w.h_vec);
  free(w.T_valid);
  w.ready = false;
}

// timeslots per CTA slice of a per-cluster pass: enough slices to fill the GPU, long enough to
// amortise the per-slice station reduction
static int pick_tslice(const DevProblem &d, int nt) {
  int target_ctas = db_sm_count();  // one wave: these kernels run 1 CTA per SM (register bound)
  int slices = (target_ctas + d.ntile - 1) / d.ntile;
  if (slices < 1) slices = 1;
  int ts = (nt + slices - 1) / slices;
  if (ts < 2) ts = 2;
  if (ts > nt) ts = nt;
  if (ts < 1) ts = 1;
  return ts;
}

int db_cluster_pass(dirac_b200_problem *pr, int k, const double *pblk_dev, const double2 *in,
                    double2 *out, int mode, int write_out, double *jte_dev, int cost_slot, int t0,
                    int t1, const double2 *wt, double beta = 1.0, bool jte_zeroed = false,
                    const double *pblk_old = nullptr, bool form_hidden = false);

// one streaming pass of cluster k over timeslots [t0,t1): see ClusterPassArgs for the modes.
// Returns the kernel it launched (DB_CP_*; callers other than the test hook ignore it).
int db_cluster_pass(dirac_b200_problem *pr, int k, const double *pblk_dev, const double2 *in,
                    double2 *out, int mode, int write_out, double *jte_dev, int cost_slot, int t0,
                    int t1, const double2 *wt, double beta, bool jte_zeroed,
                    const double *pblk_old, bool form_hidden) {
  DevProblem &d = pr->d;
  if (t1 <= t0) {
    if (mode <= 1 || mode == 4)
      DB_CHECK(cudaMemsetAsync(d.scal + cost_slot, 0, sizeof(double), d.stream));
    if (jte_dev) DB_CHECK(cudaMemsetAsync(jte_dev, 0, sizeof(double) * 8 * d.N, d.stream));
    return DB_CP_NONE;
  }
  ClusterPassArgs a;
  a.coh_k = d.coh + (size_t)k * 4 * d.R;
  a.in = in; a.flag = d.flag; a.pblk = pblk_dev; a.tiles = d.tiles; a.out = out; a.jte = jte_dev;
  a.blpq = d.blpq; a.jte_part = pr->lm.jte_part; a.gcounter = d.counters + 16;
  a.partials = pr->partials; a.cost = d.scal + cost_slot; a.counter = d.counters; a.R = d.R;
  a.N = d.N; a.Nbase = d.Nbase; a.t_begin = t0; a.t_end = t1; a.tslice = pick_tslice(d, t1 - t0);
  a.mode = mode; a.write_out = write_out; a.wt = wt; a.beta = beta;
  a.pblk_old = pblk_old; a.form_hidden = form_hidden;
  // passes without the gradient accumulator fit two CTAs per SM: twice as many, half as long
  if (!(jte_dev && (mode <= 1 || mode == 4)) && a.tslice > 1)
    a.tslice = (a.tslice + 1) / 2;
  if (jte_dev && (mode <= 1 || mode == 4) && !jte_zeroed)
    DB_CHECK(cudaMemsetAsync(jte_dev, 0, sizeof(double) * 8 * d.N, d.stream));
  // kind 2: gradient-carrying passes (INIT, TRIAL); kind 8: ADD / SUB / cost-only passes
  db_prof_begin((jte_dev && (mode <= 1 || mode == 4)) ? 2 : 8, (double)(t1 - t0) * d.Nbase * (129.0 + (write_out ? 64.0 : 0.0) +
                                                 (wt ? 64.0 : 0.0)), d.stream);
  const int kernel = db_launch_cluster_pass(&a, d.ntile, d.stream);
  db_prof_end(d.stream);
  db_count_launch(1);
  return kernel;
}

// Gram tensor of cluster k over timeslots t0, t0+step, ... < t1 into Tdst [Nbase][16]
static void gram(dirac_b200_problem *pr, int k, int t0, int t1, int step, double *Tdst) {
  DevProblem &d = pr->d;
  GramArgs a;
  a.coh = d.coh; a.flag = d.flag; a.tiles = d.tiles; a.T = Tdst; a.R = d.R; a.N = d.N;
  a.Nbase = d.Nbase; a.k0 = k; a.t_begin = t0; a.t_end = t1; a.t_step = step;
  db_prof_begin(3, (double)((t1 - t0 + step - 1) / step) * d.Nbase * 65.0 + 128.0 * d.Nbase,
                d.stream);
  db_launch_coh_gram(&a, d.ntile, 1, d.stream);
  db_prof_end(d.stream);
  db_count_launch(1);
}

static AssembleArgs assemble_args(const DevProblem &d, const double *T, const double *pblk_dev,
                                  double *Hst) {
  AssembleArgs a;
  memset(&a, 0, sizeof(a));
  a.T = T; a.pblk = pblk_dev; a.Hst = Hst; a.N = d.N; a.Nbase = d.Nbase;
  return a;
}

// station sums of the diagonal blocks of nb systems (each reads its Gram tensors twice)
static void station_sums(dirac_b200_problem *pr, const AssembleArgs &a, int nb) {
  DevProblem &d = pr->d;
  db_prof_begin(4, nb * 256.0 * d.Nbase, d.stream);
  db_launch_station_sums(&a, nb, d.stream);
  db_prof_end(d.stream);
  db_count_launch(1);
}

// the matrices of nb systems from their station sums: full, or (lower) the lower triangle and the
// diagonal only, each Gram tensor read once
static void assemble_tiles(dirac_b200_problem *pr, const AssembleArgs &a, int nb) {
  DevProblem &d = pr->d;
  const double n = 8.0 * d.N;
  db_prof_begin(4, nb * (a.lower ? 128.0 * d.Nbase + 4.0 * n * (n + 1) : 256.0 * d.Nbase + 8.0 * n * n),
                d.stream);
  db_launch_assemble_tiles(&a, nb, d.stream);
  db_prof_end(d.stream);
  db_count_launch(1);
}

// J^T J at pblk_dev from the Gram tensors T: station sums into w.Hst, then the full undamped matrix
// into JTJ (JTJ == null: the station sums only; the solve writes the damped matrix, enqueue_solve)
static void assemble(dirac_b200_problem *pr, const double *T, const double *pblk_dev,
                     double *JTJ) {
  AssembleArgs a = assemble_args(pr->d, T, pblk_dev, pr->lm.Hst);
  station_sums(pr, a, 1);
  if (!JTJ) return;
  a.JTJ = JTJ;
  assemble_tiles(pr, a, 1);
}

// weighted J^T J of cluster k over timeslots [t0,t1) by streaming (robust LM)
static void weighted_jtj(dirac_b200_problem *pr, int k, int t0, int t1, const double *pblk_dev,
                         const double2 *wt, double *JTJ) {
  DevProblem &d = pr->d;
  LMWork &w = pr->lm;
  const int n = w.n8;
  DB_CHECK(cudaMemsetAsync(JTJ, 0, sizeof(double) * (size_t)n * n, d.stream));
  DB_CHECK(cudaMemsetAsync(w.HP, 0, sizeof(double) * 20 * d.N, d.stream));
  DB_CHECK(cudaMemsetAsync(w.HQ, 0, sizeof(double) * 20 * d.N, d.stream));
  if (t1 <= t0) return;
  WeightedJtjArgs a;
  a.coh_k = d.coh + (size_t)k * 4 * d.R;
  a.wt = wt; a.flag = d.flag; a.pblk = pblk_dev; a.tiles = d.tiles; a.JTJ = JTJ; a.HP = w.HP;
  a.HQ = w.HQ; a.R = d.R; a.N = d.N; a.Nbase = d.Nbase; a.t_begin = t0; a.t_end = t1;
  a.tslice = pick_tslice(d, t1 - t0);
  db_prof_begin(6, (double)(t1 - t0) * d.Nbase * 129.0 + 8.0 * 64.0 * d.N * d.N, d.stream);
  db_launch_weighted_jtj(&a, d.ntile, d.stream);
  db_prof_end(d.stream);
  db_count_launch(2);
}

// chunk ck of cluster k covers timeslots [t0,t1)  (lmfit.c:893-905)
void db_chunk_range(const DevProblem &d, int k, int ck, int *t0, int *t1);
static void chunk_range(const DevProblem &d, int k, int ck, int *t0, int *t1) {
  db_chunk_range(d, k, ck, t0, t1);
}
void db_chunk_range(const DevProblem &d, int k, int ck, int *t0, int *t1) {
  int nchunk = d.h_clus[k].nchunk;
  int tilechunk = (d.tilesz + nchunk - 1) / nchunk;
  int a = ck * tilechunk;
  int b = a + tilechunk;
  if (a > d.tilesz) a = d.tilesz;
  if (b > d.tilesz) b = d.tilesz;
  *t0 = a;
  *t1 = b;
}

// ------------------------------------------------------------------------------------------------
// damped solve (J^T J + mu I) dp = J^T e on the device.  returns 1 if solved.
// linsolv: 0 Cholesky (dpotrf/dpotrs, clmfit.c:373-395), 1 QR (dgels, :396-409),
//          2 SVD with singular-value cut at eps1 (:410-436)
// ------------------------------------------------------------------------------------------------
// enqueues the factorisation and the solve; the status lands in w.devinfo[0..1] (read by the caller
// together with the trial results).  The SVD variant finishes on the host and returns solved.
static int enqueue_solve(dirac_b200_problem *pr, double mu, int linsolv, double eps1) {
  DevProblem &d = pr->d;
  LMWork &w = pr->lm;
  const int n = w.n8;
  int *hinfo = (int *)(w.h_vec + 4 * n + 4 * d.N);
  hinfo[0] = hinfo[1] = 0;
  if (linsolv == 0 && w.own_chol) {
    // one cluster kernel: damping, factorisation and both triangular solves (kernels_chol.cu)
    db_prof_begin(5, 0.0, d.stream);
    db_launch_chol_solve(w.jtj0_cur ? w.jtj0_cur : w.JTJ0, n, mu, w.JTe, w.Dp, w.cswork, w.devinfo,
                         d.stream);
    db_prof_end(d.stream);
    db_count_launch(1);
    w.step_fused = w.step_armed;  // the kernel's epilogue formed the trial point (db_chol_set_step)
    return 1;
  }
  if (linsolv == 0 && w.sys_T) {
    // the lower triangle of J^T J + mu I straight from the Gram tensors into the buffer dpotrf factors
    // in place: a system rejected at this mu is rebuilt the same way at the next one
    AssembleArgs a = assemble_args(d, w.sys_T, w.sys_p, const_cast<double *>(w.sys_H));
    a.JTJ = w.JTJ;
    a.mu = mu;
    a.lower = 1;
    assemble_tiles(pr, a, 1);
  } else {
    db_prof_begin(4, 16.0 * n * n, d.stream);
    db_launch_copy_add_diag(w.jtj0_cur ? w.jtj0_cur : w.JTJ0, w.JTJ, n, mu, d.stream);
    db_prof_end(d.stream);
    db_count_launch(1);
  }
  // the blocked substitutions read b from J^T e; every other solver works on Dp in place
  if (linsolv != 0 || !w.bt_ws)
    DB_CHECK(cudaMemcpyAsync(w.Dp, w.JTe, sizeof(double) * n, cudaMemcpyDeviceToDevice, d.stream));
  db_prof_begin(5, 0.0, d.stream);
  if (linsolv == 0) {
    CS_CHECK(cusolverDnDpotrf(w.cs, CUBLAS_FILL_MODE_LOWER, n, w.JTJ, n, w.cswork, w.lwork,
                              w.devinfo));
    if (w.bt_ws) {
      // the two substitutions by the blocked dataflow kernels (cusolverDnDpotrs: 0.68 ms at n = 4096);
      // their prologue clears the status word dpotrs would set
      db_launch_bigtri_solve(w.JTJ, n, n, w.JTe, w.Dp, w.bt_ws, w.devinfo + 1, d.stream);
      db_count_launch(2);
    } else {
      CS_CHECK(cusolverDnDpotrs(w.cs, CUBLAS_FILL_MODE_LOWER, n, 1, w.JTJ, n, w.Dp, n,
                                w.devinfo + 1));
      db_count_launch(2);
    }
  } else if (linsolv == 1) {
    // A = QR ; dp = R^-1 Q^T b   (A symmetric: row/column-major views coincide)
    CS_CHECK(cusolverDnDgeqrf(w.cs, n, n, w.JTJ, n, w.tau, w.cswork, w.lwork, w.devinfo));
    CS_CHECK(cusolverDnDormqr(w.cs, CUBLAS_SIDE_LEFT, CUBLAS_OP_T, n, 1, n, w.JTJ, n, w.tau, w.Dp,
                              n, w.cswork, w.lwork, w.devinfo + 1));
    const double one = 1.0;
    CB_CHECK(cublasDtrsm(w.cb, CUBLAS_SIDE_LEFT, CUBLAS_FILL_MODE_UPPER, CUBLAS_OP_N,
                         CUBLAS_DIAG_NON_UNIT, n, 1, &one, w.JTJ, n, w.Dp, n));
    db_count_launch(3);
  } else {
    if (!w.svdS) {
      w.svdS = dalloc<double>(n);
      w.svdU = dalloc<double>((size_t)n * n);
      w.svdVT = dalloc<double>((size_t)n * n);
    }
    CS_CHECK(cusolverDnDgesvd(w.cs, 'A', 'A', n, n, w.JTJ, n, w.svdS, w.svdU, n, w.svdVT, n,
                              w.cswork, w.lwork, nullptr, w.devinfo));
    db_count_launch(1);
    // dp = V diag(1/s | s>eps1) U^T b, small: finish on the host vectors
    double *hS = (double *)malloc(sizeof(double) * n);
    double *hb = (double *)malloc(sizeof(double) * n);
    const double one = 1.0, zero = 0.0;
    CB_CHECK(cublasDgemv(w.cb, CUBLAS_OP_T, n, n, &one, w.svdU, n, w.JTe, 1, &zero, w.Dp, 1));
    DB_CHECK(cudaMemcpyAsync(hS, w.svdS, sizeof(double) * n, cudaMemcpyDeviceToHost, d.stream));
    DB_CHECK(cudaMemcpyAsync(hb, w.Dp, sizeof(double) * n, cudaMemcpyDeviceToHost, d.stream));
    db_stream_sync(d.stream);
    for (int i = 0; i < n; i++) hb[i] = (hS[i] > eps1) ? hb[i] / hS[i] : 0.0;
    DB_CHECK(cudaMemcpyAsync(w.pnew, hb, sizeof(double) * n, cudaMemcpyHostToDevice, d.stream));
    CB_CHECK(cublasDgemv(w.cb, CUBLAS_OP_T, n, n, &one, w.svdVT, n, w.pnew, 1, &zero, w.Dp, 1));
    db_prof_end(d.stream);
    DB_CHECK(cudaMemcpyAsync(w.h_vec + 2 * n, w.Dp, sizeof(double) * n, cudaMemcpyDeviceToHost,
                             d.stream));
    db_stream_sync(d.stream);
    free(hS);
    free(hb);
    db_count_launch(2);
    return 1;
  }
  db_prof_end(d.stream);
  (void)hinfo;
  return 1;
}

static double nrm2sq(const double *v, int n) {
  double s = 0.0;
  for (int i = 0; i < n; i++) s += v[i] * v[i];
  return s;
}

// ------------------------------------------------------------------------------------------------
// Before a SAGE sweep of plain LM: J^T J of every (single-chunk) cluster at its current Jones, mu0 =
// tau max diag, and the Cholesky factor of J^T J + mu0 I — assembled and factorised as ONE batch
// (cusolverDnDpotrfBatched runs the M factorisations concurrently: ~15 us per 496x496 matrix against
// ~200 us one at a time).  A cluster's Jones only change during its own visit, so the factor is
// still exact when the visit starts; its first LM solve is then two triangular solves.
// ------------------------------------------------------------------------------------------------
void db_prefactor_sweep(dirac_b200_problem *pr, double tau) {
  DevProblem &d = pr->d;
  db_lm_init(pr);
  LMWork &w = pr->lm;
  const int n = w.n8;
  const size_t nn = (size_t)n * n;
  // own batched factorisation (one 16-CTA cluster per matrix) when the cluster solver takes the size:
  // the factor of cluster b then lives in a k_chol_solve workspace (ld = 32*ceil(n/32))
  const bool own_batch = w.own_chol && db_tri_available(n) && !getenv("DIRAC_B200_BATCH_CUSOLVER");
  // The cluster solvers read the undamped J^T J (JB) and damp it themselves.  cuSOLVER factors the
  // lower triangle of J^T J + mu0 I written straight into LB, in place; a rejected first step is
  // re-assembled from the Gram tensors (enqueue_solve), so no undamped copy is kept.
  const bool keep_jb = w.own_chol;
  if ((double)d.M * nn * 8.0 * (keep_jb ? 2 : 1) > 24e9) return;  // batch buffers within 24 GB
  const size_t lstride = own_batch ? db_chol_ws_doubles(n) : nn;
  w.lb_stride = lstride;
  w.lb_ld = own_batch ? 32 * ((n + 31) / 32) : n;
  if (!w.LB) {
    w.JB = keep_jb ? dalloc<double>(nn * d.M) : nullptr;
    w.LB = dalloc<double>(lstride * d.M);
    w.HB = dalloc<double>((size_t)4 * d.N * d.M);
    w.mu_dev = dalloc<double>(d.M);
    w.binfo_dev = dalloc<int>(2 * d.M);
    w.LBptr_dev = (double **)dalloc<double *>(d.M);
    w.blist_dev = dalloc<int>(d.M);
    w.btix_dev = dalloc<int>(d.M);
    w.bpoff_dev = dalloc<int>(d.M);
    DB_CHECK(cudaMallocHost((void **)&w.h_mu, sizeof(double) * d.M));
    DB_CHECK(cudaMallocHost((void **)&w.h_binfo, sizeof(int) * 2 * d.M));
    std::vector<int> tix(d.M), poff(d.M);
    std::vector<double *> ptr(d.M);
    for (int k = 0; k < d.M; k++) {
      tix[k] = d.h_clus[k].chunk0;
      poff[k] = d.h_chunk_poff[d.h_clus[k].chunk0];
      ptr[k] = w.LB + lstride * k;
    }
    DB_CHECK(cudaMemcpy(w.btix_dev, tix.data(), sizeof(int) * d.M, cudaMemcpyHostToDevice));
    DB_CHECK(cudaMemcpy(w.bpoff_dev, poff.data(), sizeof(int) * d.M, cudaMemcpyHostToDevice));
    DB_CHECK(cudaMemcpy(w.LBptr_dev, ptr.data(), sizeof(double *) * d.M, cudaMemcpyHostToDevice));
    if (w.bc) db_bigchol_bind_batch(w.bc, w.LB, (long long)lstride, d.M);
  }
  std::vector<int> list;
  // Gram tensors still missing: one launch per run of consecutive single-chunk clusters (their slots
  // are consecutive too), i.e. one launch for a sky without hybrid clusters
  for (int k = 0; k < d.M;) {
    const int tix = d.h_clus[k].chunk0;
    if (d.h_clus[k].nchunk != 1 || w.T_valid[tix]) {
      k++;
      continue;
    }
    int k1 = k + 1;
    while (k1 < d.M && d.h_clus[k1].nchunk == 1 && !w.T_valid[d.h_clus[k1].chunk0] &&
           d.h_clus[k1].chunk0 == tix + (k1 - k))
      k1++;
    GramArgs a;
    a.coh = d.coh; a.flag = d.flag; a.tiles = d.tiles; a.T = w.T + (size_t)tix * d.Nbase * 16;
    a.R = d.R; a.N = d.N; a.Nbase = d.Nbase; a.k0 = k; a.t_begin = 0; a.t_end = d.tilesz;
    a.t_step = 1;
    db_prof_begin(3, (double)(k1 - k) * ((double)d.tilesz * d.Nbase * 65.0 + 128.0 * d.Nbase),
                  d.stream);
    db_launch_coh_gram(&a, d.ntile, k1 - k, d.stream);
    db_prof_end(d.stream);
    db_count_launch(1);
    for (int kk = k; kk < k1; kk++) w.T_valid[d.h_clus[kk].chunk0] = 1;
    k = k1;
  }
  for (int k = 0; k < d.M; k++) {
    w.pref_slot[k] = -1;
    if (d.h_clus[k].nchunk != 1) continue;
    w.pref_slot[k] = (int)list.size();
    list.push_back(k);
  }
  const int nb = (int)list.size();
  if (nb == 0) return;
  DB_CHECK(cudaMemcpyAsync(w.blist_dev, list.data(), sizeof(int) * nb, cudaMemcpyHostToDevice,
                           d.stream));
  AssembleArgs b = assemble_args(d, w.T, d.pp, w.HB);
  b.list = w.blist_dev; b.tix = w.btix_dev; b.poff = w.bpoff_dev;
  station_sums(pr, b, nb);
  // mu0 = tau * max_i (J^T J)_ii (clmfit.c:342-352) of every matrix, from the station sums
  db_launch_batch_mu0(w.HB, w.mu_dev, d.N, tau, nb, d.stream);
  db_count_launch(1);
  if (keep_jb) {
    b.JTJ = w.JB;
    b.stride = (long long)nn;
    assemble_tiles(pr, b, nb);
  }
  if (!own_batch) {
    b.JTJ = w.LB;
    b.stride = (long long)lstride;
    b.mu_dev = w.mu_dev;
    b.lower = 1;
    assemble_tiles(pr, b, nb);
  }
  db_prof_begin(5, 0.0, d.stream);
  if (own_batch) {
    db_launch_chol_factor_batched(w.JB, n, w.mu_dev, w.LB, (long long)lstride, w.binfo_dev, nb,
                                  d.stream);
    db_count_launch(1);
  } else if (!w.bc) {
    CS_CHECK(cusolverDnDpotrfBatched(w.cs, CUBLAS_FILL_MODE_LOWER, n, w.LBptr_dev, n, w.binfo_dev, nb));
    db_count_launch(1);
  } else {
    // Large systems (8N = 4096 at 512 stations: 23 GFLOP each): one blocked panel loop over all of
    // them (bigchol.cu), its trailing updates DGEMMs over the whole batch
    db_bigchol_factor_batch(w.bc, nb, w.binfo_dev, 1, d.stream);
  }
  db_prof_end(d.stream);
  DB_CHECK(cudaMemcpyAsync(w.h_mu, w.mu_dev, sizeof(double) * nb, cudaMemcpyDeviceToHost, d.stream));
  DB_CHECK(cudaMemcpyAsync(w.h_binfo, w.binfo_dev, sizeof(int) * (own_batch ? 2 * nb : nb),
                           cudaMemcpyDeviceToHost, d.stream));
  w.binfo_step = own_batch ? 2 : 1;
  db_stream_sync(d.stream);  // list goes out of scope; mu0 is needed on the host
}

// ------------------------------------------------------------------------------------------------
// the LM iteration loop shared by the four reference variants.  On entry the hidden data of the
// chunk is in w.dbuf and pblk_dev holds p, or, if `hidden_from` is given, the trial passes form the
// hidden data per row from that residual and the entry Jones in w.pold; the trial of the last
// iteration then writes its residual d - f(p_trial) into w.dbuf (LmOut::res_in_dbuf: that trial
// was accepted, w.dbuf holds the residual at the final Jones).  If `have_first` the caller already
// produced ||e||^2 (in *first_cost) and J^T e (in w.JTe) at p with the same weights (the fused first
// pass).
// wt == null: plain LM, J^T J from the cached Gram tensor; wt != null: robust LM round.
// `nu_damp` is the integer damping multiplier that the robust driver carries across its IRLS rounds
// (robustlm.c keeps `nu` alive over the nw loop).  `evaluated_trial` reports whether w.plast holds
// the last evaluated trial point (the reference's `ed` after a rejected step, clmfit.c:478).
// ------------------------------------------------------------------------------------------------
// LM accept/reject decisions taken at rounding level (|dF| <= 1e-11 ||e||^2) since the last reset.
// The ordered-subsets variants reject trial steps along a subset's gradient until the step is
// ~1e-15 |p|; whether the last one counts as an improvement is decided by the rounding of two sums
// over all rows, yet it resets mu and nu and steers every later iteration.  The compiled reference and
// its CPU restatement part ways on such runs (tests/golden/make_golden_c2r.py), so parity of the
// solved Jones is only defined when this stays 0.
static long g_noise_decisions = 0;
static long g_lm_stat[4] = {0, 0, 0, 0};  // accepted, accepted with mu/3, rejected, -
extern "C" void dirac_b200_lm_stats(long *out4, int reset) {
  for (int i = 0; i < 4; i++) {
    if (out4) out4[i] = g_lm_stat[i];
    if (reset) g_lm_stat[i] = 0;
  }
}
extern "C" long dirac_b200_noise_decisions(int reset) {
  const long v = g_noise_decisions;
  if (reset) g_noise_decisions = 0;
  return v;
}

// Consensus (ADMM) terms of one (cluster, chunk) block: the LM minimises
//   ||d - f(p)||^2 + y^T (p - bz) + rho/2 |p - bz|^2       (Dirac.h:1524)
// whose Gauss-Newton system is (J^T J + rho/2 I + mu I) dp = J^T e - y/2 - rho/2 (p - bz): the
// right-hand side is corrected on the device after every pass that produced J^T e, rho/2 rides on the
// damping handed to the solver, and the host adds the two extra terms to the costs it compares.
struct LmAug {
  const double *y_dev, *bz_dev;    // device, this block (8N)
  const double *y_host, *bz_host;  // host, this block
  double rho;
};
static const LmAug *g_aug = nullptr;
static std::vector<double> g_hpnew;
static double *hpnew_aug(LMWork &w) {
  if ((int)g_hpnew.size() < w.n8) g_hpnew.resize(w.n8);
  return g_hpnew.data();
}
static double aug_cost(const LmAug *a, const double *p, int n) {
  double s = 0.0;
  for (int i = 0; i < n; i++) {
    const double dlt = p[i] - a->bz_host[i];
    s += a->y_host[i] * dlt + 0.5 * a->rho * dlt * dlt;
  }
  return s;
}
extern "C" void db_launch_lm_aug_rhs(double *jte, const double *p, const double *y, const double *bz,
                                     double rho, int n, cudaStream_t st);

struct LmOut {
  double init_eL2, eL2, jacTe_inf, Dp_L2, mu;
  int k, stop;
  bool res_in_dbuf;
};

// Subsets of the ordered-subsets LM of a chunk of `ntiles` tiles (clmfit.c:1313-1356): Nsubsets
// pieces of Ntper tiles.  They coincide with the pieces of the data only when the tile count is a
// multiple of the subset count.
struct OsLayout {
  int Nsubsets, Ntper;
  bool misaligned;
};
static OsLayout os_layout(int ntiles) {
  OsLayout o;
  o.Nsubsets = ntiles < 10 ? ntiles : 10;
  o.Ntper = o.Nsubsets > 0 ? (ntiles + o.Nsubsets - 1) / o.Nsubsets : ntiles;
  o.misaligned = o.Nsubsets > 0 && (ntiles % o.Nsubsets) != 0 && !db_opt(DB_OPT_OS_CONSISTENT);
  return o;
}

// what os_subset_system ran: the subset's tiles [s0, s1) and, on the misaligned branch, the number
// of Jacobian rows nJ that are paired with data
struct OsPath {
  bool misaligned;
  int s0, s1;
  long long nJ;
};

// J^T e (w.JTe) and J^T J (w.JTJ0) of ordered subset l of chunk ck of cluster k, tiles [t0, t1), at
// pblk_dev; the hidden data are in w.dbuf, wt are the sqrt-weights (robust LM) or null.
static OsPath os_subset_system(dirac_b200_problem *pr, int k, int t0, int t1, int l,
                               const double *pblk_dev, const double2 *wt) {
  DevProblem &d = pr->d;
  LMWork &w = pr->lm;
  const int ntiles = t1 - t0;
  const OsLayout L = os_layout(ntiles);
  const int Ntper = L.Ntper;
  OsPath path;
  path.misaligned = L.misaligned;
  path.nJ = 0;
  int s0 = t0 + l * Ntper;
  int s1 = (l * Ntper + Ntper < ntiles) ? s0 + Ntper : t1;
  if (s0 > t1) s0 = t1;
  if (!L.misaligned) {
    // J^T e restricted to the subset; e is the current (weighted) residual d - f(p)
    db_cluster_pass(pr, k, pblk_dev, w.dbuf, nullptr, 1, 0, w.JTe, 2, s0, s1, wt);
    if (wt) {
      weighted_jtj(pr, k, s0, s1, pblk_dev, wt, w.JTJ0);
    } else {
      gram(pr, k, s0, s1, 1, w.Tsub);
      assemble(pr, w.Tsub, pblk_dev, w.JTJ0);
    }
  } else {
    // The reference pairs row i of the subset's Jacobian with the residual (and weight) of data
    // index edI[l] + i, Npersubset = ceil(n/Nsubsets) apart, while the subset's tiles are
    // Ntpersubset = ceil(ntiles/Nsubsets) apart (clmfit.c:1313-1356,1400; robustlm.c:2835-2935):
    // when ntiles is not a multiple of Nsubsets that is another tile, baseline and component, and
    // the Jacobian is cut (or zero padded) to Nos[l] rows.  Reproduced literally: the residual of
    // the whole chunk at p, gathered with the reference's offset into the subset's rows, enters the
    // J^T e pass as a given vector; the cut and the weights enter as per-component sqrt-weights.
    const long long nn = 8ll * ntiles * d.Nbase;
    const long long Nper = (nn + L.Nsubsets - 1) / L.Nsubsets;
    const long long kl = (long long)l * Nper;
    const int tl = l * Ntper;
    long long Nos;
    int tileI;
    if (tl + Ntper < ntiles) {
      Nos = Nper;
      tileI = Ntper;
    } else {
      Nos = nn - kl;
      tileI = ntiles - tl;
    }
    long long nJ = tileI > 0 ? 8ll * d.Nbase * tileI : 0;
    if (Nos < nJ) nJ = Nos;
    if (nJ < 0) nJ = 0;
    s0 = t0 + tl;
    s1 = s0 + (tileI > 0 ? tileI : 0);
    if (s0 > t1) s0 = s1 = t1;
    os_init(pr);
    // residual of the whole chunk at p (unweighted), then the shifted gather
    db_cluster_pass(pr, k, pblk_dev, w.dbuf, w.ebuf, 1, 1, nullptr, 2, t0, t1, nullptr);
    if (s1 > s0) {
      db_launch_os_shift(w.ebuf, wt, w.os_eps, w.os_w, d.R, (long long)s0 * d.Nbase,
                         (long long)(s1 - s0) * d.Nbase, (long long)t0 * d.Nbase, kl, nJ, d.stream);
      db_count_launch(1);
    }
    db_cluster_pass(pr, k, pblk_dev, w.os_eps, nullptr, 4, 0, w.JTe, 2, s0, s1, w.os_w);
    // the cut of the Jacobian and the shifted weights are in os_w
    weighted_jtj(pr, k, s0, s1, pblk_dev, w.os_w, w.JTJ0);
    path.nJ = nJ;
  }
  path.s0 = s0;
  path.s1 = s1;
  return path;
}

static void lm_core(dirac_b200_problem *pr, int k, int ck, int t0, int t1, double *pblk_dev,
                    const double2 *wt, int itmax, const double *opts, int linsolv, int os,
                    int os_shift, int randomize, bool have_first, double first_cost, int *nu_damp,
                    bool *evaluated_trial, const double2 *hidden_from, LmOut *out) {
  DevProblem &d = pr->d;
  LMWork &w = pr->lm;
  const int n = w.n8;
  const int ntiles = t1 - t0;
  const double tau = opts[0], eps1 = opts[1], eps2 = opts[2], eps2_sq = opts[2] * opts[2],
               eps3 = opts[3];
  double *hp = w.h_vec;            // current p
  double *hjte = w.h_vec + n;      // J^T e
  double *hDp = w.h_vec + 2 * n;   // step
  double *hpnew = w.h_vec + 3 * n; // trial p
  double *hH = w.h_vec + 4 * n;    // station sums [N][4]

  double p_eL2;
  // Prefactored visit: nothing the host knows is needed to enqueue the first trial (mu0 and the factor
  // come from the batch), so the entry values (p, J^T e, ||e||^2) ride back with the trial's results
  // and the entry tests of clmfit.c:300-340 are applied after the fact (a trial that should not have
  // been taken is simply discarded: it only wrote scratch buffers).
  const LmAug *aug = (!os && !wt) ? g_aug : nullptr;
  const double half_rho = aug ? 0.5 * aug->rho : 0.0;
  if (aug) w.pref_slot[k] = -1;  // the batch factor does not know about rho/2
  const bool defer = have_first && !os && !wt && linsolv == 0 && itmax > 0 && w.pref_slot[k] >= 0 &&
                     std::isnan(first_cost);
  DB_CHECK(cudaMemcpyAsync(hp, pblk_dev, sizeof(double) * n, cudaMemcpyDeviceToHost, d.stream));
  if (aug && have_first)  // J^T e of the fused first pass -> gradient of the augmented cost
    db_launch_lm_aug_rhs(w.JTe, pblk_dev, aug->y_dev, aug->bz_dev, aug->rho, n, d.stream);
  if (have_first) {
    p_eL2 = first_cost;
    if (!defer) {
      if (!os)
        DB_CHECK(cudaMemcpyAsync(hjte, w.JTe, sizeof(double) * n, cudaMemcpyDeviceToHost,
                                 d.stream));
      if (std::isnan(first_cost))
        DB_CHECK(cudaMemcpyAsync(d.h_scal + 2, d.scal + 2, sizeof(double), cudaMemcpyDeviceToHost,
                                 d.stream));
      db_stream_sync(d.stream);
      if (std::isnan(first_cost)) p_eL2 = d.h_scal[2];
    } else {
      p_eL2 = 1.0;  // placeholder: J^T e and ||e||^2 (slot 2) come back with the first trial
    }
  } else {
    // e = wt.(d - f(p)), ||e||^2, J^T e     (clmfit.c:241-252 / robustlm.c:2235-2251)
    db_cluster_pass(pr, k, pblk_dev, w.dbuf, nullptr, 1, 0, os ? nullptr : w.JTe, 1, t0, t1, wt);
    if (aug) db_launch_lm_aug_rhs(w.JTe, pblk_dev, aug->y_dev, aug->bz_dev, aug->rho, n, d.stream);
    if (!os)
      DB_CHECK(cudaMemcpyAsync(hjte, w.JTe, sizeof(double) * n, cudaMemcpyDeviceToHost, d.stream));
    p_eL2 = db_read_scalar(pr, 1);
  }
  if (aug && !defer) p_eL2 += aug_cost(aug, hp, n);
  double init_p_eL2 = p_eL2;
  int stop = 0;
  if (!isfinite(p_eL2)) stop = 7;
  int nu = *nu_damp, nu2;
  double mu = 0.0, Dp_L2 = DBL_MAX, jacTe_inf = 0.0;
  *evaluated_trial = false;
  bool res_in_dbuf = false;
  bool pending_entry = defer;  // entry values not on the host yet
  w.jtj_spec = nullptr;
  int kiter_adjust = 0;

  // ordered subsets (clmfit.c:1313-1356)
  const OsLayout osl = os_layout(ntiles);
  const int Nsubsets = osl.Nsubsets;
  const int max_os_iter = os ? (int)ceil(0.1 * (double)Nsubsets) : 1;
  const bool os_misaligned = os && osl.misaligned;

  // Gram tensor of this chunk (time-invariant part of the unweighted J^T J), built once
  const int tix = d.h_clus[k].chunk0 + ck;
  double *Tfull = w.T + (size_t)tix * d.Nbase * 16;
  if (!wt && !os && !w.T_valid[tix] && ntiles > 0) {
    gram(pr, k, t0, t1, 1, Tfull);
    w.T_valid[tix] = 1;
  }

  // Host/device handshake: ONE synchronisation per trial.  Everything between two decisions —
  // damping, factorisation, solve, p + dp, trial pass (cost and, speculatively, J^T e at the trial
  // point) — is enqueued back to back; the scalars the decision needs come back together.
  double *hsc = w.h_vec + 4 * n + 4 * d.N + 8;  // [n: diag][4: |dp|^2, dp.jte, cost, -]
  double *hjte_new = hpnew;                     // the trial point itself is formed on the device
  int kiter;
  std::vector<int> subI;
  for (kiter = 0; kiter < itmax && !stop; ++kiter) {
    if (!pending_entry && p_eL2 <= eps3) {
      stop = 6;
      break;
    }
    if (os && randomize) {
      // random permutation of the subsets, drawn like the reference's (random_permutation,
      // lmfit.c:1085-1099: inside-out shuffle on the caller-seeded rand()), once per LM iteration
      // (clmfit.c:1376-1379)
      subI.resize(Nsubsets);
      for (int i = 0; i < Nsubsets; ++i) {
        const int j = rand() % (i + 1);
        subI[i] = subI[j];
        subI[j] = i;
      }
    }
    for (int ositer = 0; ositer < max_os_iter; ositer++) {
      double mx = 0.0;
      // first iteration of a prefactored cluster: J^T J, mu0 and the factor are already there
      const int slot = (!wt && !os && kiter == 0 && linsolv == 0) ? w.pref_slot[k] : -1;
      const bool prefac = slot >= 0;
      const bool need_mx = (kiter == 0) && !prefac;
      w.jtj0_cur = (prefac && w.JB) ? w.JB + (size_t)slot * n * n : nullptr;
      // unweighted systems of the cuSOLVER Cholesky: each solve assembles J^T J + mu I itself
      const bool in_place = !w.own_chol && linsolv == 0 && !wt && !os;
      w.sys_T = in_place ? Tfull : nullptr;
      w.sys_p = pblk_dev;
      w.sys_H = prefac ? w.HB + (size_t)slot * 4 * d.N : w.Hst;
      if (os) {
        const int l = randomize ? subI[ositer] : (os_shift + kiter + ositer) % Nsubsets;
        os_subset_system(pr, k, t0, t1, l, pblk_dev, wt);
        DB_CHECK(cudaMemcpyAsync(hjte, w.JTe, sizeof(double) * n, cudaMemcpyDeviceToHost,
                                 d.stream));
      } else if (prefac) {
        w.pref_slot[k] = -1;  // valid for this visit only
      } else if (wt) {
        weighted_jtj(pr, k, t0, t1, pblk_dev, wt, w.JTJ0);
      } else if (w.jtj_spec) {
        // already assembled at this point while the host was deciding on the previous trial
        w.jtj0_cur = w.jtj_spec;
        w.jtj_spec = nullptr;
      } else {
        assemble(pr, Tfull, pblk_dev, in_place ? nullptr : w.JTJ0);
      }
      if (need_mx) {
        if (wt || os_misaligned) {
          db_launch_extract_diag(w.JTJ0, w.JTe_new, n, d.stream);  // JTe_new is free scratch here
          db_count_launch(1);
          DB_CHECK(cudaMemcpyAsync(hsc, w.JTe_new, sizeof(double) * n, cudaMemcpyDeviceToHost,
                                   d.stream));
        } else {
          DB_CHECK(cudaMemcpyAsync(hH, w.Hst, sizeof(double) * 4 * d.N, cudaMemcpyDeviceToHost,
                                   d.stream));
        }
      }
      if (need_mx || os) db_stream_sync(d.stream);
      if (need_mx) {
        if (wt || os_misaligned) {
          for (int i = 0; i < n; i++)
            if (fabs(hsc[i]) > fabs(mx)) mx = hsc[i];
        } else {
          // the diagonal is (h00 x4, h11 x4) per station
          for (int s = 0; s < d.N; s++) {
            if (fabs(hH[4 * s]) > fabs(mx)) mx = hH[4 * s];
            if (fabs(hH[4 * s + 1]) > fabs(mx)) mx = hH[4 * s + 1];
          }
        }
      }
      double p_L2 = 0.0;
      if (!pending_entry) {
        jacTe_inf = 0.0;
        for (int i = 0; i < n; i++) {
          double a = fabs(hjte[i]);
          if (a > jacTe_inf) jacTe_inf = a;
        }
        p_L2 = nrm2sq(hp, n);
        if (jacTe_inf <= eps1) {
          Dp_L2 = 0.0;
          stop = 1;
          // clevmar/rlevmar leave the iteration loop here without ++k (clmfit.c:335-339); in the OS
          // variants the break only leaves the subset loop and k still advances (clmfit.c:1419-1423)
          if (!os) kiter_adjust = 1;
          break;
        }
      }
      if (kiter == 0) mu = prefac ? w.h_mu[slot] : tau * (mx + half_rho);  // clmfit.c:342-352
      bool use_factor = prefac;
      // adaptive damping loop (clmfit.c:356-540)
      while (1) {
        int issolved;
        bool skip_info = false;
        // the cluster solvers form p + dp, |dp|^2, dp.J^T e themselves and clear the trial pass's
        // accumulator (solution_epilogue, kernels_chol.cu); other solvers leave it to k_lm_step
        w.step_fused = false;
        w.step_armed = w.own_chol && linsolv == 0;
        if (w.step_armed)
          db_chol_set_step(pblk_dev, w.pnew, d.scal + 8, os ? nullptr : w.JTe_new);
        if (use_factor) {
          // (J^T J + mu0 I) = L L^T came out of the batch: only the two triangular solves remain
          use_factor = false;
          db_prof_begin(5, 0.0, d.stream);
          if (w.own_chol && db_tri_available(n)) {
            // no status of its own: the factor's status came back with the batch
            skip_info = true;
            db_launch_tri_solve_ld(w.LB + (size_t)slot * w.lb_stride, w.lb_ld, n, w.JTe, w.Dp,
                                   d.stream);
            w.step_fused = w.step_armed;
          } else if (w.bt_ws) {
            // no status of its own either
            skip_info = true;
            db_launch_bigtri_solve(w.LB + (size_t)slot * w.lb_stride, n, n, w.JTe, w.Dp, w.bt_ws,
                                   nullptr, d.stream);
          } else {
            DB_CHECK(cudaMemsetAsync(w.devinfo, 0, 2 * sizeof(int), d.stream));
            DB_CHECK(cudaMemcpyAsync(w.Dp, w.JTe, sizeof(double) * n, cudaMemcpyDeviceToDevice,
                                     d.stream));
            CS_CHECK(cusolverDnDpotrs(w.cs, CUBLAS_FILL_MODE_LOWER, n, 1,
                                      w.LB + (size_t)slot * w.lb_stride, n, w.Dp, n, w.devinfo + 1));
          }
          db_prof_end(d.stream);
          db_count_launch(1);
          issolved = (w.h_binfo[slot * w.binfo_step] == 0) ? 1 : 0;
        } else {
          issolved = enqueue_solve(pr, mu + half_rho, linsolv, eps1);
        }
        // p + dp, |dp|^2, dp.J^T e on the device; trial pass; everything back in one go
        if (w.step_armed) db_chol_set_step(nullptr, nullptr, nullptr, nullptr);
        if (!w.step_fused)
          db_launch_lm_step(pblk_dev, w.Dp, w.JTe, w.pnew, d.scal + 8, os ? nullptr : w.JTe_new, n,
                            d.stream);
        if (hidden_from) {
          // the last iteration ends with this trial if it is accepted: its J^T e would never be read,
          // its residual is the one the visit leaves behind
          const bool last = kiter == itmax - 1;
          db_cluster_pass(pr, k, w.pnew, hidden_from, last ? w.dbuf : nullptr, 1, last ? 1 : 0,
                          last ? nullptr : w.JTe_new, 1, t0, t1, nullptr, 1.0, true, w.pold,
                          true);
        } else {
          db_cluster_pass(pr, k, w.pnew, w.dbuf, nullptr, 1, 0, os ? nullptr : w.JTe_new, 1, t0, t1,
                          wt, 1.0, true);
        }
        if (aug)
          db_launch_lm_aug_rhs(w.JTe_new, w.pnew, aug->y_dev, aug->bz_dev, aug->rho, n, d.stream);
        if (!w.step_fused) db_count_launch(1);  // k_lm_step
        int *hinfo = (int *)(w.h_vec + 4 * n + 4 * d.N);
        DB_CHECK(cudaMemcpyAsync(d.h_scal, d.scal, sizeof(double) * (64 + 3 * n + 2),
                                 cudaMemcpyDeviceToHost, d.stream));
        // While the host waits for these results and decides, the GPU already assembles J^T J at the
        // trial point into the buffer the current system does not occupy: if the step is accepted
        // (the usual case) the next iteration finds its matrix ready, otherwise it is dropped.
        double *spec_buf = nullptr;
        if (w.own_chol && linsolv == 0 && !wt && !os && kiter + 1 < itmax && w.T_valid[tix]) {
          const double *cur = w.jtj0_cur ? w.jtj0_cur : w.JTJ0;
          spec_buf = (cur == w.JTJ0) ? w.JTJ : w.JTJ0;
          DB_CHECK(cudaEventRecord(w.ev_mail, d.stream));
          assemble(pr, Tfull, w.pnew, spec_buf);
          db_event_sync(w.ev_mail);
        } else {
          db_stream_sync(d.stream);
        }
        {
          const double *hm = d.h_scal + 64;
          memcpy(hDp, hm, sizeof(double) * n);
          hsc[n] = d.h_scal[8];
          hsc[n + 1] = d.h_scal[9];
          hsc[n + 2] = d.h_scal[1];
          if (!os) memcpy(hjte_new, hm + (w.JTe_new - w.Dp), sizeof(double) * n);
          if (pending_entry) memcpy(hjte, hm + (w.JTe - w.Dp), sizeof(double) * n);
          memcpy(hinfo, hm + 3 * n, 2 * sizeof(int));
          if (skip_info) hinfo[0] = hinfo[1] = 0;
        }
        if (pending_entry) {
          // the deferred entry tests, in the reference's order
          pending_entry = false;
          p_eL2 = init_p_eL2 = d.h_scal[2];
          if (!isfinite(p_eL2)) {
            stop = 7;
            kiter_adjust = 1;
            break;
          }
          if (p_eL2 <= eps3) {
            stop = 6;
            kiter_adjust = 1;
            break;
          }
          jacTe_inf = 0.0;
          for (int i = 0; i < n; i++) {
            double a = fabs(hjte[i]);
            if (a > jacTe_inf) jacTe_inf = a;
          }
          p_L2 = nrm2sq(hp, n);
          if (jacTe_inf <= eps1) {
            Dp_L2 = 0.0;
            stop = 1;
            kiter_adjust = 1;  // deferred entry tests only run for the non-OS LM
            break;
          }
        }
        if (issolved && linsolv != 2) issolved = (hinfo[0] == 0 && hinfo[1] == 0) ? 1 : 0;
        if (issolved) {
          Dp_L2 = hsc[n];
          if (Dp_L2 <= eps2_sq * p_L2) {
            stop = 2;
            break;
          }
          if (Dp_L2 >= (p_L2 + eps2) / (1e-12 * 1e-12)) {  // CLM_EPSILON, Dirac_common.h:45
            stop = 4;
            break;
          }
          // only now does the trial count as evaluated (the reference stops before evaluating it)
          if (wt)  // only the robust driver looks at the last evaluated point
            DB_CHECK(cudaMemcpyAsync(w.plast, w.pnew, sizeof(double) * n, cudaMemcpyDeviceToDevice,
                                     d.stream));
          *evaluated_trial = true;
          double pDp_eL2 = hsc[n + 2];
          if (aug) {
            for (int i = 0; i < n; i++) hpnew_aug(w)[i] = hp[i] + hDp[i];
            pDp_eL2 += aug_cost(aug, hpnew_aug(w), n);
          }
          if (!isfinite(pDp_eL2)) {
            stop = 7;
            break;
          }
          const double dL = mu * Dp_L2 + hsc[n + 1];  // dp^T (mu dp + J^T e)
          const double dF = p_eL2 - pDp_eL2;
          if (fabs(dF) <= 1e-11 * p_eL2) g_noise_decisions++;  // see dirac_b200_noise_decisions
          if (dL > 0.0 && dF > 0.0) {
            double tmp = (2.0 * dF / dL - 1.0);
            tmp = 1.0 - tmp * tmp * tmp;
            mu = mu * ((tmp >= 0.3333333334) ? tmp : 0.3333333334);  // CLM_ONE_THIRD
            g_lm_stat[0]++;                                // accepted steps
            if (!(tmp >= 0.3333333334)) g_lm_stat[1]++;    // ... that shrink mu by exactly 1/3
            nu = 2;
            for (int i = 0; i < n; i++) hp[i] += hDp[i];
            DB_CHECK(cudaMemcpyAsync(pblk_dev, w.pnew, sizeof(double) * n,
                                     cudaMemcpyDeviceToDevice, d.stream));
            if (!os) {
              memcpy(hjte, hjte_new, sizeof(double) * n);
              double *t = w.JTe; w.JTe = w.JTe_new; w.JTe_new = t;
            }
            p_eL2 = pDp_eL2;
            w.jtj_spec = spec_buf;
            res_in_dbuf = hidden_from && kiter == itmax - 1;
            break;
          }
        }
        g_lm_stat[2]++;
        mu *= (double)nu;
        nu2 = nu << 1;
        if (nu2 <= nu) {
          stop = 5;
          break;
        }
        nu = nu2;
      }
      if (stop) break;
    }
  }
  if (kiter >= itmax && !kiter_adjust) stop = 3;
  kiter -= kiter_adjust;
  *nu_damp = nu;
  out->init_eL2 = init_p_eL2;
  out->eL2 = p_eL2;
  out->jacTe_inf = jacTe_inf;
  out->Dp_L2 = Dp_L2;
  out->mu = mu;
  out->k = kiter;
  out->stop = stop;
  out->res_in_dbuf = res_in_dbuf;
}

static void fill_info(double *info, const LmOut &o) {
  if (!info) return;
  info[0] = o.init_eL2; info[1] = o.eL2; info[2] = o.jacTe_inf; info[3] = o.Dp_L2; info[4] = o.mu;
  info[5] = (double)o.k; info[6] = (double)o.stop;
  info[7] = info[8] = info[9] = 0.0;
}

// ------------------------------------------------------------------------------------------------
// LM on chunk ck of cluster k (clevmar / oslevmar).  `r` holds the residual of the full model over
// the whole interval; on return the chunk's rows of `r` are the residual with the updated Jones.
// pblk_dev points at the 8N parameters inside the device copy of pp (updated in place).
// info[0] = ||e||^2 at entry, info[1] = ||e||^2 at exit (lmfit.c:963-964 uses exactly these).
// ------------------------------------------------------------------------------------------------
void db_lm_set_aug(const double *y_dev, const double *bz_dev, const double *y_host,
                   const double *bz_host, double rho) {
  static LmAug a;
  if (!y_dev) {
    g_aug = nullptr;
    return;
  }
  a.y_dev = y_dev; a.bz_dev = bz_dev; a.y_host = y_host; a.bz_host = bz_host; a.rho = rho;
  g_aug = &a;
}

void db_lm_chunk(dirac_b200_problem *pr, int k, int ck, double *pblk_dev, double2 *r, int itmax,
                 const double *opts, int linsolv, int os, int randomize, double *info,
                 bool hidden_ready) {
  static const double defopts[4] = {1e-3, 1e-17, 1e-17, 1e-17};
  DevProblem &d = pr->d;
  db_lm_init(pr);
  LMWork &w = pr->lm;
  int t0, t1;
  chunk_range(d, k, ck, &t0, &t1);
  if (hidden_ready) {
    // the caller formed the hidden data of the WHOLE cluster in w.dbuf with the row-based chunk map
    // (db_cluster_hidden) and will form the residual the same way after the last chunk
    int nu = 2;
    bool ev;
    LmOut o;
    lm_core(pr, k, ck, t0, t1, pblk_dev, nullptr, itmax, opts ? opts : defopts, linsolv, os, 0,
            randomize, false, 0.0, &nu, &ev, nullptr, &o);
    fill_info(info, o);
    return;
  }
  // hidden data d = r + f(p_old); e = d - f(p_old); ||e||^2; J^T e  (lmfit.c:890-891 fused with
  // the first func/jacf evaluation, clmfit.c:241-252)
  // (sharded runs weight the residual share of the hidden data with beta, SAGE: d = f + beta r)
  const double beta = pr->world > 1 ? pr->beta : 1.0;
  // A plain LM visit of a one-chunk cluster never stores the hidden data: every pass forms it again
  // from r and the entry Jones (w.pold), which costs no traffic, and the trial of the last iteration
  // writes the residual, so that the closing pass is only needed when the visit ends otherwise.  A
  // cluster of several chunks keeps d: the last trial covers only the chunk's rows of the residual.
  const bool form = !os && pr->world <= 1 && d.h_clus[k].nchunk == 1 && r == pr->res &&
                    db_cluster_pass_forms_hidden(d.N, d.Nbase);
  // the sharded closing pass recovers the old residual from the Jones the visit started with
  if (beta != 1.0 || form)
    DB_CHECK(cudaMemcpyAsync(w.pold, pblk_dev, sizeof(double) * w.n8, cudaMemcpyDeviceToDevice,
                             d.stream));
  db_cluster_pass(pr, k, pblk_dev, r, form ? nullptr : w.dbuf, 0, form ? 0 : 1,
                  os ? nullptr : w.JTe, 2, t0, t1, nullptr, beta);
  // ||e||^2 at entry stays on the device for now: lm_core fetches it together with p and J^T e
  // (NaN = "still in d.scal[2]")
  const double c0 = nan("");
  int nu = 2;
  bool ev;
  LmOut o;
  lm_core(pr, k, ck, t0, t1, pblk_dev, nullptr, itmax, opts ? opts : defopts, linsolv, os, 0,
          randomize, true, c0, &nu, &ev, form ? r : nullptr, &o);
  // residual of the chunk with the final Jones: r = d - f(p) (+ (1-beta) r when sharded)
  // (lmfit.c:980-981)
  if (o.res_in_dbuf) {
    pr->res = w.dbuf;
    w.dbuf = r;
  } else if (form) {
    db_cluster_pass(pr, k, pblk_dev, r, r, 3, 1, nullptr, 1, t0, t1, nullptr, 1.0, false,
                    w.pold, true);
  } else {
    db_cluster_pass(pr, k, pblk_dev, w.dbuf, r, 3, 1, nullptr, 1, t0, t1, nullptr, beta,
                    false, beta != 1.0 ? w.pold : nullptr);
  }
  fill_info(info, o);
}

// Hybrid cluster whose chunks do not tile the interval evenly (tilesz % nchunk != 0): the reference
// adds / subtracts the cluster's model with the ROW-based chunk map px = row / ceil(R/nchunk)
// (mylm_fit_single_pth, lmfit.c:86,890,980) while the LM fits of its chunks run over the timeslot
// ranges [ck*ceil(tilesz/nchunk), ...) (lmfit.c:893-905); near the boundaries the hidden data then
// carries another chunk's Jones.  sign > 0: w.dbuf = beta r + f_k(pp); sign < 0: r = w.dbuf - f_k(pp)
// (+ (1-beta) r when beta != 1, i.e. when sharded).
bool db_cluster_needs_rowmap(const dirac_b200_problem *pr, int k) {
  const int nchunk = pr->d.h_clus[k].nchunk;
  return nchunk > 1 && (pr->d.tilesz % nchunk) != 0;
}
void db_cluster_hidden(dirac_b200_problem *pr, int k, double2 *r, int sign, double beta) {
  DevProblem &d = pr->d;
  db_lm_init(pr);
  LMWork &w = pr->lm;
  const double2 *coh_k = d.coh + (size_t)k * 4 * d.R;
  const int *poff = d.chunk_poff + d.h_clus[k].chunk0;
  if (sign > 0)
    db_launch_cluster_rowmap(coh_k, r, nullptr, w.dbuf, d.flag, d.pp, poff, d.h_clus[k].nchunk,
                             d.blpq, d.R, d.Nbase, 1, beta, d.stream);
  else
    db_launch_cluster_rowmap(coh_k, w.dbuf, beta != 1.0 ? r : nullptr, r, d.flag, d.pp, poff,
                             d.h_clus[k].nchunk, d.blpq, d.R, d.Nbase, -1, beta, d.stream);
  db_count_launch(1);
}

// digamma (updatenu.c:36-49)
static double digamma_(double x) {
  double result = 0.0, xx, xx2, xx4;
  for (; x < 7.0; ++x) result -= 1.0 / x;
  x -= 0.5;
  xx = 1.0 / x;
  xx2 = xx * xx;
  xx4 = xx2 * xx2;
  result += log(x) + (1. / 24.) * xx2 - (7.0 / 960.0) * xx4 + (31.0 / 8064.0) * xx4 * xx2 -
            (127.0 / 30720.0) * xx4 * xx4;
  return result;
}

// nu of the 30-point grid on [nulow, nuhigh) with the smallest |psi((nu+1)/2) - ln((nu+1)/2) -
// psi(nu/2) + ln(nu/2) - sumq + 1|   (q_update_threadfn + idamin, updatenu.c:86-104,237-262)
static double pick_nu(double sumq, double nulow, double nuhigh) {
  const int Nd = 30;
  const double deltanu = (nuhigh - nulow) / (double)Nd;
  int best = 0;
  double bestv = 0.0;
  for (int ci = 0; ci < Nd; ci++) {
    const double thisnu = nulow + (double)ci * deltanu;
    double q = digamma_(thisnu * 0.5 + 0.5) - log((thisnu + 1.0) * 0.5);
    q += -digamma_(thisnu * 0.5) + log(thisnu * 0.5);
    q += -sumq + 1.0;
    if (ci == 0 || fabs(q) < bestv) {
      bestv = fabs(q);
      best = ci;
    }
  }
  return nulow + (double)best * deltanu;
}

// The update between two IRLS rounds of the robust LM on the rows of tiles [t0, t1) (robustlm.c:
// 2533-2566): e = d - f(pe) unweighted from the hidden data in w.dbuf, lambda = sum |w_old|, w_i =
// sqrt((nu0+1)/(nu0+e_i^2)) into w.wbuf, sumq = mean |w - log w|, nu by pick_nu, then the weights
// scaled by lambda / ndata.  Returns the new nu; out3 (optional) gets (lambda, sumq, nu).
static double irls_update(dirac_b200_problem *pr, int k, int t0, int t1, const double *pe,
                          double nu0, double nulow, double nuhigh, double *out3) {
  DevProblem &d = pr->d;
  LMWork &w = pr->lm;
  const long long r0 = (long long)t0 * d.Nbase, r1 = (long long)t1 * d.Nbase;
  const double ndata = 8.0 * (double)(r1 - r0);
  db_cluster_pass(pr, k, pe, w.dbuf, w.ebuf, 1, 1, nullptr, 2, t0, t1, nullptr);
  db_launch_sum_abs(w.wbuf, d.R, r0, r1, pr->partials, d.scal + 3, d.counters, d.stream);
  db_launch_update_weights(w.ebuf, w.wbuf, d.R, r0, r1, nu0, pr->partials, d.scal + 4, d.counters,
                           d.stream);
  db_count_launch(2);
  DB_CHECK(cudaMemcpyAsync(d.h_scal + 3, d.scal + 3, 2 * sizeof(double), cudaMemcpyDeviceToHost,
                           d.stream));
  db_stream_sync(d.stream);
  const double lambda = d.h_scal[3];
  const double sumq = d.h_scal[4] / ndata;
  const double nu = pick_nu(sumq, nulow, nuhigh);
  db_launch_scale_vis(w.wbuf, d.R, r0, r1, lambda / ndata, 0, d.stream);
  db_count_launch(1);
  if (out3) {
    out3[0] = lambda;
    out3[1] = sumq;
    out3[2] = nu;
  }
  return nu;
}

// ------------------------------------------------------------------------------------------------
// robust LM on chunk ck of cluster k (rlevmar / osrlevmar): three IRLS rounds of weighted LM;
// between rounds w_i = sqrt((nu+1)/(nu+e_i^2)) from the unweighted residual, nu re-estimated,
// weights rescaled to the previous mean (robustlm.c:2533-2566).
// ------------------------------------------------------------------------------------------------
void db_rlm_chunk(dirac_b200_problem *pr, int k, int ck, double *pblk_dev, double2 *r, int itmax,
                  int linsolv, int os, int randomize, double nulow, double nuhigh,
                  double *robust_nu, double *info, bool hidden_ready) {
  static const double defopts[4] = {1e-3, 1e-17, 1e-17, 1e-17};  // opts == NULL (lmfit.c:917)
  const int wt_itmax = 3;
  DevProblem &d = pr->d;
  db_lm_init(pr);
  robust_init(pr);
  LMWork &w = pr->lm;
  const int n8 = w.n8;
  int t0, t1;
  chunk_range(d, k, ck, &t0, &t1);
  const long long r0 = (long long)t0 * d.Nbase, r1 = (long long)t1 * d.Nbase;
  // hidden data d = beta r + f(p_old)
  const double beta = pr->world > 1 ? pr->beta : 1.0;
  if (!hidden_ready) {
    if (beta != 1.0)
      DB_CHECK(cudaMemcpyAsync(w.pold, pblk_dev, sizeof(double) * w.n8, cudaMemcpyDeviceToDevice,
                               d.stream));
    db_cluster_pass(pr, k, pblk_dev, r, w.dbuf, 2, 1, nullptr, 1, t0, t1, nullptr, beta);
  }
  if (r1 > r0) db_launch_scale_vis(w.wbuf, d.R, r0, r1, 1.0, 1, d.stream);  // wt = 1
  db_count_launch(1);
  double nu_t = *robust_nu;
  int nu = 2;
  LmOut o;
  memset(&o, 0, sizeof(o));
  for (int nw = 0; nw < wt_itmax; nw++) {
    bool evaluated = false;
    lm_core(pr, k, ck, t0, t1, pblk_dev, w.wbuf, itmax, defopts, linsolv, os, nw, randomize, false,
            0.0, &nu, &evaluated, nullptr, &o);
    if (nw < wt_itmax - 1 && r1 > r0) {
      // residual the new weights are computed from: at nw == 0 the reference's `ed` is the
      // (unit-weight) residual of the LAST evaluated point, which is a rejected trial if the loop
      // stopped right after one (clmfit.c:478); later rounds recompute it at p (robustlm.c:2538)
      const double *pe = (nw == 0 && evaluated) ? w.plast : pblk_dev;
      nu_t = irls_update(pr, k, t0, t1, pe, nu_t, nulow, nuhigh, nullptr);
    }
  }
  *robust_nu = nu_t;
  // residual of the chunk with the final Jones: r = d - f(p) (+ (1-beta) r when sharded)
  if (!hidden_ready)
    db_cluster_pass(pr, k, pblk_dev, w.dbuf, r, 3, 1, nullptr, 1, t0, t1, nullptr, beta, false,
                    beta != 1.0 ? w.pold : nullptr);
  (void)n8;
  fill_info(info, o);
}

// ------------------------------------------------------------------------------------------------
// thin C-ABI: normal equations of one (cluster, chunk) against caller-supplied hidden data
// ------------------------------------------------------------------------------------------------
extern "C" double dirac_b200_normal_eq(dirac_b200_problem *pr, int clus, int chunk,
                                       const double *pblk, const double *xd, double *JTJ,
                                       double *JTe) {
  DevProblem &d = pr->d;
  db_lm_init(pr);
  LMWork &w = pr->lm;
  const int n = w.n8;
  int t0, t1;
  chunk_range(d, clus, chunk, &t0, &t1);
  db_upload_vis(pr, xd, w.dbuf);
  DB_CHECK(cudaMemcpyAsync(w.pnew, pblk, sizeof(double) * n, cudaMemcpyHostToDevice, d.stream));
  db_cluster_pass(pr, clus, w.pnew, w.dbuf, nullptr, 1, 0, w.JTe, 1, t0, t1, nullptr);
  gram(pr, clus, t0, t1, 1, w.Tsub);
  assemble(pr, w.Tsub, w.pnew, w.JTJ0);
  double c = db_read_scalar(pr, 1);
  if (JTe) DB_CHECK(cudaMemcpy(JTe, w.JTe, sizeof(double) * n, cudaMemcpyDeviceToHost));
  if (JTJ)
    DB_CHECK(cudaMemcpy(JTJ, w.JTJ0, sizeof(double) * (size_t)n * n, cudaMemcpyDeviceToHost));
  DB_CHECK(cudaGetLastError());
  return c;
}

// same with sqrt-weights wt (8 per row, API layout, full interval): the robust LM's weighted system
extern "C" double dirac_b200_normal_eq_weighted(dirac_b200_problem *pr, int clus, int chunk,
                                                const double *pblk, const double *xd,
                                                const double *wt, double *JTJ, double *JTe) {
  DevProblem &d = pr->d;
  db_lm_init(pr);
  robust_init(pr);
  LMWork &w = pr->lm;
  const int n = w.n8;
  int t0, t1;
  chunk_range(d, clus, chunk, &t0, &t1);
  db_upload_vis(pr, xd, w.dbuf);
  db_upload_vis(pr, wt, w.wbuf);
  DB_CHECK(cudaMemcpyAsync(w.pnew, pblk, sizeof(double) * n, cudaMemcpyHostToDevice, d.stream));
  db_cluster_pass(pr, clus, w.pnew, w.dbuf, nullptr, 1, 0, w.JTe, 1, t0, t1, w.wbuf);
  weighted_jtj(pr, clus, t0, t1, w.pnew, w.wbuf, w.JTJ0);
  double c = db_read_scalar(pr, 1);
  if (JTe) DB_CHECK(cudaMemcpy(JTe, w.JTe, sizeof(double) * n, cudaMemcpyDeviceToHost));
  if (JTJ)
    DB_CHECK(cudaMemcpy(JTJ, w.JTJ0, sizeof(double) * (size_t)n * n, cudaMemcpyDeviceToHost));
  DB_CHECK(cudaGetLastError());
  return c;
}

// ------------------------------------------------------------------------------------------------
// test hooks of the damped assembly: J^T J + mu I of one (cluster, chunk) at pblk, lower triangle
// only, for each mu in turn in the same buffer (factor: dpotrf(LOWER) in place after each write, so
// every later mu rebuilds over the previous factor).  out [nmu][8N][8N], info [nmu] (factor only).
// ------------------------------------------------------------------------------------------------
extern "C" void dirac_b200_assemble_damped(dirac_b200_problem *pr, int clus, int chunk,
                                           const double *pblk, int nmu, const double *mus,
                                           int factor, double *out, int *info) {
  DevProblem &d = pr->d;
  db_lm_init(pr);
  LMWork &w = pr->lm;
  const int n = w.n8;
  int t0, t1;
  chunk_range(d, clus, chunk, &t0, &t1);
  DB_CHECK(cudaMemcpyAsync(w.pnew, pblk, sizeof(double) * n, cudaMemcpyHostToDevice, d.stream));
  gram(pr, clus, t0, t1, 1, w.Tsub);
  assemble(pr, w.Tsub, w.pnew, nullptr);
  for (int i = 0; i < nmu; i++) {
    AssembleArgs a = assemble_args(d, w.Tsub, w.pnew, w.Hst);
    a.JTJ = w.JTJ;
    a.mu = mus[i];
    a.lower = 1;
    assemble_tiles(pr, a, 1);
    if (factor)
      CS_CHECK(cusolverDnDpotrf(w.cs, CUBLAS_FILL_MODE_LOWER, n, w.JTJ, n, w.cswork, w.lwork,
                                w.devinfo));
    DB_CHECK(cudaMemcpyAsync(out + (size_t)i * n * n, w.JTJ, sizeof(double) * (size_t)n * n,
                             cudaMemcpyDeviceToHost, d.stream));
    if (factor)
      DB_CHECK(cudaMemcpyAsync(info + i, w.devinfo, sizeof(int), cudaMemcpyDeviceToHost, d.stream));
    db_stream_sync(d.stream);
  }
  DB_CHECK(cudaGetLastError());
}

// the batched assembly of the sweep's first systems over the local clusters list[0..nb) (first
// chunk each, Jones from the full vector pp, which replaces the problem's): mu0 = tau max diag -> mu_out [nb]; out [nb][8N][8N]
// gets J^T J + mu0 I, lower triangle only (lower) or the full undamped matrix
extern "C" void dirac_b200_assemble_batch(dirac_b200_problem *pr, const double *pp, const int *list,
                                          int nb, double tau, int lower, double *mu_out, double *out) {
  DevProblem &d = pr->d;
  db_lm_init(pr);
  DB_CHECK(cudaMemcpy(d.pp, pp, sizeof(double) * d.npar, cudaMemcpyHostToDevice));
  LMWork &w = pr->lm;
  const size_t nn = (size_t)w.n8 * w.n8;
  std::vector<int> tix(d.M), poff(d.M);
  for (int k = 0; k < d.M; k++) {
    tix[k] = d.h_clus[k].chunk0;
    poff[k] = d.h_chunk_poff[tix[k]];
  }
  for (int y = 0; y < nb; y++) {
    const int k = list[y];
    int t0, t1;
    chunk_range(d, k, 0, &t0, &t1);
    gram(pr, k, t0, t1, 1, w.T + (size_t)tix[k] * d.Nbase * 16);
    w.T_valid[tix[k]] = 1;
  }
  int *ibuf = dalloc<int>(nb + 2 * d.M);
  double *H = dalloc<double>((size_t)4 * d.N * nb), *mu = dalloc<double>(nb);
  double *A = dalloc<double>(nn * nb);
  DB_CHECK(cudaMemcpy(ibuf, list, sizeof(int) * nb, cudaMemcpyHostToDevice));
  DB_CHECK(cudaMemcpy(ibuf + nb, tix.data(), sizeof(int) * d.M, cudaMemcpyHostToDevice));
  DB_CHECK(cudaMemcpy(ibuf + nb + d.M, poff.data(), sizeof(int) * d.M, cudaMemcpyHostToDevice));
  AssembleArgs b = assemble_args(d, w.T, d.pp, H);
  b.list = ibuf; b.tix = ibuf + nb; b.poff = ibuf + nb + d.M;
  b.JTJ = A;
  b.stride = (long long)nn;
  station_sums(pr, b, nb);
  db_launch_batch_mu0(H, mu, d.N, tau, nb, d.stream);
  if (lower) {
    b.mu_dev = mu;
    b.lower = 1;
  }
  assemble_tiles(pr, b, nb);
  DB_CHECK(cudaMemcpyAsync(mu_out, mu, sizeof(double) * nb, cudaMemcpyDeviceToHost, d.stream));
  DB_CHECK(cudaMemcpyAsync(out, A, sizeof(double) * nn * nb, cudaMemcpyDeviceToHost, d.stream));
  db_stream_sync(d.stream);
  db_free(ibuf); db_free(H); db_free(mu); db_free(A);
  DB_CHECK(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------
// test hooks (not in the public header): the ordered-subsets system, the IRLS update and the chunk
// solves of the LM, each through the code the solvers run, on caller-supplied hidden data
// ------------------------------------------------------------------------------------------------
// J^T J and J^T e that lm_core forms for subset l of chunk `chunk` of cluster clus at pblk, on hidden
// data xd with sqrt-weights wt (API layout, full interval) or none.  path = (misaligned, s0, s1, nJ).
extern "C" void dirac_b200_os_normal_eq(dirac_b200_problem *pr, int clus, int chunk, int l,
                                        const double *pblk, const double *xd, const double *wt,
                                        double *JTJ, double *JTe, long long *path) {
  DevProblem &d = pr->d;
  db_lm_init(pr);
  robust_init(pr);
  LMWork &w = pr->lm;
  const int n = w.n8;
  int t0, t1;
  chunk_range(d, clus, chunk, &t0, &t1);
  db_upload_vis(pr, xd, w.dbuf);
  if (wt) db_upload_vis(pr, wt, w.wbuf);
  DB_CHECK(cudaMemcpyAsync(w.pnew, pblk, sizeof(double) * n, cudaMemcpyHostToDevice, d.stream));
  const OsPath p = os_subset_system(pr, clus, t0, t1, l, w.pnew, wt ? w.wbuf : nullptr);
  DB_CHECK(cudaMemcpyAsync(JTe, w.JTe, sizeof(double) * n, cudaMemcpyDeviceToHost, d.stream));
  DB_CHECK(cudaMemcpyAsync(JTJ, w.JTJ0, sizeof(double) * (size_t)n * n, cudaMemcpyDeviceToHost,
                           d.stream));
  db_stream_sync(d.stream);
  DB_CHECK(cudaGetLastError());
  path[0] = p.misaligned ? 1 : 0;
  path[1] = p.s0;
  path[2] = p.s1;
  path[3] = p.nJ;
}

// the update between two IRLS rounds on chunk `chunk` of cluster clus: residual at pblk of the
// hidden data xd, new weights from wt_inout (API layout, full interval; rows outside the chunk are
// left as they are) with nu0, nu of [nulow, nuhigh).  out3 = (lambda, sumq, nu).
extern "C" void dirac_b200_irls_update(dirac_b200_problem *pr, int clus, int chunk,
                                       const double *pblk, const double *xd, double *wt_inout,
                                       double nu0, double nulow, double nuhigh, double *out3) {
  DevProblem &d = pr->d;
  db_lm_init(pr);
  robust_init(pr);
  LMWork &w = pr->lm;
  int t0, t1;
  chunk_range(d, clus, chunk, &t0, &t1);
  db_upload_vis(pr, xd, w.dbuf);
  db_upload_vis(pr, wt_inout, w.wbuf);
  DB_CHECK(cudaMemcpyAsync(w.pnew, pblk, sizeof(double) * w.n8, cudaMemcpyHostToDevice, d.stream));
  irls_update(pr, clus, t0, t1, w.pnew, nu0, nulow, nuhigh, out3);
  db_download_vis(pr, w.wbuf, wt_inout);
  DB_CHECK(cudaGetLastError());
}

// LM (robust == 0: clevmar / oslevmar) or robust LM (rlevmar / osrlevmar) of chunk `chunk` of
// cluster clus on hidden data xd, from pblk_inout (updated).  opts: the plain LM's (tau, eps1..3) or
// null; the robust LM uses its own.  nu_inout: the robust LM's nu.  info[10] as the reference's.
extern "C" void dirac_b200_lm_chunk(dirac_b200_problem *pr, int clus, int chunk, double *pblk_inout,
                                    const double *xd, int itmax, const double *opts, int linsolv,
                                    int os, int robust, double nulow, double nuhigh,
                                    double *nu_inout, double *info) {
  DevProblem &d = pr->d;
  db_lm_init(pr);
  LMWork &w = pr->lm;
  const int n = w.n8;
  db_upload_vis(pr, xd, w.dbuf);
  double *pblk_dev = w.pold;
  DB_CHECK(cudaMemcpyAsync(pblk_dev, pblk_inout, sizeof(double) * n, cudaMemcpyHostToDevice,
                           d.stream));
  if (robust)
    db_rlm_chunk(pr, clus, chunk, pblk_dev, pr->res, itmax, linsolv, os, 0, nulow, nuhigh, nu_inout,
                 info, true);
  else
    db_lm_chunk(pr, clus, chunk, pblk_dev, pr->res, itmax, opts, linsolv, os, 0, info, true);
  DB_CHECK(cudaMemcpyAsync(pblk_inout, pblk_dev, sizeof(double) * n, cudaMemcpyDeviceToHost,
                           d.stream));
  db_stream_sync(d.stream);
  DB_CHECK(cudaGetLastError());
}

// One streaming pass of chunk `chunk` of cluster clus through db_cluster_pass, as the LM visits make it:
// mode 0-4 (ClusterPassArgs), output written or not, J^T e or not, the hidden data formed per row from
// `in` and pblk_old (form_hidden), hidden-data weight beta.  pblk, pblk_old (or null): 8N Jones; in,
// wt (or null) and out_init: API layout, full interval.  The device output vector holds out_init
// before the pass, or is the input vector itself (inplace).  out gets that vector after the pass (all
// rows), jte [8N] J^T e (0 without), cost the slot the mode writes (slot 2 for mode 0, 1 for modes 1
// and 4; 0 for ADD / SUB, which have none).  Returns the kernel launched (DB_CP_*), or -1 before any
// device work for a bad cluster, chunk or mode, mode 4 without J^T e, ADD / SUB with it, form_hidden
// outside modes 1 and 3, with weights or where the linear-mapped kernel does not run, and a missing
// pblk_old where form_hidden or a SUB with beta != 1 needs it.
extern "C" int dirac_b200_cluster_pass_eval(dirac_b200_problem *pr, int clus, int chunk, int mode,
                                            int write_out, int with_jte, int form_hidden, double beta,
                                            const double *pblk, const double *pblk_old,
                                            const double *in, const double *wt,
                                            const double *out_init, int inplace, double *out,
                                            double *jte, double *cost) {
  DevProblem &d = pr->d;
  if (clus < 0 || clus >= d.M || chunk < 0 || chunk >= d.h_clus[clus].nchunk) return -1;
  if (mode < 0 || mode > 4 || (mode == 4 && !with_jte) || ((mode == 2 || mode == 3) && with_jte))
    return -1;
  if (form_hidden &&
      ((mode != 1 && mode != 3) || wt || !db_cluster_pass_forms_hidden(d.N, d.Nbase)))
    return -1;
  if (!pblk_old && (form_hidden || (mode == 3 && beta != 1.0))) return -1;
  db_lm_init(pr);
  LMWork &w = pr->lm;
  const int n = w.n8;
  int t0, t1;
  chunk_range(d, clus, chunk, &t0, &t1);
  double2 *vin = dalloc<double2>((size_t)4 * d.R);
  double2 *vout = inplace ? vin : dalloc<double2>((size_t)4 * d.R);
  double2 *vwt = wt ? dalloc<double2>((size_t)4 * d.R) : nullptr;
  double *pb = dalloc<double>((size_t)2 * n);
  db_upload_vis(pr, in, vin);
  if (!inplace) db_upload_vis(pr, out_init, vout);
  if (wt) db_upload_vis(pr, wt, vwt);
  DB_CHECK(cudaMemcpyAsync(pb, pblk, sizeof(double) * n, cudaMemcpyHostToDevice, d.stream));
  if (pblk_old)
    DB_CHECK(cudaMemcpyAsync(pb + n, pblk_old, sizeof(double) * n, cudaMemcpyHostToDevice, d.stream));
  const int slot = mode == 0 ? 2 : 1;
  const int kernel = db_cluster_pass(pr, clus, pb, vin, vout, mode, write_out,
                                     with_jte ? w.JTe : nullptr, slot, t0, t1, vwt, beta, false,
                                     pblk_old ? pb + n : nullptr, form_hidden != 0);
  db_download_vis(pr, vout, out);
  if (with_jte)
    DB_CHECK(cudaMemcpy(jte, w.JTe, sizeof(double) * n, cudaMemcpyDeviceToHost));
  else
    memset(jte, 0, sizeof(double) * n);
  *cost = (mode <= 1 || mode == 4) ? db_read_scalar(pr, slot) : 0.0;
  db_free(vin);
  if (!inplace) db_free(vout);
  db_free(vwt);
  db_free(pb);
  DB_CHECK(cudaGetLastError());
  return kernel;
}

// db_cluster_hidden: the row-mapped add (sign > 0) or subtract (sign < 0) of cluster clus's model at
// the full Jones vector pp (it replaces the problem's), with hidden-data weight beta, on the residual
// r and the hidden data dh (API layout, full interval).  out gets what the call writes: the hidden
// data (sign > 0) or the residual (sign < 0).  Returns -1 for a bad cluster or sign 0 before any
// device work.
extern "C" int dirac_b200_cluster_hidden_eval(dirac_b200_problem *pr, int clus, int sign, double beta,
                                              const double *pp, const double *r, const double *dh,
                                              double *out) {
  DevProblem &d = pr->d;
  if (clus < 0 || clus >= d.M || sign == 0) return -1;
  db_lm_init(pr);
  LMWork &w = pr->lm;
  double2 *vr = dalloc<double2>((size_t)4 * d.R);
  DB_CHECK(cudaMemcpyAsync(d.pp, pp, sizeof(double) * d.npar, cudaMemcpyHostToDevice, d.stream));
  db_upload_vis(pr, r, vr);
  db_upload_vis(pr, dh, w.dbuf);
  db_cluster_hidden(pr, clus, vr, sign, beta);
  db_download_vis(pr, sign > 0 ? w.dbuf : vr, out);
  db_free(vr);
  DB_CHECK(cudaGetLastError());
  return 0;
}

// micro-benchmark of the all-cluster predict (cost_mode 1, no output): average device time in us
extern "C" double dirac_b200_bench_predict(dirac_b200_problem *pr, int out_mode, int reps) {
  DevProblem &d = pr->d;
  cudaEvent_t e0, e1;
  DB_CHECK(cudaEventCreate(&e0));
  DB_CHECK(cudaEventCreate(&e1));
  for (int i = 0; i < 2; i++) db_predict_dev(pr, d.pp, pr->res, out_mode, 1, 0.0, 0);
  DB_CHECK(cudaEventRecord(e0, d.stream));
  for (int i = 0; i < reps; i++) db_predict_dev(pr, d.pp, pr->res, out_mode, 1, 0.0, 0);
  DB_CHECK(cudaEventRecord(e1, d.stream));
  db_event_sync(e1);
  float ms = 0.f;
  DB_CHECK(cudaEventElapsedTime(&ms, e0, e1));
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  return 1e3 * ms / reps;
}

extern "C" double dirac_b200_bench_grad(dirac_b200_problem *pr, int reps) {
  DevProblem &d = pr->d;
  cudaEvent_t e0, e1;
  DB_CHECK(cudaEventCreate(&e0));
  DB_CHECK(cudaEventCreate(&e1));
  db_predict_dev(pr, d.pp, pr->res, 1, 0, 0.0, 0);
  for (int i = 0; i < 2; i++) db_grad_dev(pr, d.pp, pr->g, 0, 0.0);
  DB_CHECK(cudaEventRecord(e0, d.stream));
  for (int i = 0; i < reps; i++) db_grad_dev(pr, d.pp, pr->g, 0, 0.0);
  DB_CHECK(cudaEventRecord(e1, d.stream));
  db_event_sync(e1);
  float ms = 0.f;
  DB_CHECK(cudaEventElapsedTime(&ms, e0, e1));
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  return 1e3 * ms / reps;
}

// micro-benchmark of one k_cluster_pass configuration on the resident problem: average device time
// (us, CUDA events on the launching stream) of `reps` back-to-back launches over the full interval.
// with_grad: also accumulate J^T e; write_out: write the residual.
extern "C" double dirac_b200_bench_cluster_pass(dirac_b200_problem *pr, int clus, int mode,
                                                int with_grad, int write_out, int reps) {
  DevProblem &d = pr->d;
  db_lm_init(pr);
  LMWork &w = pr->lm;
  double *pblk = d.pp + d.h_chunk_poff[d.h_clus[clus].chunk0];
  cudaEvent_t e0, e1;
  DB_CHECK(cudaEventCreate(&e0));
  DB_CHECK(cudaEventCreate(&e1));
  for (int i = 0; i < 3; i++)
    db_cluster_pass(pr, clus, pblk, pr->res, w.dbuf, mode, write_out, with_grad ? w.JTe : nullptr,
                    1, 0, d.tilesz, nullptr);
  DB_CHECK(cudaEventRecord(e0, d.stream));
  for (int i = 0; i < reps; i++)
    db_cluster_pass(pr, (clus + i) % d.M, pblk, pr->res, w.dbuf, mode, write_out,
                    with_grad ? w.JTe : nullptr, 1, 0, d.tilesz, nullptr);
  DB_CHECK(cudaEventRecord(e1, d.stream));
  db_event_sync(e1);
  float ms = 0.f;
  DB_CHECK(cudaEventElapsedTime(&ms, e0, e1));
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  return 1e3 * ms / reps;
}
