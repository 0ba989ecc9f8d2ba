// Blocked Cholesky of the sweep's first large LM systems (8N > 1024; C4: 32 systems of 4096 x 4096)
// as one batch, on cuBLAS / cuSOLVER calls.
//
// Right-looking, LOWER, in place, column-major with ld = n: the layout dpotrf(LOWER) leaves, so the
// substitutions downstream (kernels_bigtri.cu, dpotrs) read the factor unchanged.  Panels of BC_BLOCK
// columns (the last one ragged: n = 8N is only a multiple of 8); for panel j, over all systems at once
//   L_jj = chol(A_jj)                 cusolverDnDpotrfBatched
//   X = L_jj^-1                       cublasDtrsmBatched on the identity (BC_BLOCK x BC_BLOCK)
//   L_ij = A_ij X^T, i > j            one cublasDgemmStridedBatched into a scratch panel, copied back
//                                     (a tall cublasDtrsmBatched took 1.8x as long)
//   A_cc.. -= L_c.j L_cj^T, c > j     one cublasDgemmStridedBatched per block column c, rows from its
//                                     diagonal block down: no FLOPs on the upper part
// Most FLOPs are in the trailing DGEMMs (FP64 tensor cores), and every call spans the whole batch,
// where cusolverDnDpotrf on one 4096 system leaves most SMs idle in its panel phases.  The panels
// (diagonal factors and solves) run far below the DGEMM rate, so they look ahead: block column j+1 is
// updated first and its panel runs on a second stream while the rest of panel j's update runs.  A single
// system stays with dpotrf: the same blocking on one system, with look-ahead on a second stream, took
// twice as long as dpotrf at n = 4096 on H100 (DESIGN.md §5.2).
//
// The strict upper triangle of the diagonal blocks is scratch (the DGEMM of a block column covers
// its whole diagonal block); the strict upper triangle outside them is neither read nor written.
//
// info as dpotrf: the 1-based global index of the first non-positive pivot, 0 if none.  Each diagonal
// block's status goes to its own slot; a last small kernel keeps the first failing panel's.
#include <vector>

#include "problem.h"

#define BC_CS(call)                                                                        \
  do {                                                                                     \
    cusolverStatus_t s__ = (call);                                                         \
    if (s__ != CUSOLVER_STATUS_SUCCESS) {                                                  \
      fprintf(stderr, "dirac_b200: cuSOLVER error %d at %s:%d\n", (int)s__, __FILE__, __LINE__); \
      exit(1);                                                                             \
    }                                                                                      \
  } while (0)
#define BC_CB(call)                                                                        \
  do {                                                                                     \
    cublasStatus_t s__ = (call);                                                           \
    if (s__ != CUBLAS_STATUS_SUCCESS) {                                                    \
      fprintf(stderr, "dirac_b200: cuBLAS error %d at %s:%d\n", (int)s__, __FILE__, __LINE__); \
      exit(1);                                                                             \
    }                                                                                      \
  } while (0)


struct BigChol {
  int n, nbk, np;       // order, panel width, panels
  int maxb;             // systems the batch pointers cover (0: none bound)
  double *A0;           // batch: system b at A0 + b * stride
  long long stride;
  double **ptr;         // device [np][2][maxb]: diagonal block, block below it, of every panel
  int *pinfo;           // device [np][maxb]: status of each diagonal block
  bool inv_panel;       // panel solve as L_jj^-1 (trsm on nbk x nbk) and one DGEMM, not a tall trsm
  double *X, *W;        // inv_panel: [maxb][nbk][nbk] inverses, [maxb][nbk][n] the solved panel
  double **Xptr;        // inv_panel: [maxb] pointers into X
  bool lookahead;       // panel j+1 on a second stream while the rest of panel j's update runs
};

namespace {

// library handles: process-wide, as lm.cu's (creating them costs tens of ms)
// ([1]: the look-ahead stream's)
struct Lib {
  cublasHandle_t cb[2];
  cusolverDnHandle_t cs[2];
  cudaStream_t side;
  cudaEvent_t ev_main, ev_side;
};
Lib &lib() {
  static Lib L;
  static bool made = false;
  if (!made) {
    for (int i = 0; i < 2; i++) {
      BC_CB(cublasCreate(&L.cb[i]));
      BC_CS(cusolverDnCreate(&L.cs[i]));
    }
    DB_CHECK(cudaStreamCreateWithFlags(&L.side, cudaStreamNonBlocking));
    DB_CHECK(cudaEventCreateWithFlags(&L.ev_main, cudaEventDisableTiming));
    DB_CHECK(cudaEventCreateWithFlags(&L.ev_side, cudaEventDisableTiming));
    BC_CB(cublasSetStream(L.cb[1], L.side));
    BC_CS(cusolverDnSetStream(L.cs[1], L.side));
    made = true;
  }
  return L;
}

inline int width(int n, int nbk, int j) { return (n - j * nbk) < nbk ? n - j * nbk : nbk; }

__global__ void k_bigchol_info(const int *pinfo, int np, int nbk, int ld, int nb, int *info,
                               int info_step) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nb) return;
  int v = 0;
  for (int j = 0; j < np; j++) {
    const int l = pinfo[(size_t)j * ld + b];
    if (l != 0) {
      v = l > 0 ? j * nbk + l : l;
      break;
    }
  }
  info[(size_t)b * info_step] = v;
}

// A_cc.. -= L_c.j L_cj^T for the block columns c in [c0, c1) of nb systems stride apart
void trailing(cublasHandle_t cb, double *A, long long stride, int nb, int n, int nbk, int j, int c0,
              int c1) {
  const double mone = -1.0, one = 1.0;
  const int wj = width(n, nbk, j);
  for (int c = c0; c < c1; c++) {
    const int r = c * nbk, m = n - r;
    const double *Lc = A + (size_t)j * nbk * n + r;
    double *C = A + (size_t)r * n + r;
    BC_CB(cublasDgemmStridedBatched(cb, CUBLAS_OP_N, CUBLAS_OP_T, m, width(n, nbk, c), wj, &mone, Lc, n,
                                    stride, Lc, n, stride, &one, C, n, stride, nb));
  }
}

__global__ void k_bigchol_eye(double *X, int w, long long stride, int nb) {
  const long long ww = (long long)w * w;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < ww * nb;
       t += (long long)gridDim.x * blockDim.x) {
    const long long e = t % ww;
    X[(t / ww) * stride + e] = (e % w == e / w) ? 1.0 : 0.0;
  }
}

// dst[b][c][r] = src[b][c][r] for r < m, c < w (column-major, leading dimension ld for both)
__global__ void k_bigchol_put(const double *src, long long sstride, double *dst, long long dstride,
                              int ld, int m, int w, int nb) {
  const long long mw = (long long)m * w;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < mw * nb;
       t += (long long)gridDim.x * blockDim.x) {
    const long long b = t / mw, e = t - b * mw;
    const long long off = (e / m) * ld + e % m;
    dst[b * dstride + off] = src[b * sstride + off];
  }
}

}  // namespace

BigChol *db_bigchol_create(int n, int nbk, bool inv_panel, bool lookahead) {
  lib();
  BigChol *bc = new BigChol();
  bc->n = n;
  bc->nbk = nbk;
  bc->np = (n + nbk - 1) / nbk;
  bc->maxb = 0;
  bc->A0 = nullptr;
  bc->stride = 0;
  bc->ptr = nullptr;
  bc->pinfo = nullptr;
  bc->inv_panel = inv_panel;
  bc->lookahead = lookahead;
  bc->X = bc->W = nullptr;
  bc->Xptr = nullptr;
  return bc;
}

void db_bigchol_bind_batch(BigChol *bc, double *A0, long long stride, int maxb) {
  if (bc->A0 == A0 && bc->stride == stride && bc->maxb >= maxb) return;
  const int n = bc->n, nbk = bc->nbk, np = bc->np;
  std::vector<double *> h((size_t)2 * np * maxb);
  for (int j = 0; j < np; j++) {
    const int r = j * nbk;
    for (int b = 0; b < maxb; b++) {
      double *Ajj = A0 + stride * b + (size_t)r * n + r;
      h[(size_t)(2 * j) * maxb + b] = Ajj;
      h[(size_t)(2 * j + 1) * maxb + b] = Ajj + width(n, nbk, j);
    }
  }
  if (bc->ptr) db_free(bc->ptr);
  if (bc->pinfo) db_free(bc->pinfo);
  bc->ptr = (double **)db_malloc(sizeof(double *) * h.size());
  bc->pinfo = (int *)db_malloc(sizeof(int) * (size_t)np * maxb);
  DB_CHECK(cudaMemcpy(bc->ptr, h.data(), sizeof(double *) * h.size(), cudaMemcpyHostToDevice));
  if (bc->inv_panel) {
    if (bc->X) { db_free(bc->X); db_free(bc->W); db_free(bc->Xptr); }
    bc->X = (double *)db_malloc(sizeof(double) * nbk * nbk * maxb);
    bc->W = (double *)db_malloc(sizeof(double) * (size_t)nbk * n * maxb);
    std::vector<double *> xp(maxb);
    for (int b = 0; b < maxb; b++) xp[b] = bc->X + (size_t)nbk * nbk * b;
    bc->Xptr = (double **)db_malloc(sizeof(double *) * maxb);
    DB_CHECK(cudaMemcpy(bc->Xptr, xp.data(), sizeof(double *) * maxb, cudaMemcpyHostToDevice));
  }
  bc->A0 = A0;
  bc->stride = stride;
  bc->maxb = maxb;
}

void db_bigchol_destroy(BigChol *bc) {
  if (!bc) return;
  if (bc->ptr) db_free(bc->ptr);
  if (bc->pinfo) db_free(bc->pinfo);
  if (bc->X) { db_free(bc->X); db_free(bc->W); db_free(bc->Xptr); }
  delete bc;
}

// diagonal blocks of panel j and the solve of the block columns below them, on stream st with the
// handles bound to it
static void panel(BigChol *bc, int nb, int j, cublasHandle_t cb, cusolverDnHandle_t cs, cudaStream_t st) {
  const int n = bc->n, nbk = bc->nbk, mb = bc->maxb;
  const int wj = width(n, nbk, j), m = n - j * nbk - wj;
  const double one = 1.0;
  BC_CS(cusolverDnDpotrfBatched(cs, CUBLAS_FILL_MODE_LOWER, wj, bc->ptr + (size_t)2 * j * mb, n,
                                bc->pinfo + (size_t)j * mb, nb));
  if (m > 0 && bc->inv_panel) {
    // X = L_jj^-1 (a small triangular solve on the identity), then L_ij = A_ij X^T by one DGEMM into W
    // and W back into place
    const double zero = 0.0;
    const long long xs = (long long)nbk * nbk, ws = (long long)nbk * n;
    double *Aij = bc->A0 + (size_t)j * nbk * n + j * nbk + wj;
    k_bigchol_eye<<<2 * db_sm_count(), 256, 0, st>>>(bc->X, wj, xs, nb);
    BC_CB(cublasDtrsmBatched(cb, CUBLAS_SIDE_LEFT, CUBLAS_FILL_MODE_LOWER, CUBLAS_OP_N,
                             CUBLAS_DIAG_NON_UNIT, wj, wj, &one, bc->ptr + (size_t)2 * j * mb, n,
                             bc->Xptr, wj, nb));
    BC_CB(cublasDgemmStridedBatched(cb, CUBLAS_OP_N, CUBLAS_OP_T, m, wj, wj, &one, Aij, n, bc->stride,
                                    bc->X, wj, xs, &zero, bc->W, n, ws, nb));
    k_bigchol_put<<<4 * db_sm_count(), 256, 0, st>>>(bc->W, ws, Aij, bc->stride, n, m, wj, nb);
  } else if (m > 0) {
    BC_CB(cublasDtrsmBatched(cb, CUBLAS_SIDE_RIGHT, CUBLAS_FILL_MODE_LOWER, CUBLAS_OP_T,
                             CUBLAS_DIAG_NON_UNIT, m, wj, &one, bc->ptr + (size_t)2 * j * mb, n,
                             bc->ptr + (size_t)(2 * j + 1) * mb, n, nb));
  }
}

// the nb systems bound by db_bigchol_bind_batch (nb <= maxb) in place; info[b * info_step] as dpotrf.
// phase_ms (tuning hook, else null; without look-ahead only): device time of the diagonal factors and
// panel solves, and of the trailing updates, added to [0..1]
static void factor_batch(BigChol *bc, int nb, int *info, int info_step, cudaStream_t st,
                         double *phase_ms) {
  Lib &L = lib();
  const int n = bc->n, nbk = bc->nbk, np = bc->np, mb = bc->maxb;
  BC_CB(cublasSetStream(L.cb[0], st));
  BC_CS(cusolverDnSetStream(L.cs[0], st));
  if (bc->lookahead) {
    panel(bc, nb, 0, L.cb[0], L.cs[0], st);
    for (int j = 0; j + 1 < np; j++) {
      // block column j+1 first, then its panel on the side stream while the rest of the update runs
      trailing(L.cb[0], bc->A0, bc->stride, nb, n, nbk, j, j + 1, j + 2);
      DB_CHECK(cudaEventRecord(L.ev_main, st));
      DB_CHECK(cudaStreamWaitEvent(L.side, L.ev_main, 0));
      panel(bc, nb, j + 1, L.cb[1], L.cs[1], L.side);
      DB_CHECK(cudaEventRecord(L.ev_side, L.side));
      trailing(L.cb[0], bc->A0, bc->stride, nb, n, nbk, j, j + 2, np);
      DB_CHECK(cudaStreamWaitEvent(st, L.ev_side, 0));
    }
  } else {
    cudaEvent_t ev[3];
    if (phase_ms)
      for (int i = 0; i < 3; i++) DB_CHECK(cudaEventCreate(&ev[i]));
    for (int j = 0; j < np; j++) {
      if (phase_ms) DB_CHECK(cudaEventRecord(ev[0], st));
      panel(bc, nb, j, L.cb[0], L.cs[0], st);
      if (phase_ms) DB_CHECK(cudaEventRecord(ev[1], st));
      trailing(L.cb[0], bc->A0, bc->stride, nb, n, nbk, j, j + 1, np);
      if (phase_ms) {
        DB_CHECK(cudaEventRecord(ev[2], st));
        DB_CHECK(cudaEventSynchronize(ev[2]));
        for (int i = 0; i < 2; i++) {
          float ms = 0.f;
          DB_CHECK(cudaEventElapsedTime(&ms, ev[i], ev[i + 1]));
          phase_ms[i] += ms;
        }
      }
    }
    if (phase_ms)
      for (int i = 0; i < 3; i++) cudaEventDestroy(ev[i]);
  }
  k_bigchol_info<<<(nb + 127) / 128, 128, 0, st>>>(bc->pinfo, np, nbk, mb, nb, info, info_step);
  db_count_launch((bc->inv_panel ? 5 : 2) * np + np * (np - 1) / 2 + 1);
}

void db_bigchol_factor_batch(BigChol *bc, int nb, int *info, int info_step, cudaStream_t st) {
  factor_batch(bc, nb, info, info_step, st, nullptr);
}

// ------------------------------------------------------------------------------------------------
// test and tuning hooks
// ------------------------------------------------------------------------------------------------
namespace {
// a well-conditioned SPD matrix per system: A_ij = 1 / (1 + |i - j| + b), A_ii += n
__global__ void k_bigchol_fill(double *A, int n, long long stride, int nb) {
  const long long nn = (long long)n * n;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < nn * nb;
       t += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(t / nn);
    const long long e = t - (long long)b * nn;
    const int i = (int)(e % n), jj = (int)(e / n);
    double v = 1.0 / (1.0 + fabs((double)(i - jj)) + b);
    if (i == jj) v += n;
    A[(size_t)b * stride + e] = v;
  }
}
}  // namespace

extern "C" {
// The blocked batch factorisation of nb systems of order n > 512 from host buffers (column-major,
// ld = n, system b at A + b n^2), factor back into A, info [nb] as dpotrf.  Returns -1 for n <= 512
// (the cluster solvers' sizes).
int dirac_b200_big_factor(int n, int nb, double *A, int *info) {
  if (n <= 512 || nb < 1) return -1;
  const size_t nn = (size_t)n * n;
  double *dA = (double *)db_malloc(sizeof(double) * nn * nb);
  int *dinfo = (int *)db_malloc(sizeof(int) * nb);
  DB_CHECK(cudaMemcpy(dA, A, sizeof(double) * nn * nb, cudaMemcpyHostToDevice));
  cudaStream_t st;
  DB_CHECK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  BigChol *bc = db_bigchol_create(n, BC_BLOCK, BC_INV_PANEL, BC_LOOKAHEAD);
  db_bigchol_bind_batch(bc, dA, (long long)nn, nb);
  db_bigchol_factor_batch(bc, nb, dinfo, 1, st);
  DB_CHECK(cudaStreamSynchronize(st));
  DB_CHECK(cudaMemcpy(A, dA, sizeof(double) * nn * nb, cudaMemcpyDeviceToHost));
  DB_CHECK(cudaMemcpy(info, dinfo, sizeof(int) * nb, cudaMemcpyDeviceToHost));
  db_bigchol_destroy(bc);
  cudaStreamDestroy(st);
  db_free(dA);
  db_free(dinfo);
  DB_CHECK(cudaGetLastError());
  return 0;
}

// Device time of factorising `batch` SPD systems of order n, mean over `reps` (each on freshly
// written matrices, the writes not timed), in *us_out.  variant 0: cusolverDnDpotrf one system at a
// time; 1: cusolverDnDpotrf on 4 streams side by side (the sweep's batch before the blocked one);
// 2-4: the blocked batch with panels of 256 columns: panel solves by a tall trsm (2), by the inverse
// of the diagonal block (3), and that with look-ahead (4: what the LM runs).  For 2 and 3 us_out[1..2]
// get the time of the panels (diagonal factors and solves) and of the trailing updates, from one more
// round timed phase by phase.
// Returns the number of systems with a non-zero status (0 expected), -1 for a bad argument.
int dirac_b200_bench_big_factor(int n, int batch, int reps, int variant, double *us_out) {
  if (n <= 512 || batch < 1 || reps < 1 || variant < 0 || variant > 4) return -1;
  const size_t nn = (size_t)n * n;
  double *dA = (double *)db_malloc(sizeof(double) * nn * batch);
  int *dinfo = (int *)db_malloc(sizeof(int) * batch);
  cudaStream_t st;
  DB_CHECK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  enum { NS = 4 };
  cudaStream_t fs[NS];
  cusolverDnHandle_t fh[NS];
  cudaEvent_t fev[NS], e0, e1;
  double *fwork[NS];
  int lw = 0;
  {
    cusolverDnHandle_t h;
    BC_CS(cusolverDnCreate(&h));
    BC_CS(cusolverDnDpotrf_bufferSize(h, CUBLAS_FILL_MODE_LOWER, n, dA, n, &lw));
    cusolverDnDestroy(h);
  }
  for (int i = 0; i < NS; i++) {
    DB_CHECK(cudaStreamCreateWithFlags(&fs[i], cudaStreamNonBlocking));
    BC_CS(cusolverDnCreate(&fh[i]));
    BC_CS(cusolverDnSetStream(fh[i], fs[i]));
    DB_CHECK(cudaEventCreateWithFlags(&fev[i], cudaEventDisableTiming));
    fwork[i] = (double *)db_malloc(sizeof(double) * (lw > 1 ? lw : 1));
  }
  DB_CHECK(cudaEventCreate(&e0));
  DB_CHECK(cudaEventCreate(&e1));
  BigChol *bc = db_bigchol_create(n, BC_BLOCK, variant >= 3, variant == 4);
  db_bigchol_bind_batch(bc, dA, (long long)nn, batch);
  double total_ms = 0.0;
  int bad = 0;
  std::vector<int> h(batch);
  for (int r = 0; r < reps + 1; r++) {  // the first round warms up
    k_bigchol_fill<<<4 * db_sm_count(), 256, 0, st>>>(dA, n, (long long)nn, batch);
    DB_CHECK(cudaEventRecord(e0, st));
    if (variant == 0 || variant == 1) {
      const int ns = variant == 0 ? 1 : NS;
      for (int i = 0; i < ns; i++) DB_CHECK(cudaStreamWaitEvent(fs[i], e0, 0));
      for (int b = 0; b < batch; b++)
        BC_CS(cusolverDnDpotrf(fh[b % ns], CUBLAS_FILL_MODE_LOWER, n, dA + nn * b, n, fwork[b % ns],
                               lw, dinfo + b));
      for (int i = 0; i < ns; i++) {
        DB_CHECK(cudaEventRecord(fev[i], fs[i]));
        DB_CHECK(cudaStreamWaitEvent(st, fev[i], 0));
      }
    } else {
      db_bigchol_factor_batch(bc, batch, dinfo, 1, st);
    }
    DB_CHECK(cudaEventRecord(e1, st));
    DB_CHECK(cudaEventSynchronize(e1));
    float ms = 0.f;
    DB_CHECK(cudaEventElapsedTime(&ms, e0, e1));
    if (r > 0) total_ms += ms;
    DB_CHECK(cudaMemcpy(h.data(), dinfo, sizeof(int) * batch, cudaMemcpyDeviceToHost));
    for (int b = 0; b < batch; b++) bad += h[b] != 0;
  }
  us_out[0] = 1e3 * total_ms / reps;
  if (variant == 2 || variant == 3) {
    double ph[2] = {0.0, 0.0};
    k_bigchol_fill<<<4 * db_sm_count(), 256, 0, st>>>(dA, n, (long long)nn, batch);
    factor_batch(bc, batch, dinfo, 1, st, ph);
    DB_CHECK(cudaStreamSynchronize(st));
    for (int i = 0; i < 2; i++) us_out[1 + i] = 1e3 * ph[i];
  }
  db_bigchol_destroy(bc);
  for (int i = 0; i < NS; i++) {
    cusolverDnDestroy(fh[i]);
    cudaStreamDestroy(fs[i]);
    cudaEventDestroy(fev[i]);
    db_free(fwork[i]);
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  cudaStreamDestroy(st);
  db_free(dA);
  db_free(dinfo);
  DB_CHECK(cudaGetLastError());
  return bad;
}
}  // extern "C"
