// Internal declarations shared by the sm_90a kernels and the host-side solver code.
// Nothing here is part of the public C-ABI (see include/dirac_b200.h).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#define DB_CHECK(call)                                                                          \
  do {                                                                                          \
    cudaError_t err__ = (call);                                                                 \
    if (err__ != cudaSuccess) {                                                                 \
      fprintf(stderr, "dirac_b200: CUDA error %s at %s:%d: %s\n", cudaGetErrorName(err__),      \
              __FILE__, __LINE__, cudaGetErrorString(err__));                                   \
      exit(1); /* reference convention: message on stderr + exit(1), lmfit.c:831-836 */         \
    }                                                                                           \
  } while (0)

// ------------------------------------------------------------------------------------------------
// HBM layout.
//   rows           r = t*Nbase + b, b = canonical baseline index of (p,q) (baseline_utils.c:445-461)
//   visibilities   planar: vis[c*R + r] is the complex XX,XY,YX,YY (c=0..3) of row r as double2
//   coherencies    planar per cluster: coh[(k*4 + c)*R + r]
//   flags          one byte per row (0 ok; !=0 -> model is zero for this row, lmfit.c:78-81)
//   Jones          pp[] exactly as the C API passes it: [chunk-cluster][station][8] doubles
// A warp streams 32 consecutive q of one p: 512 contiguous bytes per component per timeslot.
// ------------------------------------------------------------------------------------------------

// Tile of baselines handled by one CTA: p in [8*pb, 8*pb+8), q in [32*qb, 32*qb+32), q > p.
#define TILE_P 8
#define TILE_Q 32
#define TILE_THREADS (TILE_P * TILE_Q)

struct TileDesc {
  short pb, qb;
};

struct ClusterDesc {
  int nchunk;      // hybrid time chunks of this cluster (clus_source_t.nchunk)
  int chunk0;      // index of the first chunk of this cluster in DevProblem::chunk_poff
};

struct DevProblem {
  int N, Nbase, tilesz, M, Mt;
  long long R;             // Nbase*tilesz rows
  long long npar;          // length of the Jones vector pp (8*N*Mt, or the global length of a shard)
  int device;
  // resident data
  double2 *coh;            // [M][4][R]
  double2 *x;              // [4][R] data (as given by the caller)
  unsigned char *flag;     // [R]
  double *pp;              // [8*N*Mt] current Jones (device copy)
  ClusterDesc *clus;       // [M]
  int *chunk_poff;         // [Mt] offsets of each (cluster,chunk) block in pp (carr[k].p[ck])
  TileDesc *tiles;         // [ntile]
  int ntile;
  short2 *blpq;            // [Nbase] (p,q) of canonical baseline b (linear-mapped kernels)
  // host mirrors
  ClusterDesc *h_clus;
  int *h_chunk_poff;
  // scratch
  double *scal;            // small device scalar area (cost accumulators ...)
  double *h_scal;          // pinned mirror
  unsigned int *counters;  // last-block counters
  cudaStream_t stream;
};

// canonical baseline index of (p,q), p<q
__host__ __device__ __forceinline__ long long baseline_index(int p, int q, int N) {
  return (long long)p * (N - 1) - (long long)p * (p - 1) / 2 + (q - p - 1);
}

// ------------------------------------------------------------------------------------------------
// 2x2 complex algebra on double2 (x = re, y = im), row-major [00,01,10,11]
// ------------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ double2 cmul(double2 a, double2 b) {
  return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}
// a * conj(b)
__host__ __device__ __forceinline__ double2 cmulc(double2 a, double2 b) {
  return make_double2(a.x * b.x + a.y * b.y, a.y * b.x - a.x * b.y);
}
// conj(a) * b
__host__ __device__ __forceinline__ double2 cmulcl(double2 a, double2 b) {
  return make_double2(a.x * b.x + a.y * b.y, a.x * b.y - a.y * b.x);
}
__host__ __device__ __forceinline__ double2 cadd(double2 a, double2 b) {
  return make_double2(a.x + b.x, a.y + b.y);
}
__host__ __device__ __forceinline__ double2 csub(double2 a, double2 b) {
  return make_double2(a.x - b.x, a.y - b.y);
}
__host__ __device__ __forceinline__ void cfma(double2 &acc, double2 a, double2 b) {  // acc += a*b
  acc.x = fma(a.x, b.x, acc.x);
  acc.x = fma(-a.y, b.y, acc.x);
  acc.y = fma(a.x, b.y, acc.y);
  acc.y = fma(a.y, b.x, acc.y);
}
__host__ __device__ __forceinline__ void cfmac(double2 &acc, double2 a, double2 b) {  // acc += a*conj(b)
  acc.x = fma(a.x, b.x, acc.x);
  acc.x = fma(a.y, b.y, acc.x);
  acc.y = fma(a.y, b.x, acc.y);
  acc.y = fma(-a.x, b.y, acc.y);
}
__host__ __device__ __forceinline__ void cfmacl(double2 &acc, double2 a, double2 b) {  // acc += conj(a)*b
  acc.x = fma(a.x, b.x, acc.x);
  acc.x = fma(a.y, b.y, acc.x);
  acc.y = fma(a.x, b.y, acc.y);
  acc.y = fma(-a.y, b.x, acc.y);
}

// The 2x2 products below are written as explicit FMA chains: 8 fp64 instructions per complex
// output (2 DMUL + 6 DFMA, or 8 DFMA when accumulating) instead of the 10-12 that separate complex
// multiplies and adds compile to.  The fp64 pipe (64 lanes/clk/SM) is the second bound of every
// streaming kernel here, right behind HBM.
// a0*b0 + a1*b1
__host__ __device__ __forceinline__ double2 cdot2(double2 a0, double2 b0, double2 a1, double2 b1) {
  double re = a0.x * b0.x;
  re = fma(-a0.y, b0.y, re);
  re = fma(a1.x, b1.x, re);
  re = fma(-a1.y, b1.y, re);
  double im = a0.x * b0.y;
  im = fma(a0.y, b0.x, im);
  im = fma(a1.x, b1.y, im);
  im = fma(a1.y, b1.x, im);
  return make_double2(re, im);
}
// a0*conj(b0) + a1*conj(b1)
__host__ __device__ __forceinline__ double2 cdot2c(double2 a0, double2 b0, double2 a1, double2 b1) {
  double re = a0.x * b0.x;
  re = fma(a0.y, b0.y, re);
  re = fma(a1.x, b1.x, re);
  re = fma(a1.y, b1.y, re);
  double im = a0.y * b0.x;
  im = fma(-a0.x, b0.y, im);
  im = fma(a1.y, b1.x, im);
  im = fma(-a1.x, b1.y, im);
  return make_double2(re, im);
}
// acc += a0*conj(b0) + a1*conj(b1)
__host__ __device__ __forceinline__ void cdot2c_acc(double2 &acc, double2 a0, double2 b0, double2 a1,
                                           double2 b1) {
  acc.x = fma(a0.x, b0.x, acc.x);
  acc.x = fma(a0.y, b0.y, acc.x);
  acc.x = fma(a1.x, b1.x, acc.x);
  acc.x = fma(a1.y, b1.y, acc.x);
  acc.y = fma(a0.y, b0.x, acc.y);
  acc.y = fma(-a0.x, b0.y, acc.y);
  acc.y = fma(a1.y, b1.x, acc.y);
  acc.y = fma(-a1.x, b1.y, acc.y);
}
// C = A*B          (lmfit.c:37-42 "amb")
__host__ __device__ __forceinline__ void mat_ab(const double2 *a, const double2 *b, double2 *c) {
  c[0] = cdot2(a[0], b[0], a[1], b[2]);
  c[1] = cdot2(a[0], b[1], a[1], b[3]);
  c[2] = cdot2(a[2], b[0], a[3], b[2]);
  c[3] = cdot2(a[2], b[1], a[3], b[3]);
}
// C = A*B^H        (lmfit.c:50-58 "ambt")
__host__ __device__ __forceinline__ void mat_abh(const double2 *a, const double2 *b, double2 *c) {
  c[0] = cdot2c(a[0], b[0], a[1], b[1]);
  c[1] = cdot2c(a[0], b[2], a[1], b[3]);
  c[2] = cdot2c(a[2], b[0], a[3], b[1]);
  c[3] = cdot2c(a[2], b[2], a[3], b[3]);
}
// C += A*B^H
__host__ __device__ __forceinline__ void mat_abh_acc(const double2 *a, const double2 *b, double2 *c) {
  cdot2c_acc(c[0], a[0], b[0], a[1], b[1]);
  cdot2c_acc(c[1], a[0], b[2], a[1], b[3]);
  cdot2c_acc(c[2], a[2], b[0], a[3], b[1]);
  cdot2c_acc(c[3], a[2], b[2], a[3], b[3]);
}
// C = A^H*B
__host__ __device__ __forceinline__ void mat_ahb(const double2 *a, const double2 *b, double2 *c) {
  c[0] = cadd(cmulcl(a[0], b[0]), cmulcl(a[2], b[2]));
  c[1] = cadd(cmulcl(a[0], b[1]), cmulcl(a[2], b[3]));
  c[2] = cadd(cmulcl(a[1], b[0]), cmulcl(a[3], b[2]));
  c[3] = cadd(cmulcl(a[1], b[1]), cmulcl(a[3], b[3]));
}

// 128-bit streaming loads / stores of planar visibilities: read once, do not pollute L1
__device__ __forceinline__ double2 ld_stream(const double2 *p) {
  double2 v;
  asm volatile("ld.global.nc.L1::no_allocate.v2.f64 {%0,%1}, [%2];" : "=d"(v.x), "=d"(v.y) : "l"(p));
  return v;
}
__device__ __forceinline__ void st_stream(double2 *p, double2 v) {
  asm volatile("st.global.L1::no_allocate.v2.f64 [%0], {%1,%2};" ::"l"(p), "d"(v.x), "d"(v.y)
               : "memory");
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Jones matrix of one station from a parameter block (8 doubles, 64-byte aligned)
__device__ __forceinline__ void load_jones(const double *pblk, int sta, double2 *J) {
  const double2 *s = reinterpret_cast<const double2 *>(pblk + 8 * (long long)sta);
  J[0] = __ldg(s + 0);
  J[1] = __ldg(s + 1);
  J[2] = __ldg(s + 2);
  J[3] = __ldg(s + 3);
}

// chunk of row r for a cluster with nchunk hybrid chunks: px = r / ceil(R/nchunk)  (lmfit.c:86,655)
__device__ __forceinline__ int row_chunk(long long r, long long R, int nchunk) {
  return nchunk == 1 ? 0 : (int)(r / ((R + nchunk - 1) / nchunk));
}

// ------------------------------------------------------------------------------------------------
// kernel argument blocks
// ------------------------------------------------------------------------------------------------
struct GradArgs {
  const double2 *coh;        // [M][4][R]
  const double2 *res;        // [4][R] residual e = data - model (written by k_stream_all<0>)
  const unsigned char *flag;
  const double *pp;
  const ClusterDesc *clus;
  const int *chunk_poff;
  const TileDesc *tiles;
  double *g;                 // [8*N*Mt] gradient, zeroed by the caller
  long long R;
  int N, Nbase, tilesz, M;
  int robust;                // 0: R = e ; 1: R_i = e_i/(nu + e_i^2)
  double nu;
  double scale;              // +2 (Gaussian convention of robust_lbfgs.c:554) or -2 (robust, :299)
  // row window of k_grad_tma_window: time blocks tb0, tb0+1, ... (gridDim.y of them), and only the
  // rows [w_lo, w_hi) of the interval contribute (the full-interval kernel reads neither)
  int tb0;
  long long w_lo, w_hi;
};

struct ClusterPassArgs {
  const double2 *coh_k;      // [4][R] coherencies of this cluster
  const double2 *in;         // [4][R] input vector (residual r, or hidden data d)
  const unsigned char *flag;
  const double *pblk;        // 8N Jones of this (cluster,chunk) at which the model is evaluated
  const TileDesc *tiles;
  double2 *out;              // [4][R]
  double *jte;               // [8N] J^T e accumulator (zeroed by the caller), may be null
  double *partials;
  double *cost;
  unsigned int *counter;
  long long R;
  int N, Nbase;
  int t_begin, t_end, tslice;  // timeslots per CTA slice
  int mode;  // 4: GIVEN e = in (no model subtracted): J^T (wt^2 . in) of a caller-formed residual
             // 0: INIT  d = in + m -> out ; e = d - m
             // 1: TRIAL e = in - m -> out
             // 2: ADD   out = in + m          (no cost / jte)
             // 3: SUB   out = in - m          (no cost / jte)
  int write_out;
  double beta;               // SAGE hidden-data weight: INIT d = beta*in + m ; SUB out = d - m + (1-beta)*r_old
  const double *pblk_old;    // mode 3 with beta != 1: the Jones the hidden data was
                             // formed with; the old residual is recovered as (d - f(p_old))/beta, so
                             // out = d - f(p) + (1-beta)/beta (d - f(p_old)) costs no extra traffic
  int form_hidden;           // modes 1 and 3: `in` is the residual r and the hidden data is formed per
                             // row as d = beta r + f(pblk_old), never stored (linear-mapped variant only)
  const short2 *blpq;        // [Nbase] (p,q) of baseline b (linear-mapped variant)
  double *jte_part;          // [groups][slices][8N] per-CTA station sums (linear-mapped variant)
  unsigned int *gcounter;    // [groups] arrival counters of the time slices of a baseline group
  const double2 *wt;         // [4][R] sqrt-weights (re,im) of the robust LM, or null.  With
                             // weights: cost = ||wt.e||^2 and J^T e -> J^T (wt^2 . e); the vector
                             // written for mode 1 stays the UNWEIGHTED e
};

// weighted normal matrix of the robust LM (J <- wt.J, robustlm.c:2298-2307), one polarisation
// product c = (i,j) of the visibility per pass of the CTA over its rows
struct WeightedJtjArgs {
  const double2 *coh_k;      // [4][R]
  const double2 *wt;         // [4][R] sqrt-weights
  const unsigned char *flag;
  const double *pblk;
  const TileDesc *tiles;
  double *JTJ;               // [8N][8N], zeroed by the caller; off-diagonal blocks accumulate here
  double *HP, *HQ;           // [N][2][10] station sums of the p-role / q-role diagonal terms, zeroed
  long long R;
  int N, Nbase;
  int t_begin, t_end, tslice;
};

// all-cluster TMA-pipelined passes (kernels_tma.cu)
struct StreamAllArgs {
  const double2 *coh;        // [M][4][R]
  const double2 *x;          // [4][R]
  const unsigned char *flag;
  const double *pp;          // Jones (device)
  const double *pk;          // search direction (MODE 1)
  const ClusterDesc *clus;
  const int *chunk_poff;
  const short2 *blpq;
  double2 *out;              // MODE 0
  double2 *E0, *E1, *E2;     // MODE 1
  double *poly_part;         // MODE 1, partial == 0: per-CTA sums of the line quartic, [5][grid]
                             // (null: not formed)
  double *partials, *cost;
  unsigned int *counter;
  long long R;
  int N, Nbase, tilesz, M;
  int out_mode, cost_mode;
  double inv_nu;
  int partial;
  long long row0;            // absolute row of the first row the pointers address (time-chunked
                             // launches shift the base pointers; hybrid chunk maps need the row)
  long long w_lo, w_hi;      // MODE 2: rows [w_lo, w_hi) of the launch (relative to the shifted
                             // pointers) are evaluated, the others of its timeslots are skipped
};

struct GramArgs {
  const double2 *coh;        // [M][4][R], cluster of blockIdx.y is k0 + blockIdx.y
  const unsigned char *flag;
  const TileDesc *tiles;
  double *T;                 // [nk][Nbase][16]
  long long R;
  int N, Nbase;
  int k0;
  int t_begin, t_end, t_step;  // timeslots t_begin, t_begin+t_step, ... < t_end
};

// J^T J of one system, or of a batch (matrix y of the batch belongs to local cluster list[y]).
// Baseline b of the station pair p < q is the b-th pair in (p, q) lexicographic order (problem.cu).
struct AssembleArgs {
  const double *T;       // [Nbase][16] Gram tensors; batch: [Mt][Nbase][16], slot tix[list[y]]
  const double *pblk;    // 8N Jones; batch: the Jones vector, cluster block at poff[list[y]]
  const int *list;       // batch: [nb] local cluster indices; null: one system
  const int *tix;        // batch: [M] Gram slot of cluster k (first chunk)
  const int *poff;       // batch: [M] offset of cluster k's (first) block in pblk
  double *JTJ;           // [8N][8N]; batch: matrix y at JTJ + y * stride
  long long stride;
  double *Hst;           // [N][4] station sums (H00, H11, Re H01, Im H01); batch: [nb][N][4]
  const double *mu_dev;  // batch: damping of matrix y; null: mu
  double mu;             // added to the diagonal
  int lower;             // 1: write only the lower triangle (column-major) and the diagonal
  int N, Nbase;
};

// test / tuning options (dirac_b200_set_option): 0 = default
enum { DB_OPT_CP_ROWS = 0, DB_OPT_LINE_DIRECT = 1, DB_OPT_OS_CONSISTENT = 2,
       DB_OPT_RTR_NU_UNJOINED = 3, DB_OPT_ADMM_LM = 4, DB_OPT_SWEEP_RESIDUAL = 5,
       DB_OPT_COUNT = 8 };
int db_opt(int id);
int db_sm_count();  // SMs of the current device
// slices of the time axis the linear-mapped gradient pass may use (sizes LMWork::jte_part)
static inline int db_cp_max_slices(int Nbase, int tilesz) {
  const int nbg = (Nbase + 255) / 256;
  int nsl = (db_sm_count() + nbg - 1) / nbg;
  if ((tilesz + 31) / 32 > nsl) nsl = (tilesz + 31) / 32;  // slices hold at most 32 rows
  return nsl;
}

extern "C" {
void db_launch_coh_to_planar(const double2 *src, double2 *dst, long long r0, int nr, int M,
                             long long R, cudaStream_t st);
void db_launch_coh_from_planar(const double2 *src, double2 *dst, long long r0, int nr, int M,
                               long long R, cudaStream_t st);
void db_launch_vis_to_planar(const double2 *src, double2 *dst, long long R, cudaStream_t st);
void db_launch_vis_from_planar(const double2 *src, double2 *dst, long long R, cudaStream_t st);
void db_launch_grad_tma(const GradArgs *a, int ntile, cudaStream_t st);
// the gradient of rows [r_lo, r_hi) only: the time blocks that overlap them
void db_launch_grad_window_tma(const GradArgs *a, int ntile, long long r_lo, long long r_hi,
                               cudaStream_t st);
// every channel of a band: a holds the first channel's coh / res, the grid's z axis the channels
void db_launch_grad_band_tma(const GradArgs *a, int ntile, int nchan, cudaStream_t st);
int db_cluster_pass_nblocks(int ntile, int nt, int tslice);
// the kernel db_launch_cluster_pass launched (DB_CP_NONE: db_cluster_pass had no timeslot to visit)
enum { DB_CP_LIN = 0, DB_CP_LIN_GRAD = 1, DB_CP_SPLIT = 2, DB_CP_TILE = 3, DB_CP_NONE = 4 };
int db_launch_cluster_pass(const ClusterPassArgs *a, int ntile, cudaStream_t st);
// whether plain (unweighted) passes of this array take k_cluster_pass_lin, the one variant that
// forms the hidden data itself (ClusterPassArgs::form_hidden)
int db_cluster_pass_forms_hidden(int N, int Nbase);
void db_launch_coh_gram(const GramArgs *a, int ntile, int nk, cudaStream_t st);
void db_launch_station_sums(const AssembleArgs *a, int nb, cudaStream_t st);
void db_launch_assemble_tiles(const AssembleArgs *a, int nb, cudaStream_t st);
void db_launch_batch_mu0(const double *Hst, double *mu, int N, double tau, int nb, cudaStream_t st);
void db_launch_copy_add_diag(const double *A0, double *A, int n, double mu, cudaStream_t st);
// kernels_chol.cu: (A + mu I) x = b on one thread-block cluster
int db_chol_max_n();
int db_chol_available();
size_t db_chol_ws_doubles(int n);
int db_tri_available(int n);
void db_chol_set_step(const double *pcur, double *pnew, double *sc, double *zero);
void db_launch_tri_solve(const double *L, int n, const double *b, double *x, cudaStream_t st);
void db_launch_tri_solve_ld(const double *L, int ld, int n, const double *b, double *x,
                            cudaStream_t st);
void db_launch_chol_factor_batched(const double *A, int n, const double *mu, double *ws,
                                   long long ws_stride, int *info, int nb, cudaStream_t st);
void db_launch_chol_solve(const double *A, int n, double mu, const double *b, double *x, double *ws,
                          int *info, cudaStream_t st);
int db_bigtri_available(int n);
size_t db_bigtri_ws_doubles(int n);
void db_launch_bigtri_solve(const double *L, int ld, int n, const double *b, double *x, double *ws,
                            int *status, cudaStream_t st);
int db_stream_all_nblocks(int Nbase, int tilesz);
void db_launch_predict_tma(const StreamAllArgs *a, cudaStream_t st);
void db_launch_cost_window_tma(const StreamAllArgs *a, cudaStream_t st);
// kernels_band.cu: MODE 0 of k_stream_all over the nchan channels of a band in one launch; a holds the
// first channel's coh / x / out, the others follow at strides M 4 R and 4 R.  The cost's partials
// need db_band_nblocks entries.
int db_band_nblocks(int Nbase, int tilesz, int nchan);
void db_launch_band_tma(const StreamAllArgs *a, int nchan, cudaStream_t st);
void db_launch_band_tma(const StreamAllArgs *a, int nchan, cudaStream_t st);
// returns the grid (the columns of a->poly_part it wrote, when set)
unsigned db_launch_line_setup_tma(const StreamAllArgs *a, cudaStream_t st);
// k_line_poly_finish: the five quartic coefficients from the [5][nparts] per-CTA sums of
// k_stream_all<1>, into out[0..4]
void db_launch_line_poly_finish(const double *part, unsigned nparts, double *partials, double *out,
                                unsigned int *counter, cudaStream_t st);
// (TB, NST, WARPS) of the last k_stream_all<1> launch since the reset (-1 each: none)
void db_line_setup_shape_reset();
void db_line_setup_shape(int *shape);
}
