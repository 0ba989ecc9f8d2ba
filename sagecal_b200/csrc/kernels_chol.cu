// Damped normal-equation solve (A + mu I) x = b for one cluster's 8N x 8N system, as ONE kernel on a
// thread-block cluster (replaces the dpotrf + dpotrs pair of clmfit.c:373-395 / the cuSOLVER calls).
//
// The system is tiny (n = 496 for 62 stations: 41 MFLOP) and strictly latency bound: cuSOLVER spends
// ~200 us in potrf and ~90 us in potrs on it, almost all of it launch gaps and grid-wide dependencies.
// Here a cluster of CL CTAs (16 SMs when the device grants it, else 8) runs a right-looking blocked
// Cholesky with 32 x 32 blocks and synchronises with barrier.cluster (~380 cycles) instead of kernel
// boundaries:
//   - the matrix lives in an L2-resident column-major workspace (ld = 32*nblk, identity padding);
//   - one warp = one 32 x 32 block operation, lane l owns row l of the block in registers;
//   - per panel j:   trsm of the blocks below L_jj  ->  cluster barrier  ->  rank-32 update of the
//     trailing blocks; the warp that updates block (j+1,j+1) factors it in registers right away
//     (32 pivots by warp shuffles), so potf2 never needs a phase of its own  ->  cluster barrier;
//   - the two triangular solves run in CTA 0 once the factor is complete, with the blocks of the
//     next column prefetched into registers while warp 0 walks the 32-step substitution chain.
// info: 0, or (1-based) index of the first non-positive pivot, like dpotrf.
#include <cooperative_groups.h>
#include <cstdio>
#include <cstdlib>

#include "internal.cuh"
#include "tma.cuh"

namespace {

constexpr int CH_WARPS = 8;
constexpr int CH_THREADS = CH_WARPS * 32;
constexpr unsigned FULL = 0xffffffffu;
#ifndef FAST_RSQRT_NEWTON
#define FAST_RSQRT_NEWTON 0  // the cubic step alone lands within a few ulp (tests/test_chol_solver.py)
#endif
constexpr unsigned long long X_PENDING = 0xFFF8DEADBEEF0001ull;

// optional epilogue of both solver kernels: the LM trial point and its scalars (k_lm_step fused in)
struct StepArgs {
  const double *pcur;  // current parameters (nullptr: no epilogue)
  double *pnew;        // pcur + x
  double *sc;          // sc[0] = |x|^2, sc[1] = x . b
  double *zero;        // vector to clear (accumulator of the trial pass), may be null
};

struct CholArgs {
  const double *A;  // n x n symmetric, lower triangle read (column-major, ld = n)
  const double *b;  // right-hand side (n)
  double *x;        // solution (n)
  double *ws;       // workspace: npad*npad factor | npad reciprocal diagonal | nblk*2048 inverses | npad rhs | npad y
  int *info;
  double mu;
  int n, nblk;
  long long *ts;  // optional phase timestamps (globaltimer ns), tuning only
  StepArgs st;
  // batched factorisation (one thread-block cluster per matrix, blockIdx.x / cluster size = matrix):
  // A, ws, info advance by the strides below, mu comes from mu_ptr[matrix], no right-hand side, the
  // kernel returns once the factor stands in the workspace (ld = 32*nblk, identity padding)
  int factor_only;
  const double *mu_ptr;
  long long ws_stride;
};
__device__ __forceinline__ double rhs_at(const CholArgs &p, int r) {
  return (p.b != nullptr && r < p.n) ? p.b[r] : 0.0;
}

// release/acquire at cluster scope orders the workspace stores (L2) before the other CTAs' .cg loads
__device__ __forceinline__ void cluster_barrier() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n"
               "barrier.cluster.wait.acquire.aligned;\n" ::
                   : "memory");
}
__device__ __forceinline__ void stamp(const CholArgs &p, int &i) {
  if (p.ts && threadIdx.x == 0) {
    long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    p.ts[i] = t;
  }
  i++;
}
__device__ __forceinline__ unsigned cluster_rank() {
  unsigned r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ unsigned cluster_size() {
  unsigned r;
  asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
  return r;
}

// lane l <- row l of the 32 x 32 block at `base` (column-major, ld): 32 coalesced 256-byte reads
__device__ __forceinline__ void load_rows(double (&a)[32], const double *base, int ld, int lane) {
#pragma unroll
  for (int c = 0; c < 32; c++) a[c] = __ldcg(base + (size_t)c * ld + lane);
}
__device__ __forceinline__ void store_rows(const double (&a)[32], double *base, int ld, int lane) {
#pragma unroll
  for (int c = 0; c < 32; c++) base[(size_t)c * ld + lane] = a[c];
}
// warp copy of a block into shared memory, column-major with ld 32
__device__ __forceinline__ void stage_block(double *dst, const double *base, int ld, int lane) {
#pragma unroll
  for (int i = 0; i < 16; i++) {
    const int e = i * 32 + lane;  // double2 index: 16 per column
    const int c = e >> 4, r2 = e & 15;
    const double2 v = __ldcg(reinterpret_cast<const double2 *>(base + (size_t)c * ld) + r2);
    reinterpret_cast<double2 *>(dst + c * 32)[r2] = v;
  }
}

// Cholesky of a 32 x 32 block held one row per lane.  returns 0 or the 1-based failing pivot.
// The pivot chain is what bounds the whole factorisation, so two columns are eliminated per step:
// with d0 = a_kk, e = a_k+1,k, d1 = a_k+1,k+1 the second pivot is d1 - e^2/d0 = (d1 d0 - e^2)/d0, whose
// inverse root rsqrt(d1 d0 - e^2) sqrt(d0) does not wait for the first one: both rsqrt run side by
// side.  Columns k, k+1 of L reach the other lanes through shared memory (cols: 32 x 32 scratch, fresh
// columns every step, one __syncwarp per pair); the three pivot entries travel by shuffle.
// branch-free 1/sqrt(d) for normal positive d (anything else yields NaN/Inf, caught by the pivot
// test): hardware seed, one third-order and one second-order correction.  No slow-path branch, so the
// scheduler can overlap it with the trailing updates of the previous pivot pair.
__device__ __forceinline__ double fast_rsqrt(double d) {
  double y;
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(d));
  double e = fma(-d * y, y, 1.0);
  y = fma(y * e, fma(0.375, e, 0.5), y);
  if (FAST_RSQRT_NEWTON) {
    e = fma(-d * y, y, 1.0);
    y = fma(y, 0.5 * e, y);
  }
  return y;
}

__device__ __forceinline__ int potf2_warp(double (&a)[32], double &myrd, double *cols, int lane) {
  int bad = 0;
  // Four columns per step: pivot pair (k, k+1) as described above; columns k+2, k+3 then receive its
  // rank-2 update straight from registers (four shuffles), so the second pivot pair (k+2, k+3) starts
  // without a trip through shared memory; only then are the four finished columns published and the
  // rest of the block updated once (rank 4).  Halves the per-column share of the smem round trip and
  // of the trailing-update issue time on the chain.
#pragma unroll
  for (int k = 0; k < 32; k += 4) {
    // ---- pair A
    const double d0 = __shfl_sync(FULL, a[k], k);
    const double e = __shfl_sync(FULL, a[k], k + 1);
    const double d1 = __shfl_sync(FULL, a[k + 1], k + 1);
    const double num = fma(d1, d0, -e * e);
    if (!bad) {
      if (!(d0 > 0.0)) bad = k + 1;
      else if (!(num > 0.0)) bad = k + 2;
    }
    const double r0 = fast_rsqrt(d0), rn = fast_rsqrt(num);
    const double r1 = rn * (d0 * r0);
    const double l0 = a[k] * r0;
    const double l1 = fma(-l0, e * r0, a[k + 1]) * r1;
    a[k] = l0;
    a[k + 1] = l1;
    if (lane == k) myrd = r0;
    if (lane == k + 1) myrd = r1;
    // ---- rank-2 update of columns k+2, k+3 from registers
    {
      const double l0_2 = __shfl_sync(FULL, l0, k + 2), l1_2 = __shfl_sync(FULL, l1, k + 2);
      const double l0_3 = __shfl_sync(FULL, l0, k + 3), l1_3 = __shfl_sync(FULL, l1, k + 3);
      a[k + 2] = fma(-l1, l1_2, fma(-l0, l0_2, a[k + 2]));
      a[k + 3] = fma(-l1, l1_3, fma(-l0, l0_3, a[k + 3]));
    }
    // ---- pair B
    const double f0 = __shfl_sync(FULL, a[k + 2], k + 2);
    const double g = __shfl_sync(FULL, a[k + 2], k + 3);
    const double f1 = __shfl_sync(FULL, a[k + 3], k + 3);
    const double numb = fma(f1, f0, -g * g);
    if (!bad) {
      if (!(f0 > 0.0)) bad = k + 3;
      else if (!(numb > 0.0)) bad = k + 4;
    }
    const double s0 = fast_rsqrt(f0), sn = fast_rsqrt(numb);
    const double s1 = sn * (f0 * s0);
    const double l2 = a[k + 2] * s0;
    const double l3 = fma(-l2, g * s0, a[k + 3]) * s1;
    a[k + 2] = l2;
    a[k + 3] = l3;
    if (lane == k + 2) myrd = s0;
    if (lane == k + 3) myrd = s1;
    if (k < 28) {
      cols[k * 32 + lane] = l0;
      cols[(k + 1) * 32 + lane] = l1;
      cols[(k + 2) * 32 + lane] = l2;
      cols[(k + 3) * 32 + lane] = l3;
      __syncwarp();
#pragma unroll
      for (int m = k + 4; m < 32; m += 2) {
        const double2 c0 = lds_v2(reinterpret_cast<const double2 *>(cols + k * 32 + m));
        const double2 c1 = lds_v2(reinterpret_cast<const double2 *>(cols + (k + 1) * 32 + m));
        const double2 c2 = lds_v2(reinterpret_cast<const double2 *>(cols + (k + 2) * 32 + m));
        const double2 c3 = lds_v2(reinterpret_cast<const double2 *>(cols + (k + 3) * 32 + m));
        a[m] = fma(-l3, c3.x, fma(-l2, c2.x, fma(-l1, c1.x, fma(-l0, c0.x, a[m]))));
        a[m + 1] = fma(-l3, c3.y, fma(-l2, c2.y, fma(-l1, c1.y, fma(-l0, c0.y, a[m + 1]))));
      }
    }
  }
#pragma unroll
  for (int c = 1; c < 32; c++)
    if (c > lane) a[c] = 0.0;
  return bad;
}

// x <- x L^-T for the staged diagonal block Ls (column-major) with reciprocal diagonal rds
__device__ __forceinline__ void trsm_warp(double (&x)[32], const double *Ls, const double *rds) {
#pragma unroll
  for (int c = 0; c < 32; c++) {
    x[c] *= rds[c];
    const double xc = x[c];
    int m0 = c + 1;
    if (m0 & 1) {  // odd start: one scalar element, then aligned pairs (c is static after unrolling)
      if (m0 < 32) x[m0] = fma(-xc, Ls[c * 32 + m0], x[m0]);
      m0++;
    }
#pragma unroll
    for (int m = m0; m < 32; m += 2) {
      const double2 l = lds_v2(reinterpret_cast<const double2 *>(Ls + c * 32 + m));
      x[m] = fma(-xc, l.x, x[m]);
      x[m + 1] = fma(-xc, l.y, x[m + 1]);
    }
  }
}

// c <- c - a B^T with B staged column-major (B[k][m] at m*32+k)
__device__ __forceinline__ void update_warp(double (&c)[32], const double (&a)[32],
                                            const double *Bs) {
#pragma unroll
  for (int m = 0; m < 32; m++) {
    const double am = -a[m];
#pragma unroll
    for (int k = 0; k < 32; k += 2) {
      const double2 bv = lds_v2(reinterpret_cast<const double2 *>(Bs + m * 32 + k));
      c[k] = fma(am, bv.x, c[k]);
      c[k + 1] = fma(am, bv.y, c[k + 1]);
    }
  }
}

// shared-memory offset (doubles) of the backward-solve control block: behind the per-warp staging
// areas and behind the column tiles of CTA 0 (which owns the most), identical in every CTA
__host__ __device__ inline size_t ctrl_off(int nblk, int cl) {
  size_t t = 0;
  for (int j = 0; j < nblk; j += cl) t += 1024 + (size_t)(nblk - 1 - j) * 1056;
  const size_t stage = (size_t)CH_WARPS * (32 * 32 + 32) + 2048;  // + cooperative diagonal block
  return t > stage ? t : stage;
}

// doubles of tile storage the solve-only kernel needs (max over CTAs and over the two directions)
__host__ __device__ inline size_t tri_tiles(int nblk, int cl) {
  size_t best = 0;
  for (int c = 0; c < cl && c < nblk; c++) {
    size_t f = 0, b = 0;
    for (int j = c; j < nblk; j += cl) {
      f += (size_t)j * 1056;
      b += (size_t)(nblk - 1 - j) * 1056;
    }
    if (f > best) best = f;
    if (b > best) best = b;
  }
  return best;
}

// row `lane` of block (I,K) of A + mu I (identity on the padding)
__device__ __forceinline__ void load_rows_A(double (&a)[32], const CholArgs &p, int I, int K,
                                            int lane) {
  const int r = I * 32 + lane;
  if (I * 32 + 32 <= p.n && K * 32 + 32 <= p.n) {
    // interior block: 32 independent coalesced loads, no guards
    const double *base = p.A + (size_t)(K * 32) * p.n + r;
#pragma unroll
    for (int c = 0; c < 32; c++) a[c] = __ldg(base + (size_t)c * p.n);
    if (I == K) {
#pragma unroll
      for (int c = 0; c < 32; c++)
        if (c == lane) a[c] += p.mu;
    }
    return;
  }
#pragma unroll
  for (int c = 0; c < 32; c++) {
    const int cc = K * 32 + c;
    double v;
    if (r < p.n && cc < p.n) {
      v = __ldg(p.A + (size_t)cc * p.n + r);
      if (r == cc) v += p.mu;
    } else {
      v = (r == cc) ? 1.0 : 0.0;
    }
    a[c] = v;
  }
}

__device__ __forceinline__ double dot32(const double (&a)[32], const double *v) {
  double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
#pragma unroll
  for (int m = 0; m < 32; m += 4) {
    const double2 v0 = lds_v2(reinterpret_cast<const double2 *>(v + m));
    const double2 v1 = lds_v2(reinterpret_cast<const double2 *>(v + m + 2));
    s0 = fma(a[m], v0.x, s0);
    s1 = fma(a[m + 1], v0.y, s1);
    s2 = fma(a[m + 2], v1.x, s2);
    s3 = fma(a[m + 3], v1.y, s3);
  }
  return (s0 + s1) + (s2 + s3);
}

// CTA 0: collect the solution from the arrival slots, store it, and (LM) form the trial point
// p + x with |x|^2 and x.b (clmfit.c:440-449,487-497) — what used to be a kernel of its own.
__device__ __forceinline__ void solution_epilogue(const double *xs, double *x, const double *b, int n,
                                                  const StepArgs &st, double *red) {
  double s0 = 0.0, s1 = 0.0;
  for (int i = threadIdx.x; i < n; i += CH_THREADS) {
    const unsigned addr = smem_u32(xs + i);
    unsigned long long bits;
    do {
      asm volatile("ld.volatile.shared.u64 %0, [%1];" : "=l"(bits) : "r"(addr) : "memory");
    } while (bits == X_PENDING);
    const double xv = __longlong_as_double((long long)bits);
    x[i] = xv;
    if (st.pcur) {
      st.pnew[i] = st.pcur[i] + xv;
      s0 = fma(xv, xv, s0);
      s1 = fma(xv, b[i], s1);
      if (st.zero) st.zero[i] = 0.0;
    }
  }
  if (st.pcur) {
    s0 = warp_sum(s0);
    s1 = warp_sum(s1);
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) {
      red[w] = s0;
      red[CH_WARPS + w] = s1;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      double t0 = 0.0, t1 = 0.0;
      for (int i = 0; i < CH_WARPS; i++) {
        t0 += red[i];
        t1 += red[CH_WARPS + i];
      }
      st.sc[0] = t0;
      st.sc[1] = t1;
    }
  }
}

// y_j = L_jj^-1 b_j by one warp (L_jj staged column-major in Ls): the forward solve of block j
__device__ __forceinline__ double fwd_block(double val, const double *Ls, double myrd, int lane) {
#pragma unroll 4
  for (int c = 0; c < 32; c++) {
    const double yc = __shfl_sync(FULL, val * myrd, c);
    if (lane == c) val = yc;
    if (lane > c) val = fma(-yc, Ls[c * 32 + lane], val);
  }
  return val;
}

__global__ void __launch_bounds__(CH_THREADS, 1) k_chol_solve(CholArgs p) {
  extern __shared__ __align__(16) double sm[];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int crank = (int)cluster_rank(), CL = (int)cluster_size();
  if (p.factor_only) {
    const int mat = (int)(blockIdx.x / CL);
    p.A += (size_t)mat * p.n * p.n;
    p.ws += (size_t)mat * p.ws_stride;
    p.info += 2 * mat;
    p.mu = p.mu_ptr[mat];
    p.b = nullptr;
  }
  const int G = CL * CH_WARPS;     // warps of the cluster
  const int g = w * CL + crank;    // spread consecutive work items over the SMs first
  const int ld = p.nblk * 32, nblk = p.nblk;
  double *ws = p.ws;
  double *wrd = p.ws + (size_t)ld * ld;
  double *winv = wrd + ld;  // per diagonal block 2048 doubles: [1024, 2048) holds L_jj^-T
  double *wb = winv + (size_t)nblk * 2048;  // running right-hand side (forward solve rides along)
  double *wy = wb + ld;                     // y = L^-1 b
  double *Bs = sm + (size_t)w * (32 * 32 + 32);  // per-warp staging block + 32 reciprocals
  double *rds = Bs + 32 * 32;

  int si = 0;
  stamp(p, si);
  if (g == 0 && lane == 0) p.info[0] = p.info[1] = 0;  // [0] factor status, [1] solve status
  if (!p.factor_only) {
    // the solution blocks double as their own arrival flags: a NaN pattern no computation produces
    unsigned long long *xs0 = reinterpret_cast<unsigned long long *>(sm + ctrl_off(nblk, CL));
    for (int i = threadIdx.x; i < ld; i += CH_THREADS) xs0[i] = X_PENDING;
  }

  // Panel j = -1 only factors block (0,0).  Panel 0 reads its blocks from A (+ mu on the diagonal,
  // identity padding), later panels from the workspace, so A is never copied as a whole.
  for (int j = -1; j < nblk - 1; j++) {
    const int nrem = nblk - 1 - j;
    // j = -1: only block (0,0) is factored (by CTA 0, through the same code as every later diagonal
    // block).  (A dry run of the block kernels on the idle CTAs during that time was tried to warm the
    // instruction caches and measured no effect.)
    const bool first = (j < 0);
    const int jj = first ? 0 : j;
    if (!first) {
      // ---- panel: L_Ij = A_Ij L_jj^-T
      const int ntr = nrem;
      for (int t = g; t < ntr; t += G) {
        const int I = j + 1 + t;
        __syncwarp();
        stage_block(Bs, ws + (size_t)(jj * 32) * ld + jj * 32, ld, lane);
        rds[lane] = __ldcg(wrd + jj * 32 + lane);
        double x[32];
        double *blk = ws + (size_t)(jj * 32) * ld + I * 32;
        if (jj == 0) load_rows_A(x, p, I, 0, lane);
        else load_rows(x, blk, ld, lane);
        __syncwarp();
        trsm_warp(x, Bs, rds);
        store_rows(x, blk, ld, lane);
      }
      if (g == G - 1) {
        // the forward solve rides along: y_j = L_jj^-1 b_j on an otherwise idle warp
        __syncwarp();
        stage_block(Bs, ws + (size_t)(j * 32) * ld + j * 32, ld, lane);
        const double myrd = __ldcg(wrd + j * 32 + lane);
        const int r = j * 32 + lane;
        const double bj = (j == 0) ? rhs_at(p, r) : __ldcg(wb + r);
        __syncwarp();
        wy[r] = fwd_block(bj, Bs, myrd, lane);
      }
      cluster_barrier();
      stamp(p, si);
    }
    // ---- trailing update A_IK -= L_Ij L_Kj^T, j < K <= I; block (j+1,j+1) is factored at once
    const int T = first ? 0 : nrem * (nrem + 1) / 2;
    if (crank == 0) {
      // The diagonal block is on the critical path (its factorisation follows): the 8 warps of CTA 0
      // update 4 columns each, warp 0 then factors it in registers.  (j = -1: block (0,0), no update)
      double *coopA = sm + (size_t)CH_WARPS * (32 * 32 + 32);  // L_{j+1,j}, column-major
      double *coopC = coopA + 1024;
      const int J1 = j + 1;
      double cv[4];
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const int k = 4 * w + i, r = J1 * 32 + lane, cc = J1 * 32 + k;
        if (jj == 0 && j <= 0) {
          cv[i] = (r < p.n && cc < p.n) ? p.A[(size_t)cc * p.n + r] + (r == cc ? p.mu : 0.0)
                                        : (r == cc ? 1.0 : 0.0);
        } else {
          cv[i] = __ldcg(ws + (size_t)cc * ld + r);
        }
      }
      if (!first) {
        const double *src = ws + (size_t)(j * 32) * ld + J1 * 32;
        double yv = 0.0, bI = 0.0;
        if (w == 1) {
          const int r = J1 * 32 + lane;
          yv = __ldcg(wy + j * 32 + lane);
          bI = (j == 0) ? rhs_at(p, r) : __ldcg(wb + r);
        }
        for (int e = threadIdx.x; e < 512; e += CH_THREADS) {
          const int c = e >> 4, r2 = e & 15;
          reinterpret_cast<double2 *>(coopA + c * 32)[r2] =
              __ldcg(reinterpret_cast<const double2 *>(src + (size_t)c * ld) + r2);
        }
        if (w == 1) rds[lane] = yv;
        __syncthreads();
        double a[32];
#pragma unroll
        for (int m = 0; m < 32; m++) a[m] = coopA[m * 32 + lane];
#pragma unroll
        for (int m = 0; m < 32; m++) {
          const double2 b0 = lds_v2(reinterpret_cast<const double2 *>(coopA + m * 32 + 4 * w));
          const double2 b1 = lds_v2(reinterpret_cast<const double2 *>(coopA + m * 32 + 4 * w + 2));
          cv[0] = fma(-a[m], b0.x, cv[0]);
          cv[1] = fma(-a[m], b0.y, cv[1]);
          cv[2] = fma(-a[m], b1.x, cv[2]);
          cv[3] = fma(-a[m], b1.y, cv[3]);
        }
        if (w == 1) wb[J1 * 32 + lane] = bI - dot32(a, rds);  // b_{j+1} -= L_{j+1,j} y_j
      }
#pragma unroll
      for (int i = 0; i < 4; i++) coopC[(4 * w + i) * 32 + lane] = cv[i];
      __syncthreads();
      if (w == 0) {
        double c[32], myrd = 0.0;
#pragma unroll
        for (int k = 0; k < 32; k++) c[k] = coopC[k * 32 + lane];
        __syncwarp();
        const int bad = potf2_warp(c, myrd, Bs, lane);
        wrd[J1 * 32 + lane] = myrd;
        if (bad && lane == 0) atomicCAS(p.info, 0, J1 * 32 + bad);
        store_rows(c, ws + (size_t)(J1 * 32) * ld + J1 * 32, ld, lane);
      }
    }
    // generic items: CTA 0 keeps its SM for the diagonal block (the other CL-1 CTAs share items 1..)
    const bool solo = (CL > 1);
    const int gu = solo ? (crank == 0 ? T : 1 + w * (CL - 1) + (crank - 1)) : g;
    const int Gu = solo ? (CL - 1) * CH_WARPS : G;
    for (int t = gu; t < T; t += Gu) {
      if (t == 0) continue;  // the diagonal block, done above
      int u = 0;
      while ((u + 1) * (u + 2) / 2 <= t) u++;
      const int v = t - u * (u + 1) / 2;
      const int I = j + 1 + u, K = j + 1 + v;
      double c[32];
      double *blk = ws + (size_t)(K * 32) * ld + I * 32;
      __syncwarp();
      stage_block(Bs, ws + (size_t)(jj * 32) * ld + K * 32, ld, lane);
      double a[32];
      load_rows(a, ws + (size_t)(jj * 32) * ld + I * 32, ld, lane);
      if (jj == 0) load_rows_A(c, p, I, K, lane);
      else load_rows(c, blk, ld, lane);
      if (v == 0) {
        // first trailing column: this warp holds row I of L_Ij, so b_I -= L_Ij y_j costs 32 FMAs
        rds[lane] = __ldcg(wy + j * 32 + lane);
        const int r = I * 32 + lane;
        const double bI = (j == 0) ? rhs_at(p, r) : __ldcg(wb + r);
        __syncwarp();
        wb[r] = bI - dot32(a, rds);
      }
      __syncwarp();
      update_warp(c, a, Bs);
      store_rows(c, blk, ld, lane);
    }
    cluster_barrier();
    stamp(p, si);
  }

  if (p.factor_only) return;  // every CTA leaves behind the same cluster barrier

  // ---- inverses of the diagonal blocks (one warp each, all concurrent): they turn the 32-step
  // substitutions of the two triangular solves into 32 x 32 matrix-vector products.
  for (int t = g; t < nblk; t += G) {
    __syncwarp();
    stage_block(Bs, ws + (size_t)(t * 32) * ld + t * 32, ld, lane);
    rds[lane] = __ldcg(wrd + t * 32 + lane);
    double x[32];
#pragma unroll
    for (int c = 0; c < 32; c++) x[c] = (c == lane) ? 1.0 : 0.0;
    __syncwarp();
    trsm_warp(x, Bs, rds);  // x[c] = (L^-1)[c][lane]
    // T[m*32 + l] = Linv[m][l]: what the back substitution multiplies with (the forward solve has
    // already happened along the factorisation, so L_jj^-1 itself is not stored)
    double *inv = winv + (size_t)t * 2048;
#pragma unroll
    for (int c = 0; c < 32; c++) inv[1024 + c * 32 + lane] = x[c];
  }
  if (g == G - 1) {
    const int j = nblk - 1;
    __syncwarp();
    stage_block(Bs, ws + (size_t)(j * 32) * ld + j * 32, ld, lane);
    const double myrd = __ldcg(wrd + j * 32 + lane);
    const int r = j * 32 + lane;
    const double bj = (j == 0) ? rhs_at(p, r) : __ldcg(wb + r);
    __syncwarp();
    wy[r] = fwd_block(bj, Bs, myrd, lane);
  }
  cluster_barrier();
  stamp(p, si);

  // ---- L^T x = y across the cluster.  CTA c owns the block columns j = c, c+CL, ...: it keeps their
  // sub-diagonal blocks and L_jj^-T in shared memory (one L2 round trip for everything), so no step
  // of the substitution waits on L2 and no SM has to stream the whole factor.  x_j = L_jj^-T (y_j -
  // sum_{I>j} L_Ij^T x_I): as soon as an x_I lands in this CTA's shared memory the warp I%8 adds its
  // term; the owner finishes the block, pushes x_j into every CTA (distributed shared memory) and
  // x_j itself is the arrival flag (the slots start as a NaN pattern no computation produces).
  double *ctrl = sm + ctrl_off(nblk, CL);  // behind the staging area: remote CTAs write here early
  double *xs = ctrl;                                                 // [ld]   solution, all CTAs
  double *partial = ctrl + ld + 2;                                   // [8][32]
  double *vbuf = partial + CH_WARPS * 32;                            // [32]
  double *tiles = sm;                                                // overlays the staging area
  const int ncol = (nblk - 1 - crank + CL) / CL;                     // own columns (crank < nblk)
  {
    // preload own columns, highest first (they are needed in that order)
    double *dst = tiles;
    for (int q = ncol - 1; q >= 0; q--) {
      const int j = crank + q * CL;
      for (int e = threadIdx.x; e < 1024; e += CH_THREADS) dst[e] = __ldcg(winv + (size_t)j * 2048 + 1024 + e);
      dst += 1024;
      for (int I = nblk - 1; I > j; I--) {
        if ((I & (CH_WARPS - 1)) == w) {
          double *tile = dst + (size_t)(nblk - 1 - I) * 1056;
          const double *src = ws + (size_t)(j * 32) * ld + I * 32;
#pragma unroll 8
          for (int c = 0; c < 32; c++) tile[c * 33 + lane] = __ldcg(src + (size_t)c * ld + lane);
        }
      }
      dst += (size_t)(nblk - 1 - j) * 1056;
    }
  }
  __syncthreads();
  {
    double *src = tiles;
    for (int q = ncol - 1; q >= 0; q--) {
      const int j = crank + q * CL;
      const double *T = src;
      const double *col = src + 1024;
      src += 1024 + (size_t)(nblk - 1 - j) * 1056;
      double part = 0.0;
      const double yj = (w == 0) ? __ldcg(wy + j * 32 + lane) : 0.0;  // off the chain: fetched now
      for (int I = nblk - 1; I > j; I--) {
        if ((I & (CH_WARPS - 1)) != w) continue;
        // wait for x_I: every lane watches one element (64-bit stores are single-copy atomic)
        {
          const unsigned addr = smem_u32(xs + I * 32 + lane);
          unsigned long long bits;
          do {
            asm volatile("ld.volatile.shared.u64 %0, [%1];" : "=l"(bits) : "r"(addr) : "memory");
          } while (bits == X_PENDING);
          __syncwarp();
        }
        const double *tile = col + (size_t)(nblk - 1 - I) * 1056 + lane * 33;  // element (r, c) at c*33 + r
        const double *xv = xs + I * 32;
        double s0 = 0.0, s1 = 0.0;
#pragma unroll 8
        for (int r = 0; r < 32; r += 2) {
          const double2 x2 = lds_v2(reinterpret_cast<const double2 *>(xv + r));
          s0 = fma(tile[r], x2.x, s0);  // L_Ij[r][lane]
          s1 = fma(tile[r + 1], x2.y, s1);
        }
        part += s0 + s1;
      }
      partial[w * 32 + lane] = part;
      __syncthreads();
      if (w == 0) {
        double v = yj;
#pragma unroll
        for (int ww = 0; ww < CH_WARPS; ww++) v -= partial[ww * 32 + lane];
        vbuf[lane] = v;
        __syncwarp();
        double s0 = 0.0, s1 = 0.0;
#pragma unroll 8
        for (int m = 0; m < 32; m += 2) {
          const double2 v2 = lds_v2(reinterpret_cast<const double2 *>(vbuf + m));
          s0 = fma(T[m * 32 + lane], v2.x, s0);
          s1 = fma(T[(m + 1) * 32 + lane], v2.y, s1);
        }
        const double xj = s0 + s1;
        const unsigned la = smem_u32(xs + j * 32 + lane);
        for (int r = 0; r < CL; r++) {
          unsigned ra;
          asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(la), "r"(r));
          asm volatile("st.shared::cluster.f64 [%0], %1;" ::"r"(ra), "d"(xj) : "memory");
        }
      }
      __syncthreads();
    }
  }
  if (crank == 0) solution_epilogue(xs, p.x, p.b, p.n, p.st, partial);
  // nobody leaves while a neighbour may still be writing into its shared memory
  asm volatile("barrier.cluster.arrive.release.aligned;\n"
               "barrier.cluster.wait.acquire.aligned;\n" ::: "memory");
  stamp(p, si);
}

// ------------------------------------------------------------------------------------------------
// Triangular solves only: L L^T x = b for a factor that already exists (column-major lower triangle,
// ld = n, as cusolverDnDpotrfBatched leaves it).  Used for the first LM solve of a cluster visit, whose
// factor comes out of the per-sweep batch.  Same cluster scheme as the tail of k_chol_solve, for both
// directions: CTA c owns block row/column c (+CL, ...); its diagonal blocks are inverted locally, its
// off-diagonal blocks sit in shared memory, every finished block of y (then x) is pushed into all
// CTAs and doubles as its own arrival flag.
// ------------------------------------------------------------------------------------------------
struct TriArgs {
  int ld;           // leading dimension of L (n for a cuSOLVER factor, 32*nblk for a k_chol_solve one)
  const double *L;  // n x n, lower triangle (column-major)
  const double *b;
  double *x;
  int n, nblk;
  StepArgs st;
};

__device__ __forceinline__ double l_elem(const TriArgs &p, int r, int c) {
  return (r < p.n && c < p.n) ? __ldg(p.L + (size_t)c * p.ld + r) : (r == c ? 1.0 : 0.0);
}

__device__ __forceinline__ void wait_block(const double *slot, int lane) {
  const unsigned addr = smem_u32(slot + lane);
  unsigned long long bits;
  do {
    asm volatile("ld.volatile.shared.u64 %0, [%1];" : "=l"(bits) : "r"(addr) : "memory");
  } while (bits == X_PENDING);
  __syncwarp();
}
__device__ __forceinline__ void publish_block(double *slot, double v, int lane, int CL) {
  const unsigned la = smem_u32(slot + lane);
  for (int r = 0; r < CL; r++) {
    unsigned ra;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(la), "r"(r));
    asm volatile("st.shared::cluster.f64 [%0], %1;" ::"r"(ra), "d"(v) : "memory");
  }
}

__global__ void __launch_bounds__(CH_THREADS, 1) k_tri_solve(TriArgs p) {
  extern __shared__ __align__(16) double sm[];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int crank = (int)cluster_rank(), CL = (int)cluster_size();
  const int nblk = p.nblk, ld = nblk * 32;
  // layout: tiles (CTA 0 of the backward pass owns the most) | ys | xs | partial | vbuf | inverses
  double *tiles = sm;
  double *ctrl = sm + tri_tiles(nblk, CL);
  double *ys = ctrl, *xs = ctrl + ld;
  double *partial = xs + ld, *vbuf = partial + CH_WARPS * 32;
  double *invs = vbuf + 32;  // per own diagonal block: Tf (32 x 33) then Tb (32 x 32)
  const int nown = (nblk - 1 - crank + CL) / CL;  // own block rows / columns: crank, crank+CL, ...

  for (int i = threadIdx.x; i < 2 * ld; i += CH_THREADS)
    reinterpret_cast<unsigned long long *>(ctrl)[i] = X_PENDING;
  // inverses of the own diagonal blocks (warp q for the q-th one; nown <= 2 in practice)
  for (int q = w; q < nown; q += CH_WARPS) {
    const int j = crank + q * CL;
    double *Tf = invs + (size_t)q * (32 * 33 + 1024), *Tb = Tf + 32 * 33;
    // stage L_jj column-major into Tb (scratch for now), reciprocal diagonal in registers
#pragma unroll 8
    for (int c = 0; c < 32; c++) Tb[c * 32 + lane] = l_elem(p, j * 32 + lane, j * 32 + c);
    __syncwarp();
    double xr[32];
#pragma unroll
    for (int c = 0; c < 32; c++) xr[c] = (c == lane) ? 1.0 : 0.0;
    // x <- e_lane L^-T (same recurrence as trsm_warp, reciprocals taken on the fly)
#pragma unroll
    for (int c = 0; c < 32; c++) {
      xr[c] = xr[c] / Tb[c * 32 + c];
      const double xc = xr[c];
#pragma unroll
      for (int m = c + 1; m < 32; m++) xr[m] = fma(-xc, Tb[c * 32 + m], xr[m]);
    }
    __syncwarp();
    // xr[c] = Linv[c][lane]
#pragma unroll
    for (int c = 0; c < 32; c++) {
      Tf[lane * 33 + c] = xr[c];   // forward: lane l reads Tf[m*33 + l] = Linv[l][m]
      Tb[c * 32 + lane] = xr[c];   // backward: lane l reads Tb[m*32 + l] = Linv[m][l]
    }
  }
  // cluster barrier: every CTA has initialised its slots before anybody publishes into them
  asm volatile("barrier.cluster.arrive.release.aligned;\n"
               "barrier.cluster.wait.acquire.aligned;\n" ::: "memory");

  // ---- forward: y_I = L_II^-1 (b_I - sum_{K<I} L_IK y_K), rows ascending
  {
    double *dst = tiles;
    for (int q = 0; q < nown; q++) {
      const int I = crank + q * CL;
      for (int K = 0; K < I; K++) {
        if ((K & (CH_WARPS - 1)) == w) {
          double *tile = dst + (size_t)K * 1056;
#pragma unroll 8
          for (int c = 0; c < 32; c++) tile[c * 33 + lane] = l_elem(p, I * 32 + lane, K * 32 + c);
        }
      }
      dst += (size_t)I * 1056;
    }
  }
  __syncthreads();
  {
    const double *src = tiles;
    for (int q = 0; q < nown; q++) {
      const int I = crank + q * CL;
      const double *Tf = invs + (size_t)q * (32 * 33 + 1024);
      const int r = I * 32 + lane;
      const double bI = (w == 0 && r < p.n) ? p.b[r] : 0.0;
      double part = 0.0;
      for (int K = 0; K < I; K++) {
        if ((K & (CH_WARPS - 1)) != w) continue;
        wait_block(ys + K * 32, lane);
        const double *tile = src + (size_t)K * 1056 + lane;  // element (lane, m) at m*33 + lane
        const double *yv = ys + K * 32;
        double s0 = 0.0, s1 = 0.0;
#pragma unroll 8
        for (int m = 0; m < 32; m += 2) {
          const double2 y2 = lds_v2(reinterpret_cast<const double2 *>(yv + m));
          s0 = fma(tile[m * 33], y2.x, s0);
          s1 = fma(tile[(m + 1) * 33], y2.y, s1);
        }
        part += s0 + s1;
      }
      src += (size_t)I * 1056;
      partial[w * 32 + lane] = part;
      __syncthreads();
      if (w == 0) {
        double v = bI;
#pragma unroll
        for (int ww = 0; ww < CH_WARPS; ww++) v -= partial[ww * 32 + lane];
        vbuf[lane] = v;
        __syncwarp();
        double s0 = 0.0, s1 = 0.0;
#pragma unroll 8
        for (int m = 0; m < 32; m += 2) {
          const double2 v2 = lds_v2(reinterpret_cast<const double2 *>(vbuf + m));
          s0 = fma(Tf[m * 33 + lane], v2.x, s0);
          s1 = fma(Tf[(m + 1) * 33 + lane], v2.y, s1);
        }
        publish_block(ys + I * 32, s0 + s1, lane, CL);
      }
      __syncthreads();
    }
  }
  // ---- backward: x_j = L_jj^-T (y_j - sum_{I>j} L_Ij^T x_I), columns descending
  {
    double *dst = tiles;
    for (int q = nown - 1; q >= 0; q--) {
      const int j = crank + q * CL;
      for (int I = nblk - 1; I > j; I--) {
        if ((I & (CH_WARPS - 1)) == w) {
          double *tile = dst + (size_t)(nblk - 1 - I) * 1056;
#pragma unroll 8
          for (int c = 0; c < 32; c++) tile[c * 33 + lane] = l_elem(p, I * 32 + lane, j * 32 + c);
        }
      }
      dst += (size_t)(nblk - 1 - j) * 1056;
    }
  }
  __syncthreads();
  {
    const double *src = tiles;
    for (int q = nown - 1; q >= 0; q--) {
      const int j = crank + q * CL;
      const double *Tb = invs + (size_t)q * (32 * 33 + 1024) + 32 * 33;
      double yj = 0.0;
      if (w == 0) {
        wait_block(ys + j * 32, lane);
        yj = ys[j * 32 + lane];
      }
      double part = 0.0;
      for (int I = nblk - 1; I > j; I--) {
        if ((I & (CH_WARPS - 1)) != w) continue;
        wait_block(xs + I * 32, lane);
        const double *tile = src + (size_t)(nblk - 1 - I) * 1056 + lane * 33;  // (r, lane) at lane*33 + r
        const double *xv = xs + I * 32;
        double s0 = 0.0, s1 = 0.0;
#pragma unroll 8
        for (int r = 0; r < 32; r += 2) {
          const double2 x2 = lds_v2(reinterpret_cast<const double2 *>(xv + r));
          s0 = fma(tile[r], x2.x, s0);
          s1 = fma(tile[r + 1], x2.y, s1);
        }
        part += s0 + s1;
      }
      src += (size_t)(nblk - 1 - j) * 1056;
      partial[w * 32 + lane] = part;
      __syncthreads();
      if (w == 0) {
        double v = yj;
#pragma unroll
        for (int ww = 0; ww < CH_WARPS; ww++) v -= partial[ww * 32 + lane];
        vbuf[lane] = v;
        __syncwarp();
        double s0 = 0.0, s1 = 0.0;
#pragma unroll 8
        for (int m = 0; m < 32; m += 2) {
          const double2 v2 = lds_v2(reinterpret_cast<const double2 *>(vbuf + m));
          s0 = fma(Tb[m * 32 + lane], v2.x, s0);
          s1 = fma(Tb[(m + 1) * 32 + lane], v2.y, s1);
        }
        publish_block(xs + j * 32, s0 + s1, lane, CL);
      }
      __syncthreads();
    }
  }
  if (crank == 0) solution_epilogue(xs, p.x, p.b, p.n, p.st, partial);
  asm volatile("barrier.cluster.arrive.release.aligned;\n"
               "barrier.cluster.wait.acquire.aligned;\n" ::: "memory");
}

size_t tri_smem(int nblk, int cl) {
  const int nown = (nblk - 1 + cl) / cl;
  return sizeof(double) * (tri_tiles(nblk, cl) + 2 * (size_t)nblk * 32 + CH_WARPS * 32 + 32 +
                           (size_t)nown * (32 * 33 + 1024));
}

__global__ void k_test_rsqrt(const double *in, double *out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = fast_rsqrt(in[i]);
}

int g_cluster = -1;  // 16, 8 or 0 (unavailable)

size_t chol_smem(int nblk, int cl) {
  // staging / column tiles, then xs, ready, partial, vbuf
  return sizeof(double) * (ctrl_off(nblk, cl) + (size_t)nblk * 32 + 2 + CH_WARPS * 32 + 32);
}

bool try_cluster(int cl, size_t smem) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(cl);
  cfg.blockDim = dim3(CH_THREADS);
  cfg.dynamicSmemBytes = smem;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = cl;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  int nclus = 0;
  if (cudaOccupancyMaxActiveClusters(&nclus, k_chol_solve, &cfg) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return nclus > 0;
}

}  // namespace

extern "C" {

// largest system the cluster solver takes (32*16 rows); larger ones stay on cuSOLVER
int db_chol_max_n() { return 512; }

size_t db_chol_ws_doubles(int n) {
  const size_t npad = (size_t)((n + 31) / 32) * 32;
  return npad * npad + 3 * npad + (npad / 32) * 2048;
}

// 1 if the device grants a cluster of 8 or 16 CTAs for the solver
int db_chol_available() {
  if (g_cluster < 0) {
    const size_t smem = chol_smem(16, 8);
    cudaFuncSetAttribute(k_chol_solve, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaFuncSetAttribute(k_chol_solve, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    const char *e = getenv("DIRAC_B200_CHOL_CLUSTER");
    const int want = e ? atoi(e) : 16;
    g_cluster = 0;
    if (want >= 16 && try_cluster(16, smem)) g_cluster = 16;
    else if (want >= 8 && try_cluster(8, smem)) g_cluster = 8;
    cudaGetLastError();
  }
  return g_cluster > 0;
}

// (A + mu I) x = b, n <= db_chol_max_n().  ws: db_chol_ws_doubles(n) doubles.  info: device int.
static long long *g_ts = nullptr;
static StepArgs g_step = {nullptr, nullptr, nullptr, nullptr};
// the next solver launches also form pnew = pcur + x, sc[0..1], and clear `zero` (pcur == nullptr: off)
void db_chol_set_step(const double *pcur, double *pnew, double *sc, double *zero) {
  g_step.pcur = pcur; g_step.pnew = pnew; g_step.sc = sc; g_step.zero = zero;
}
void db_launch_chol_solve(const double *A, int n, double mu, const double *b, double *x, double *ws,
                          int *info, cudaStream_t st) {
  CholArgs p;
  p.ts = g_ts;
  p.st = g_step;
  p.A = A; p.b = b; p.x = x; p.ws = ws; p.info = info; p.mu = mu; p.n = n; p.nblk = (n + 31) / 32;
  p.factor_only = 0; p.mu_ptr = nullptr; p.ws_stride = 0;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(g_cluster);
  cfg.blockDim = dim3(CH_THREADS);
  cfg.dynamicSmemBytes = chol_smem(p.nblk, g_cluster);
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = g_cluster;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  DB_CHECK(cudaLaunchKernelEx(&cfg, k_chol_solve, p));
}


// Batched factorisation: nb matrices A[b] (n x n, stride n*n), A[b] + mu[b] I = L L^T, one thread-block
// cluster each, all concurrent (the batch of first systems of a SAGE sweep: 64 clusters of 16 CTAs on
// 132 SMs run eight at a time).  Factor b lands at ws + b*ws_stride with ld = 32*ceil(n/32);
// info[2b] as dpotrf.  Replaces cusolverDnDpotrfBatched on this path.
void db_launch_chol_factor_batched(const double *A, int n, const double *mu, double *ws,
                                   long long ws_stride, int *info, int nb, cudaStream_t st) {
  CholArgs p;
  p.ts = nullptr;
  p.st.pcur = nullptr; p.st.pnew = nullptr; p.st.sc = nullptr; p.st.zero = nullptr;
  p.A = A; p.b = nullptr; p.x = nullptr; p.ws = ws; p.info = info; p.mu = 0.0; p.n = n;
  p.nblk = (n + 31) / 32;
  p.factor_only = 1; p.mu_ptr = mu; p.ws_stride = ws_stride;
  // Throughput, not latency, counts for the batch: small clusters (4 CTAs) keep 33 matrices in flight
  // on 132 SMs and spend less of their time in cluster barriers than the 16-CTA shape of a lone solve
  static int bcl = -1;
  if (bcl < 0) {
    const char *e = getenv("DIRAC_B200_BATCH_CL");
    bcl = e ? atoi(e) : 4;
    if (bcl != 1 && bcl != 2 && bcl != 4 && bcl != 8 && bcl != 16) bcl = 4;
    if (bcl > g_cluster) bcl = g_cluster;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(bcl * nb));
  cfg.blockDim = dim3(CH_THREADS);
  // the factorisation only needs the per-warp staging blocks and the cooperative diagonal block
  cfg.dynamicSmemBytes = ((size_t)CH_WARPS * (32 * 32 + 32) + 2048) * sizeof(double);
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = bcl;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  DB_CHECK(cudaLaunchKernelEx(&cfg, k_chol_solve, p));
}

// L L^T x = b with an existing factor (column-major lower, ld = n <= db_chol_max_n())
// 1 if the solve-only kernel fits this device's cluster size for n
int db_tri_available(int n) {
  if (n < 1 || n > db_chol_max_n() || !db_chol_available()) return 0;
  return tri_smem((n + 31) / 32, g_cluster) <= 227 * 1024;
}

void db_launch_tri_solve_ld(const double *L, int ld, int n, const double *b, double *x,
                            cudaStream_t st);
void db_launch_tri_solve(const double *L, int n, const double *b, double *x, cudaStream_t st) {
  db_launch_tri_solve_ld(L, n, n, b, x, st);
}
void db_launch_tri_solve_ld(const double *L, int ld, int n, const double *b, double *x,
                            cudaStream_t st) {
  TriArgs p;
  p.ld = ld;
  p.L = L; p.b = b; p.x = x; p.n = n; p.nblk = (n + 31) / 32;
  p.st = g_step;
  static bool configured = false;
  if (!configured) {
    size_t mx = tri_smem(16, g_cluster);
    if (mx > 227 * 1024) mx = 227 * 1024;
    cudaFuncSetAttribute(k_tri_solve, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)mx);
    cudaFuncSetAttribute(k_tri_solve, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    configured = true;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(g_cluster);
  cfg.blockDim = dim3(CH_THREADS);
  cfg.dynamicSmemBytes = tri_smem(p.nblk, g_cluster);
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = g_cluster;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  DB_CHECK(cudaLaunchKernelEx(&cfg, k_tri_solve, p));
}

// test hook: x = (L L^T)^-1 b from host buffers (L column-major lower with leading dimension
// ld >= n); returns -1 when the cluster solver is unavailable
int dirac_b200_tri_solve_ld(int n, const double *L, int ld, const double *b, double *x, int reps,
                            double *us) {
  if (!db_tri_available(n) || ld < n) return -1;
  double *dL, *db, *dx;
  DB_CHECK(cudaMalloc(&dL, sizeof(double) * ld * n));
  DB_CHECK(cudaMalloc(&db, sizeof(double) * n));
  DB_CHECK(cudaMalloc(&dx, sizeof(double) * n));
  DB_CHECK(cudaMemcpy(dL, L, sizeof(double) * ld * n, cudaMemcpyHostToDevice));
  DB_CHECK(cudaMemcpy(db, b, sizeof(double) * n, cudaMemcpyHostToDevice));
  db_launch_tri_solve_ld(dL, ld, n, db, dx, 0);
  DB_CHECK(cudaMemcpy(x, dx, sizeof(double) * n, cudaMemcpyDeviceToHost));
  if (reps > 0 && us) {
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    cudaEventRecord(e0, 0);
    for (int i = 0; i < reps; i++) db_launch_tri_solve_ld(dL, ld, n, db, dx, 0);
    cudaEventRecord(e1, 0);
    DB_CHECK(cudaEventSynchronize(e1));
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e0, e1);
    *us = 1e3 * ms / reps;
    cudaEventDestroy(e0); cudaEventDestroy(e1);
  }
  cudaFree(dL); cudaFree(db); cudaFree(dx);
  return 0;
}

// test hook: the batched factorisation of the LM's per-sweep batch from host buffers.  A: nb
// column-major n x n matrices back to back (only the lower triangles are read), mu: nb dampings.
// L: nb factors of A[b] + mu[b] I, each column-major ld x ld with ld = 32*ceil(n/32) as the solver
// leaves them (lower triangle of the leading n x n block; the rest is not part of the factor).
// info: 2*nb ints, info[2b] as dpotrf.  Returns -1 when the batch does not run on the cluster kernel
// (the LM then factorises with cuSOLVER).
int dirac_b200_chol_factor_batched(int n, int nb, const double *A, const double *mu, double *L,
                                   int *info) {
  if (!db_tri_available(n) || nb < 1) return -1;
  const size_t ld = (size_t)32 * ((n + 31) / 32), stride = db_chol_ws_doubles(n);
  double *dA, *dmu, *dws;
  int *dinfo;
  DB_CHECK(cudaMalloc(&dA, sizeof(double) * n * n * nb));
  DB_CHECK(cudaMalloc(&dmu, sizeof(double) * nb));
  DB_CHECK(cudaMalloc(&dws, sizeof(double) * stride * nb));
  DB_CHECK(cudaMalloc(&dinfo, sizeof(int) * 2 * nb));
  DB_CHECK(cudaMemset(dws, 0, sizeof(double) * stride * nb));
  DB_CHECK(cudaMemcpy(dA, A, sizeof(double) * n * n * nb, cudaMemcpyHostToDevice));
  DB_CHECK(cudaMemcpy(dmu, mu, sizeof(double) * nb, cudaMemcpyHostToDevice));
  db_launch_chol_factor_batched(dA, n, dmu, dws, (long long)stride, dinfo, nb, 0);
  for (int b = 0; b < nb; b++)
    DB_CHECK(cudaMemcpy(L + ld * ld * b, dws + stride * b, sizeof(double) * ld * ld,
                        cudaMemcpyDeviceToHost));
  DB_CHECK(cudaMemcpy(info, dinfo, sizeof(int) * 2 * nb, cudaMemcpyDeviceToHost));
  cudaFree(dA); cudaFree(dmu); cudaFree(dws); cudaFree(dinfo);
  return 0;
}

int dirac_b200_tri_solve(int n, const double *L, const double *b, double *x, int reps, double *us) {
  return dirac_b200_tri_solve_ld(n, L, n, b, x, reps, us);
}

// test hook: out[i] = fast_rsqrt(in[i]) as the pivots see it
int dirac_b200_test_rsqrt(int n, const double *in, double *out) {
  double *di, *dout;
  DB_CHECK(cudaMalloc(&di, sizeof(double) * n));
  DB_CHECK(cudaMalloc(&dout, sizeof(double) * n));
  DB_CHECK(cudaMemcpy(di, in, sizeof(double) * n, cudaMemcpyHostToDevice));
  k_test_rsqrt<<<(n + 255) / 256, 256>>>(di, dout, n);
  DB_CHECK(cudaMemcpy(out, dout, sizeof(double) * n, cudaMemcpyDeviceToHost));
  cudaFree(di); cudaFree(dout);
  return 0;
}

// host-buffer convenience wrapper (tests, diagnostics): returns 0, or -1 when the cluster solver is
// unavailable / n too large.  *info as dpotrf.
int dirac_b200_spd_solve(int n, const double *A, const double *b, double mu, double *x, int *info) {
  if (n < 1 || n > db_chol_max_n() || !db_chol_available()) return -1;
  double *dA, *db, *dx, *dws;
  int *dinfo;
  DB_CHECK(cudaMalloc(&dA, sizeof(double) * n * n));
  DB_CHECK(cudaMalloc(&db, sizeof(double) * n));
  DB_CHECK(cudaMalloc(&dx, sizeof(double) * n));
  DB_CHECK(cudaMalloc(&dws, sizeof(double) * db_chol_ws_doubles(n)));
  DB_CHECK(cudaMalloc(&dinfo, 2 * sizeof(int)));
  DB_CHECK(cudaMemcpy(dA, A, sizeof(double) * n * n, cudaMemcpyHostToDevice));
  DB_CHECK(cudaMemcpy(db, b, sizeof(double) * n, cudaMemcpyHostToDevice));
  db_launch_chol_solve(dA, n, mu, db, dx, dws, dinfo, 0);
  DB_CHECK(cudaMemcpy(x, dx, sizeof(double) * n, cudaMemcpyDeviceToHost));
  DB_CHECK(cudaMemcpy(info, dinfo, sizeof(int), cudaMemcpyDeviceToHost));
  cudaFree(dA); cudaFree(db); cudaFree(dx); cudaFree(dws); cudaFree(dinfo);
  return 0;
}

// average device time (us) of `reps` back-to-back solves of one resident system (tuning hook)
double dirac_b200_bench_spd_solve(int n, const double *A, const double *b, double mu, int reps) {
  if (n < 1 || n > db_chol_max_n() || !db_chol_available()) return -1.0;
  double *dA, *db, *dx, *dws;
  int *dinfo;
  DB_CHECK(cudaMalloc(&dA, sizeof(double) * n * n));
  DB_CHECK(cudaMalloc(&db, sizeof(double) * n));
  DB_CHECK(cudaMalloc(&dx, sizeof(double) * n));
  DB_CHECK(cudaMalloc(&dws, sizeof(double) * db_chol_ws_doubles(n)));
  DB_CHECK(cudaMalloc(&dinfo, 2 * sizeof(int)));
  DB_CHECK(cudaMemcpy(dA, A, sizeof(double) * n * n, cudaMemcpyHostToDevice));
  DB_CHECK(cudaMemcpy(db, b, sizeof(double) * n, cudaMemcpyHostToDevice));
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (int i = 0; i < 3; i++) db_launch_chol_solve(dA, n, mu, db, dx, dws, dinfo, 0);
  cudaEventRecord(e0, 0);
  for (int i = 0; i < reps; i++) db_launch_chol_solve(dA, n, mu, db, dx, dws, dinfo, 0);
  cudaEventRecord(e1, 0);
  DB_CHECK(cudaEventSynchronize(e1));
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e0, e1);
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  if (getenv("DIRAC_B200_CHOL_TS")) {
    long long *dts, hts[64] = {0};
    cudaMalloc(&dts, sizeof(hts));
    cudaMemset(dts, 0, sizeof(hts));
    g_ts = dts;
    db_launch_chol_solve(dA, n, mu, db, dx, dws, dinfo, 0);
    g_ts = nullptr;
    cudaMemcpy(hts, dts, sizeof(hts), cudaMemcpyDeviceToHost);
    for (int i = 1; i < 64 && hts[i]; i++) printf("  phase %2d: %7.2f us\n", i, 1e-3 * (hts[i] - hts[i - 1]));
    cudaFree(dts);
  }
  cudaFree(dA); cudaFree(db); cudaFree(dx); cudaFree(dws); cudaFree(dinfo);
  return 1e3 * ms / reps;
}

}  // extern "C"
