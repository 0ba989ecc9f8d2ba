// Triangular solves L L^T x = b for systems beyond the cluster kernels (8N > 512; 512 stations: n = 4096),
// on a factor cuSOLVER's dpotrf left (column-major lower, ld).  Replaces cusolverDnDpotrs, whose two
// trsv kernels take 0.68 ms for 2 x 67 MB of traffic: a dependency chain of n/64 block steps, bound by
// latency, not by bytes.
//
// Scheme: 64 x 64 blocks, nb = n/64.  A prologue kernel forms, per diagonal block, Linv_ii, and the two
// blocks that sit on the chain, M_i = Linv_ii L_{i,i-1} and N_j = (L_{j+1,j} Linv_jj)^T, and arms the
// solution slots.  One cooperative kernel then runs both directions: CTA i owns block row i forward and
// block column i backward,
//   y_i = Linv_ii s_i - M_i y_{i-1},     s_i = b_i - sum_{k<i-1} L_ik y_k
//   x_j = Linv_jj^T t_j - N_j x_{j+1},   t_j = y_j - sum_{i>j+1} L_ij^T x_i
// so everything but one 64 x 64 product from registers is done before the awaited block arrives.  The
// off-chain blocks of L stream through a per-thread cp.async ring in shared memory, the backward ones
// staged while the forward chain runs.  Each warp owns 8 rows (4 lanes per row, interleaved columns),
// waits for the incoming block itself and reduces with shuffles: the chain step has no CTA barrier.
// A solution block is its own arrival flag: the slots start as a NaN pattern no computation produces.
#include "internal.cuh"
#include <cusolverDn.h>
#include <vector>

#define BT 64           // block size
#define BT_THREADS 256  // 64 rows x 4 lanes
#define BT_STAGES 4     // cp.async ring depth (blocks of L in flight + 1)
#define BT_PENDING 0x7ff8dead0badbeefull  // quiet NaN with a payload no arithmetic produces

// "thread-private" layout of a 64 x 64 block A: thread t = 4r + q holds A[r][4c + q] at [c*256 + t]
__host__ __device__ __forceinline__ int bt_idx(int row, int col) {
  return (col >> 2) * BT_THREADS + row * 4 + (col & 3);
}

// per diagonal block b (one CTA): Linv_bb, M_b, N_b into ws in the layout above; y and x slots pending;
// *status = 0.  Shared memory: three 64 x 65 column-major tiles.
__global__ void __launch_bounds__(BT_THREADS)
k_bigtri_prep(const double *__restrict__ L, int ld, int nb, double *__restrict__ Linv,
              double *__restrict__ M, double *__restrict__ N, unsigned long long *y,
              unsigned long long *x, int *status) {
  extern __shared__ double sp[];
  double *Ls = sp, *Ic = Ls + BT * 65, *Ys = Ic + BT * 65;
  double *Ir = Ls;  // Linv row-major, once the inversion no longer reads L_bb
  const int b = blockIdx.x, tid = threadIdx.x, r = tid >> 2, q = tid & 3;
  if (tid < BT) {
    y[b * BT + tid] = BT_PENDING;
    x[b * BT + tid] = BT_PENDING;
  }
  if (b == 0 && tid == 0 && status) *status = 0;
  const double *Lbb = L + (size_t)(b * BT) * ld + b * BT;
  for (int e = tid; e < BT * BT; e += BT_THREADS) Ls[(e >> 6) * 65 + (e & 63)] = Lbb[(size_t)(e >> 6) * ld + (e & 63)];
  __syncthreads();
  // column c of Linv: L z = e_c, column-oriented (the updates of one step are independent)
  double z[BT];
  if (tid < BT) {
#pragma unroll
    for (int k = 0; k < BT; k++) z[k] = (k == tid) ? 1.0 : 0.0;
#pragma unroll
    for (int k = 0; k < BT; k++) {
      const double zk = z[k] / Ls[k * 65 + k];
      z[k] = zk;
#pragma unroll
      for (int rr = k + 1; rr < BT; rr++) z[rr] = fma(-Ls[k * 65 + rr], zk, z[rr]);
    }
  }
  __syncthreads();
  if (tid < BT) {
    double *dst = Linv + (size_t)b * BT * BT;
#pragma unroll
    for (int rr = 0; rr < BT; rr++) {
      Ic[tid * 65 + rr] = z[rr];  // Ic[c*65 + r] = Linv[r][c]
      Ir[rr * 65 + tid] = z[rr];  // Ir[k*65 + r] = Linv[k][r]
      dst[bt_idx(rr, tid)] = z[rr];
    }
  }
  // P[r][c] = sum_k X[r][k] Y[k][c] with X[r][k] at Xs[k*65 + r] and Y[k][c] at Ys[c*65 + k]
  auto product = [&](const double *Xs, double *out) {
    double p[16];
#pragma unroll
    for (int c = 0; c < 16; c++) p[c] = 0.0;
#pragma unroll 4
    for (int k = 0; k < BT; k++) {
      const double xr = Xs[k * 65 + r];
#pragma unroll
      for (int c = 0; c < 16; c++) p[c] = fma(xr, Ys[(4 * c + q) * 65 + k], p[c]);
    }
#pragma unroll
    for (int c = 0; c < 16; c++) out[c * BT_THREADS + tid] = p[c];
  };
  if (b > 0) {  // M_b = Linv_bb L_{b,b-1}
    const double *src = L + (size_t)((b - 1) * BT) * ld + b * BT;
    for (int e = tid; e < BT * BT; e += BT_THREADS) Ys[(e >> 6) * 65 + (e & 63)] = src[(size_t)(e >> 6) * ld + (e & 63)];
    __syncthreads();
    product(Ic, M + (size_t)b * BT * BT);
  }
  if (b < nb - 1) {  // N_b = Linv_bb^T L_{b+1,b}^T
    __syncthreads();
    const double *src = L + (size_t)(b * BT) * ld + (b + 1) * BT;
    for (int e = tid; e < BT * BT; e += BT_THREADS) Ys[(e & 63) * 65 + (e >> 6)] = src[(size_t)(e >> 6) * ld + (e & 63)];
    __syncthreads();
    product(Ir, N + (size_t)b * BT * BT);
  }
}

struct BigTriArgs {
  const double *L, *Linv, *M, *N;  // Linv, M, N: [nb][64*64] from k_bigtri_prep
  const double *b;
  double *y, *x;
  int ld, nb;
};

__device__ __forceinline__ void cp_async8(double *dst, const double *src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((unsigned)__cvta_generic_to_shared(dst)),
               "l"(src)
               : "memory");
}

// sum over the 4 lanes of a row (every lane gets the same bits)
__device__ __forceinline__ double quad_sum(double v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// the warp waits for a solution block and leaves it in its own 64-entry vector
__device__ __forceinline__ void await_block(const double *slot, double *vw, int lane) {
  const unsigned long long *p = reinterpret_cast<const unsigned long long *>(slot);
  unsigned long long u, v;
  do {
    asm volatile("ld.relaxed.gpu.u64 %0, [%1];" : "=l"(u) : "l"(p + lane) : "memory");
    asm volatile("ld.relaxed.gpu.u64 %0, [%1];" : "=l"(v) : "l"(p + lane + 32) : "memory");
  } while (u == BT_PENDING || v == BT_PENDING);
  __syncwarp();  // the previous block's readers are done
  vw[lane] = __longlong_as_double((long long)u);
  vw[lane + 32] = __longlong_as_double((long long)v);
  __syncwarp();
}

__global__ void __launch_bounds__(BT_THREADS, 1)
k_bigtri(BigTriArgs a) {
  extern __shared__ __align__(16) double sm[];
  double *ring = sm;                                    // [BT_STAGES][16][256]
  double *LiF = ring + BT_STAGES * 16 * BT_THREADS;     // Linv_ii, thread-private
  double *LiB = LiF + 16 * BT_THREADS;                  // Linv_ii^T, thread-private
  double *vec = LiB + 16 * BT_THREADS;                  // [8 warps][64] incoming block
  double *sv = vec + 8 * BT;                            // [64] s_i, then t_i
  const int tid = threadIdx.x, lane = tid & 31, r = tid >> 2, q = tid & 3;
  const int me = blockIdx.x, nb = a.nb;
  double *vw = vec + (tid >> 5) * BT;
  const int nf = me > 1 ? me - 1 : 0;            // off-chain blocks forward: L_{me,k}, k < me-1
  const int nbw = me < nb - 2 ? nb - 2 - me : 0;  // backward: L_{i,me}, i > me+1, descending
  const int ntot = nf + nbw;
  const double *Lf = a.L + (size_t)q * a.ld + me * BT + r;
  const double *Lb = a.L + (size_t)(me * BT + r) * a.ld + q;
  auto issue = [&](int blk) {
    if (blk < ntot) {
      double *dst = ring + (blk % BT_STAGES) * 16 * BT_THREADS + tid;
      if (blk < nf) {
        const double *src = Lf + (size_t)(blk * BT) * a.ld;
#pragma unroll
        for (int c = 0; c < 16; c++) cp_async8(dst + c * BT_THREADS, src + (size_t)(4 * c) * a.ld);
      } else {
        const double *src = Lb + (nb - 1 - (blk - nf)) * BT;
#pragma unroll
        for (int c = 0; c < 16; c++) cp_async8(dst + c * BT_THREADS, src + 4 * c);
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  // consume block blk of the stream against the warp's vector
  auto consume = [&](int blk, double acc) {
    asm volatile("cp.async.wait_group %0;" ::"n"(BT_STAGES - 2) : "memory");
    issue(blk + BT_STAGES - 1);
    const double *src = ring + (blk % BT_STAGES) * 16 * BT_THREADS + tid;
#pragma unroll
    for (int c = 0; c < 16; c++) acc = fma(-src[c * BT_THREADS], vw[4 * c + q], acc);
    return acc;
  };
  for (int s = 0; s < BT_STAGES - 1; s++) issue(s);
  const size_t off = (size_t)me * BT * BT;
  double Mr[16], Nr[16];
#pragma unroll
  for (int c = 0; c < 16; c++) {
    Mr[c] = me > 0 ? __ldg(a.M + off + c * BT_THREADS + tid) : 0.0;
    Nr[c] = me < nb - 1 ? __ldg(a.N + off + c * BT_THREADS + tid) : 0.0;
    LiF[c * BT_THREADS + tid] = __ldg(a.Linv + off + c * BT_THREADS + tid);
    LiB[c * BT_THREADS + tid] = __ldg(a.Linv + off + bt_idx(4 * c + q, r));
  }
  // ---- forward
  double acc = q == 0 ? a.b[me * BT + r] : 0.0;
  for (int k = 0; k < nf; k++) {
    await_block(a.y + (size_t)k * BT, vw, lane);
    acc = consume(k, acc);
  }
  acc = quad_sum(acc);
  if (q == 0) sv[r] = acc;
  __syncthreads();  // also: LiF / LiB staged
  double u = 0.0;
#pragma unroll
  for (int c = 0; c < 16; c++) u = fma(LiF[c * BT_THREADS + tid], sv[4 * c + q], u);
  u = quad_sum(u);
  if (me > 0) {
    await_block(a.y + (size_t)(me - 1) * BT, vw, lane);
    double p0 = 0.0, p1 = 0.0;
#pragma unroll
    for (int c = 0; c < 16; c += 2) {
      p0 = fma(Mr[c], vw[4 * c + q], p0);
      p1 = fma(Mr[c + 1], vw[4 * c + 4 + q], p1);
    }
    u -= quad_sum(p0 + p1);
  }
  const double yr = u;
  if (q == 0) asm volatile("st.relaxed.gpu.f64 [%0], %1;" ::"l"(a.y + (size_t)me * BT + r), "d"(yr) : "memory");
  // ---- backward
  acc = q == 0 ? yr : 0.0;
  for (int t = 0; t < nbw; t++) {
    await_block(a.x + (size_t)(nb - 1 - t) * BT, vw, lane);
    acc = consume(nf + t, acc);
  }
  acc = quad_sum(acc);
  __syncthreads();  // every warp has read s_i
  if (q == 0) sv[r] = acc;
  __syncthreads();
  u = 0.0;
#pragma unroll
  for (int c = 0; c < 16; c++) u = fma(LiB[c * BT_THREADS + tid], sv[4 * c + q], u);
  u = quad_sum(u);
  if (me < nb - 1) {
    await_block(a.x + (size_t)(me + 1) * BT, vw, lane);
    double p0 = 0.0, p1 = 0.0;
#pragma unroll
    for (int c = 0; c < 16; c += 2) {
      p0 = fma(Nr[c], vw[4 * c + q], p0);
      p1 = fma(Nr[c + 1], vw[4 * c + 4 + q], p1);
    }
    u -= quad_sum(p0 + p1);
  }
  if (q == 0) asm volatile("st.relaxed.gpu.f64 [%0], %1;" ::"l"(a.x + (size_t)me * BT + r), "d"(u) : "memory");
}

static const size_t bt_prep_smem = sizeof(double) * 3 * BT * 65;
static const size_t bt_smem = sizeof(double) * ((BT_STAGES + 2) * 16 * BT_THREADS + 8 * BT + BT);

extern "C" {
// 1 if this size is handled (multiple of 64, all CTAs co-resident)
int db_bigtri_available(int n) {
  if (getenv("DIRAC_B200_NO_BIGTRI")) return 0;
  return n > 512 && (n % BT) == 0 && n / BT <= db_sm_count();
}
size_t db_bigtri_ws_doubles(int n) { return (size_t)3 * (n / BT) * BT * BT + (size_t)n; }

// L L^T x = b.  ws: db_bigtri_ws_doubles(n) doubles (Linv | M | N | y).  status: cleared (may be null).
// Two launches: the prologue, then both substitutions in one cooperative kernel.
void db_launch_bigtri_solve(const double *L, int ld, int n, const double *b, double *x, double *ws,
                            int *status, cudaStream_t st) {
  const int nb = n / BT;
  const size_t blk = (size_t)nb * BT * BT;
  BigTriArgs a;
  a.L = L; a.ld = ld; a.nb = nb; a.b = b; a.x = x;
  a.Linv = ws; a.M = ws + blk; a.N = ws + 2 * blk; a.y = ws + 3 * blk;
  static bool configured = false;
  if (!configured) {
    DB_CHECK(cudaFuncSetAttribute(k_bigtri_prep, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bt_prep_smem));
    DB_CHECK(cudaFuncSetAttribute(k_bigtri, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bt_smem));
    configured = true;
  }
  k_bigtri_prep<<<nb, BT_THREADS, bt_prep_smem, st>>>(L, ld, nb, ws, ws + blk, ws + 2 * blk,
                                                      reinterpret_cast<unsigned long long *>(a.y),
                                                      reinterpret_cast<unsigned long long *>(x), status);
  void *args[] = {&a};
  DB_CHECK(cudaLaunchCooperativeKernel((const void *)k_bigtri, dim3(nb), dim3(BT_THREADS), args, bt_smem, st));
}

// test / tuning hook: x = (L L^T)^-1 b from host buffers (L column-major lower, ld = n); reps > 0
// additionally times `reps` back-to-back solves on the resident factor (us per solve in *us).
// returns -1 when the size is not handled
int dirac_b200_bigtri_solve(int n, const double *L, const double *b, double *x, int reps, double *us) {
  if (!db_bigtri_available(n)) return -1;
  double *dL, *db, *dx, *ws;
  DB_CHECK(cudaMalloc((void **)&dL, sizeof(double) * (size_t)n * n));
  DB_CHECK(cudaMalloc((void **)&db, sizeof(double) * n));
  DB_CHECK(cudaMalloc((void **)&dx, sizeof(double) * n));
  DB_CHECK(cudaMalloc((void **)&ws, sizeof(double) * db_bigtri_ws_doubles(n)));
  DB_CHECK(cudaMemcpy(dL, L, sizeof(double) * (size_t)n * n, cudaMemcpyHostToDevice));
  DB_CHECK(cudaMemcpy(db, b, sizeof(double) * n, cudaMemcpyHostToDevice));
  db_launch_bigtri_solve(dL, n, n, db, dx, ws, nullptr, 0);
  DB_CHECK(cudaDeviceSynchronize());
  DB_CHECK(cudaMemcpy(x, dx, sizeof(double) * n, cudaMemcpyDeviceToHost));
  if (reps > 0 && us) {
    cudaEvent_t e0, e1;
    DB_CHECK(cudaEventCreate(&e0));
    DB_CHECK(cudaEventCreate(&e1));
    DB_CHECK(cudaEventRecord(e0, 0));
    for (int i = 0; i < reps; i++) db_launch_bigtri_solve(dL, n, n, db, dx, ws, nullptr, 0);
    DB_CHECK(cudaEventRecord(e1, 0));
    DB_CHECK(cudaEventSynchronize(e1));
    float ms = 0.f;
    DB_CHECK(cudaEventElapsedTime(&ms, e0, e1));
    *us = 1e3 * ms / reps;
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
  }
  DB_CHECK(cudaGetLastError());
  cudaFree(dL); cudaFree(db); cudaFree(dx); cudaFree(ws);
  return 0;
}

// test / measurement hook: the LM's use of the substitutions.  A: nfac SPD matrices (n x n each,
// column-major), factored in place by cusolverDnDpotrf; b: nsolve right-hand sides.  Solve s uses
// factor s % nfac and right-hand side s, into one output vector on one workspace, back to back with no
// host synchronisation (answer s copied out on the stream) -> x[s*n ..].  reps > 0 then times `reps`
// solves rotating over the factors (us[0], us per solve) and `reps` dpotrf of a fresh copy of A_0
// (us[1], us per factorisation, the copies untimed).  Returns -1 when the size is not handled, -2
// when a matrix is not positive definite.
int dirac_b200_bigtri_sequence(int n, int nfac, const double *A, int nsolve, const double *b,
                               double *x, int reps, double *us) {
  if (!db_bigtri_available(n) || nfac < 1 || nsolve < 1) return -1;
  const size_t nn = (size_t)n * n;
  double *dA, *dcopy, *db, *dx, *dans, *ws, *work;
  int *info, lwork = 0;
  cusolverDnHandle_t cs;
  if (cusolverDnCreate(&cs) != CUSOLVER_STATUS_SUCCESS) return -1;
  DB_CHECK(cudaMalloc((void **)&dA, sizeof(double) * nn * nfac));
  DB_CHECK(cudaMalloc((void **)&dcopy, sizeof(double) * nn));
  DB_CHECK(cudaMalloc((void **)&db, sizeof(double) * (size_t)n * nsolve));
  DB_CHECK(cudaMalloc((void **)&dans, sizeof(double) * (size_t)n * nsolve));
  DB_CHECK(cudaMalloc((void **)&dx, sizeof(double) * n));
  DB_CHECK(cudaMalloc((void **)&ws, sizeof(double) * db_bigtri_ws_doubles(n)));
  DB_CHECK(cudaMalloc((void **)&info, sizeof(int) * (nfac + 1)));
  DB_CHECK(cudaMemcpy(dA, A, sizeof(double) * nn * nfac, cudaMemcpyHostToDevice));
  DB_CHECK(cudaMemcpy(dcopy, dA, sizeof(double) * nn, cudaMemcpyDeviceToDevice));
  DB_CHECK(cudaMemcpy(db, b, sizeof(double) * (size_t)n * nsolve, cudaMemcpyHostToDevice));
  cusolverDnDpotrf_bufferSize(cs, CUBLAS_FILL_MODE_LOWER, n, dA, n, &lwork);
  DB_CHECK(cudaMalloc((void **)&work, sizeof(double) * (lwork + 1)));
  int rc = 0;
  std::vector<int> hinfo(nfac);
  for (int f = 0; f < nfac; f++)
    cusolverDnDpotrf(cs, CUBLAS_FILL_MODE_LOWER, n, dA + nn * f, n, work, lwork, info + f);
  DB_CHECK(cudaMemcpy(hinfo.data(), info, sizeof(int) * nfac, cudaMemcpyDeviceToHost));
  for (int f = 0; f < nfac; f++)
    if (hinfo[f]) rc = -2;
  if (rc == 0) {
    for (int s = 0; s < nsolve; s++) {
      db_launch_bigtri_solve(dA + nn * (s % nfac), n, n, db + (size_t)n * s, dx, ws, info + nfac, 0);
      DB_CHECK(cudaMemcpyAsync(dans + (size_t)n * s, dx, sizeof(double) * n, cudaMemcpyDeviceToDevice, 0));
    }
    DB_CHECK(cudaDeviceSynchronize());
    DB_CHECK(cudaMemcpy(x, dans, sizeof(double) * (size_t)n * nsolve, cudaMemcpyDeviceToHost));
  }
  if (rc == 0 && reps > 0 && us) {
    cudaEvent_t e0, e1;
    DB_CHECK(cudaEventCreate(&e0));
    DB_CHECK(cudaEventCreate(&e1));
    float ms = 0.f, t = 0.f;
    for (int i = 0; i < 3 + nfac; i++) db_launch_bigtri_solve(dA + nn * (i % nfac), n, n, db, dx, ws, info + nfac, 0);
    DB_CHECK(cudaEventRecord(e0, 0));
    for (int i = 0; i < reps; i++) db_launch_bigtri_solve(dA + nn * (i % nfac), n, n, db, dx, ws, info + nfac, 0);
    DB_CHECK(cudaEventRecord(e1, 0));
    DB_CHECK(cudaEventSynchronize(e1));
    DB_CHECK(cudaEventElapsedTime(&ms, e0, e1));
    us[0] = 1e3 * ms / reps;
    ms = 0.f;
    for (int i = 0; i < reps + 1; i++) {
      DB_CHECK(cudaMemcpyAsync(dA, dcopy, sizeof(double) * nn, cudaMemcpyDeviceToDevice, 0));
      DB_CHECK(cudaEventRecord(e0, 0));
      cusolverDnDpotrf(cs, CUBLAS_FILL_MODE_LOWER, n, dA, n, work, lwork, info);
      DB_CHECK(cudaEventRecord(e1, 0));
      DB_CHECK(cudaEventSynchronize(e1));
      DB_CHECK(cudaEventElapsedTime(&t, e0, e1));
      if (i > 0) ms += t;  // the first one warms up
    }
    us[1] = 1e3 * ms / reps;
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
  }
  DB_CHECK(cudaGetLastError());
  cudaFree(dA); cudaFree(dcopy); cudaFree(db); cudaFree(dans); cudaFree(dx); cudaFree(ws); cudaFree(info);
  cudaFree(work);
  cusolverDnDestroy(cs);
  return rc;
}
}
