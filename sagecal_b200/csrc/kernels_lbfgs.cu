// Vector algebra of the LBFGS iteration on the device (the reference runs it on the host with
// my_ddot / my_daxpy over the whole Jones vector, lbfgs.c:33-111,479-640).
//
// k_lbfgs_direction is the complete two-loop recursion (mult_hessian, lbfgs.c:33-111) in ONE launch
// of one thread-block cluster: each of the 8 CTAs owns a slice of every vector, a dot product is a
// CTA reduction followed by an exchange of the 8 partial sums through distributed shared memory, and
// the 2M+1 dependent dot products / 2M axpys run back to back without touching the host.  No scalar
// ever leaves the device: rho_j lives in a device array, written by k_lbfgs_update.  The alpha_i of
// one recursion sit in dynamic shared memory, one double per pair, so the memory size has no cap
// below what one CTA can hold (db_lbfgs_direction_max_pairs: ~29000 pairs on an H100).
#include <cooperative_groups.h>

#include "internal.cuh"

namespace cg = cooperative_groups;

#define LB_CTAS 8
#define LB_THREADS 512

// sum over the cluster; every thread of every CTA gets the total (fixed order: deterministic)
__device__ __forceinline__ double cluster_sum(double v, double *red /*[16 + LB_CTAS]*/,
                                              cg::cluster_group &cl) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) red[w] = v;
  __syncthreads();
  if (w == 0) {
    double s = (lane < LB_THREADS / 32) ? red[lane] : 0.0;
    s = warp_sum(s);
    if (lane == 0) red[16] = s;  // this CTA's partial
  }
  cl.sync();
  double tot = 0.0;
#pragma unroll
  for (int r = 0; r < LB_CTAS; r++) tot += *cl.map_shared_rank(&red[16], r);
  cl.sync();  // partials may be overwritten by the next reduction only after everyone has read them
  return tot;
}

struct LbfgsDirArgs {
  double *pk;           // [m] out: -H g
  const double *gk;     // [m]
  const double *s, *y;  // [Mmem][m]
  const double *rho;    // [Mmem]
  int m, npairs, next;  // valid pairs, slot that will be written next (lbfgs.c "ii")
};

__global__ void __cluster_dims__(LB_CTAS, 1, 1) __launch_bounds__(LB_THREADS)
k_lbfgs_direction(LbfgsDirArgs a) {
  __shared__ double red[16 + 8];
  extern __shared__ double alphai[];  // [npairs]
  cg::cluster_group cl = cg::this_cluster();
  const int rank = (int)cl.block_rank();
  const int per = (a.m + LB_CTAS - 1) / LB_CTAS;
  const int i0 = rank * per, i1 = min(a.m, i0 + per);
  const int M = a.npairs;
  // order of the pairs, oldest ... newest (lbfgs.c:47-63)
  int ii = (a.next > 0) ? a.next - 1 : M - 1;
  auto slot = [&](int ci) { return (ci < M - ii - 1) ? ii + ci + 1 : ci - M + ii + 1; };
  for (int i = i0 + threadIdx.x; i < i1; i += LB_THREADS) a.pk[i] = a.gk[i];
  __syncthreads();
  for (int ci = 0; ci < M; ci++) {
    const int j = slot(M - ci - 1);
    const double *sj = a.s + (size_t)a.m * j, *yj = a.y + (size_t)a.m * j;
    double v = 0.0;
    for (int i = i0 + threadIdx.x; i < i1; i += LB_THREADS) v = fma(sj[i], a.pk[i], v);
    const double al = a.rho[j] * cluster_sum(v, red, cl);
    if (threadIdx.x == 0) alphai[M - ci - 1] = al;
    for (int i = i0 + threadIdx.x; i < i1; i += LB_THREADS) a.pk[i] = fma(-al, yj[i], a.pk[i]);
    __syncthreads();
  }
  if (M > 0) {
    const int j = slot(M - 1);
    const double *sj = a.s + (size_t)a.m * j, *yj = a.y + (size_t)a.m * j;
    double v1 = 0.0, v2 = 0.0;
    for (int i = i0 + threadIdx.x; i < i1; i += LB_THREADS) {
      v1 = fma(sj[i], yj[i], v1);
      v2 = fma(yj[i], yj[i], v2);
    }
    const double gamma = cluster_sum(v1, red, cl) / cluster_sum(v2, red, cl);
    for (int i = i0 + threadIdx.x; i < i1; i += LB_THREADS) a.pk[i] *= gamma;
    __syncthreads();
  }
  for (int ci = 0; ci < M; ci++) {
    const int j = slot(ci);
    const double *sj = a.s + (size_t)a.m * j, *yj = a.y + (size_t)a.m * j;
    double v = 0.0;
    for (int i = i0 + threadIdx.x; i < i1; i += LB_THREADS) v = fma(yj[i], a.pk[i], v);
    const double beta = a.rho[j] * cluster_sum(v, red, cl);
    const double c = alphai[ci] - beta;
    for (int i = i0 + threadIdx.x; i < i1; i += LB_THREADS) a.pk[i] = fma(c, sj[i], a.pk[i]);
    __syncthreads();
  }
  // search direction is -H g (lbfgs.c:560-561)
  for (int i = i0 + threadIdx.x; i < i1; i += LB_THREADS) a.pk[i] = -a.pk[i];
}

// ||g||^2 into out[0]
__global__ void __cluster_dims__(LB_CTAS, 1, 1) __launch_bounds__(LB_THREADS)
k_lbfgs_nrm2(const double *__restrict__ g, int m, double *out) {
  __shared__ double red[16 + 8];
  cg::cluster_group cl = cg::this_cluster();
  const int rank = (int)cl.block_rank();
  const int per = (m + LB_CTAS - 1) / LB_CTAS;
  const int i0 = rank * per, i1 = min(m, i0 + per);
  double v = 0.0;
  for (int i = i0 + threadIdx.x; i < i1; i += LB_THREADS) v = fma(g[i], g[i], v);
  v = cluster_sum(v, red, cl);
  if (rank == 0 && threadIdx.x == 0) out[0] = v;
}

// step of the iteration (lbfgs.c:574-617): xk1 = xk + alpha pk ; sk = xk1 - xk ; yk = -gk_old
__global__ void __launch_bounds__(256)
k_lbfgs_step(const double *__restrict__ xk, const double *__restrict__ pk,
             const double *__restrict__ gk, double *__restrict__ xk1, double *__restrict__ sk,
             double *__restrict__ yk, int m, double alpha) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
    const double x0 = xk[i];
    const double x1 = fma(alpha, pk[i], x0);
    xk1[i] = x1;
    sk[i] = x1 - x0;
    yk[i] = -gk[i];
  }
}

// yk += gk_new ; rho = 1 / (yk . sk) ; out[0] = ||gk_new||^2 ; xk = xk1
__global__ void __cluster_dims__(LB_CTAS, 1, 1) __launch_bounds__(LB_THREADS)
k_lbfgs_update(const double *__restrict__ gk, const double *__restrict__ sk, double *__restrict__ yk,
               const double *__restrict__ xk1, double *__restrict__ xk, int m, double *rho_slot,
               double *out) {
  __shared__ double red[16 + 8];
  cg::cluster_group cl = cg::this_cluster();
  const int rank = (int)cl.block_rank();
  const int per = (m + LB_CTAS - 1) / LB_CTAS;
  const int i0 = rank * per, i1 = min(m, i0 + per);
  double ys = 0.0, gg = 0.0;
  for (int i = i0 + threadIdx.x; i < i1; i += LB_THREADS) {
    const double g = gk[i];
    const double y = yk[i] + g;
    yk[i] = y;
    ys = fma(y, sk[i], ys);
    gg = fma(g, g, gg);
    xk[i] = xk1[i];
  }
  ys = cluster_sum(ys, red, cl);
  gg = cluster_sum(gg, red, cl);
  if (rank == 0 && threadIdx.x == 0) {
    *rho_slot = 1.0 / ys;
    out[0] = gg;
  }
}

extern "C" {
// the most pairs k_lbfgs_direction can hold: the opt-in shared memory of one CTA less its static part
int db_lbfgs_direction_max_pairs(void) {
  static int maxp = -1;
  if (maxp < 0) {
    int dev, optin;
    cudaFuncAttributes fa;
    DB_CHECK(cudaGetDevice(&dev));
    DB_CHECK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    DB_CHECK(cudaFuncGetAttributes(&fa, k_lbfgs_direction));
    maxp = (int)((optin - (long long)fa.sharedSizeBytes) / (long long)sizeof(double));
  }
  return maxp;
}
// npairs <= db_lbfgs_direction_max_pairs() (the caller checks)
void db_launch_lbfgs_direction(double *pk, const double *gk, const double *s, const double *y,
                               const double *rho, int m, int npairs, int next, cudaStream_t st) {
  LbfgsDirArgs a;
  a.pk = pk; a.gk = gk; a.s = s; a.y = y; a.rho = rho; a.m = m; a.npairs = npairs; a.next = next;
  const size_t smem = sizeof(double) * (size_t)npairs;
  if (smem > 48 * 1024)
    DB_CHECK(cudaFuncSetAttribute(k_lbfgs_direction, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)smem));
  k_lbfgs_direction<<<LB_CTAS, LB_THREADS, smem, st>>>(a);
}
void db_launch_lbfgs_nrm2(const double *g, int m, double *out, cudaStream_t st) {
  k_lbfgs_nrm2<<<LB_CTAS, LB_THREADS, 0, st>>>(g, m, out);
}
void db_launch_lbfgs_step(const double *xk, const double *pk, const double *gk, double *xk1,
                          double *sk, double *yk, int m, double alpha, cudaStream_t st) {
  int grid = (m + 255) / 256;
  if (grid > 592) grid = 592;
  k_lbfgs_step<<<grid, 256, 0, st>>>(xk, pk, gk, xk1, sk, yk, m, alpha);
}
void db_launch_lbfgs_update(const double *gk, const double *sk, double *yk, const double *xk1,
                            double *xk, int m, double *rho_slot, double *out, cudaStream_t st) {
  k_lbfgs_update<<<LB_CTAS, LB_THREADS, 0, st>>>(gk, sk, yk, xk1, xk, m, rho_slot, out);
}
}
