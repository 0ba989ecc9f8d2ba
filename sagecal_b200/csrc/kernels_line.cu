// Line-search support for the LBFGS stage.
//
// The reference evaluates the cost ~10-30 times per LBFGS iteration, each a full predict over all
// clusters (linesearch / linesearch_zoom / cubic_interp, lbfgs.c:116-430 calling cost_func,
// robust_lbfgs.c:674-726).  Every one of those evaluations is at a point x_k + alpha p_k, and along
// that line the model of a row is a quadratic polynomial in alpha,
//     (J_p + a D_p) C (J_q + a D_q)^H = V0 + a V1 + a^2 V2 ,
// so the residual is e(a) = E0 - a E1 - a^2 E2 with
//     E0 = x - sum_k Jp C Jq^H,  E1 = sum_k (Dp C Jq^H + Jp C Dq^H),  E2 = sum_k Dp C Dq^H .
// k_stream_all<1> (kernels_tma.cu) makes ONE pass over the coherencies and leaves E0,E1,E2 (3 x 64 B
// per row) in HBM/L2; k_line_eval then gives the Gaussian or Student's-t cost at any alpha from
// those 192 B per row (14.5 MB per vector at C2: L2 resident), and k_line_residual the residual at
// the accepted step for the gradient pass.  Same arithmetic function of alpha as the reference, 30x less HBM traffic.
#include "internal.cuh"

__device__ __forceinline__ void grid_reduce_sum_l(double v, double *partials, double *out,
                                                  unsigned int *counter) {
  __shared__ double wsum[32];
  __shared__ bool is_last;
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) wsum[w] = v;
  __syncthreads();
  const unsigned int nblocks = gridDim.x * gridDim.y;
  const unsigned int bid = blockIdx.x + gridDim.x * blockIdx.y;
  if (threadIdx.x == 0) {
    double s = 0.0;
    const int nw = (blockDim.x + 31) >> 5;
    for (int i = 0; i < nw; i++) s += wsum[i];
    partials[bid] = s;
    __threadfence();
    is_last = (atomicAdd(counter, 1u) == nblocks - 1);
  }
  __syncthreads();
  if (is_last) {
    double s = 0.0;
    for (unsigned int i = threadIdx.x; i < nblocks; i += blockDim.x)
      s += ((volatile double *)partials)[i];
    s = warp_sum(s);
    __syncthreads();
    if (lane == 0) wsum[w] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
      double tot = 0.0;
      const int nw = (blockDim.x + 31) >> 5;
      for (int i = 0; i < nw; i++) tot += wsum[i];
      *out = tot;
      *counter = 0;
    }
  }
}

// cost(alpha) from E0,E1,E2; mode 1: sum e^2, mode 2: sum log(1 + e^2/nu)
__global__ void __launch_bounds__(256)
k_line_eval(const double2 *__restrict__ E0, const double2 *__restrict__ E1,
            const double2 *__restrict__ E2, long long n4, double alpha, int mode, double inv_nu,
            double *partials, double *out, unsigned int *counter) {
  const double a2 = alpha * alpha;
  double s = 0.0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    const double2 e0 = E0[i], e1 = E1[i], e2 = E2[i];
    const double ex = (e0.x - alpha * e1.x) - a2 * e2.x;
    const double ey = (e0.y - alpha * e1.y) - a2 * e2.y;
    if (mode == 1) {
      s = fma(ex, ex, s);
      s = fma(ey, ey, s);
    } else {
      s += log(1.0 + ex * ex * inv_nu);
      s += log(1.0 + ey * ey * inv_nu);
    }
  }
  grid_reduce_sum_l(s, partials, out, counter);
}

// the five sums c[] of every thread of a 256-thread grid -> out[0..4] (per-CTA partials, fixed-order
// final sum), with c1 = -2 sum E0.E1 and c3 = 2 sum E1.E2
__device__ __forceinline__ void poly_grid_reduce(const double *c, double *partials, double *out,
                                                 unsigned int *counter) {
  __shared__ double ws[5][8];
  __shared__ bool is_last;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int j = 0; j < 5; j++) {
    const double v = warp_sum(c[j]);
    if (lane == 0) ws[j][w] = v;
  }
  __syncthreads();
  if (threadIdx.x < 5) {
    double s = 0.0;
    for (int i = 0; i < 8; i++) s += ws[threadIdx.x][i];
    partials[(size_t)blockIdx.x * 5 + threadIdx.x] = s;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = (atomicAdd(counter, 1u) == gridDim.x - 1);
  __syncthreads();
  if (is_last && threadIdx.x < 5) {
    double s = 0.0;
    for (unsigned int b = 0; b < gridDim.x; b++)
      s += ((volatile double *)partials)[(size_t)b * 5 + threadIdx.x];
    // c1 = -2 sum E0.E1, c3 = 2 sum E1.E2
    if (threadIdx.x == 1) s *= -2.0;
    if (threadIdx.x == 3) s *= 2.0;
    out[threadIdx.x] = s;
    if (threadIdx.x == 0) *counter = 0;
  }
}

// Gaussian cost along the line is the quartic sum |E0 - a E1 - a^2 E2|^2 = c0 + c1 a + ... + c4 a^4:
// the five coefficients in one deterministic reduction.  Sharded runs form E0 only after the sum over
// the ranks, so they take this pass; one GPU folds the sums into k_stream_all<1> (k_line_poly_finish)
__global__ void __launch_bounds__(256)
k_line_poly(const double2 *__restrict__ E0, const double2 *__restrict__ E1,
            const double2 *__restrict__ E2, long long n4, double *partials, double *out,
            unsigned int *counter) {
  double c[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    const double2 e0 = E0[i], e1 = E1[i], e2 = E2[i];
    c[0] = fma(e0.x, e0.x, fma(e0.y, e0.y, c[0]));
    c[1] = fma(e0.x, e1.x, fma(e0.y, e1.y, c[1]));
    c[2] = fma(e1.x, e1.x, fma(e1.y, e1.y, c[2]));
    c[2] = fma(-2.0 * e0.x, e2.x, fma(-2.0 * e0.y, e2.y, c[2]));
    c[3] = fma(e1.x, e2.x, fma(e1.y, e2.y, c[3]));
    c[4] = fma(e2.x, e2.x, fma(e2.y, e2.y, c[4]));
  }
  poly_grid_reduce(c, partials, out, counter);
}

// the quartic from the per-CTA sums k_stream_all<1> left in part ([5][nparts]): 40 B per CTA of the
// line-model pass instead of a second read of E0, E1 and E2
__global__ void __launch_bounds__(256)
k_line_poly_finish(const double *__restrict__ part, unsigned nparts, double *partials, double *out,
                   unsigned int *counter) {
  double c[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < nparts; i += gridDim.x * blockDim.x)
#pragma unroll
    for (int j = 0; j < 5; j++) c[j] += part[(size_t)j * nparts + i];
  poly_grid_reduce(c, partials, out, counter);
}

// out = sum |v|^2 over n4 double2 (the cost of a residual already in HBM)
__global__ void __launch_bounds__(256)
k_sumsq(const double2 *__restrict__ v, long long n4, double *partials, double *out,
        unsigned int *counter) {
  double s = 0.0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    const double2 e = v[i];
    s = fma(e.x, e.x, s);
    s = fma(e.y, e.y, s);
  }
  grid_reduce_sum_l(s, partials, out, counter);
}

// res = E0 - alpha E1 - alpha^2 E2
__global__ void __launch_bounds__(256)
k_line_residual(const double2 *__restrict__ E0, const double2 *__restrict__ E1,
                const double2 *__restrict__ E2, double2 *__restrict__ res, long long n4,
                double alpha) {
  const double a2 = alpha * alpha;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    const double2 e0 = E0[i], e1 = E1[i], e2 = E2[i];
    res[i] = make_double2((e0.x - alpha * e1.x) - a2 * e2.x, (e0.y - alpha * e1.y) - a2 * e2.y);
  }
}

// sharded runs: out = x - pm (pm = all-reduced partial models); cost like k_stream_all<0>
__global__ void __launch_bounds__(256)
k_residual_cost(const double2 *__restrict__ x, const double2 *__restrict__ pm,
                double2 *__restrict__ out, long long n4, int out_mode, int cost_mode, double inv_nu,
                double *partials, double *cost, unsigned int *counter) {
  double s = 0.0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    const double2 xv = x[i], m = pm[i];
    const double2 e = make_double2(xv.x - m.x, xv.y - m.y);
    if (out_mode == 1) out[i] = e;
    if (out_mode == 2) out[i] = m;
    if (cost_mode == 1) {
      s = fma(e.x, e.x, s);
      s = fma(e.y, e.y, s);
    } else if (cost_mode == 2) {
      s += log(1.0 + e.x * e.x * inv_nu);
      s += log(1.0 + e.y * e.y * inv_nu);
    }
  }
  if (cost_mode) grid_reduce_sum_l(s, partials, cost, counter);
}

// y = a*x + b*y elementwise over n4 double2
__global__ void __launch_bounds__(256)
k_axpby(const double2 *__restrict__ x, double2 *__restrict__ y, long long n4, double a, double b) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    const double2 xv = x[i], yv = y[i];
    y[i] = make_double2(a * xv.x + b * yv.x, a * xv.y + b * yv.y);
  }
}

// out = beta*in + model_k (sign > 0) or in - model_k + (1-beta)*in2 (sign < 0) for ONE cluster whose
// hybrid chunk of a row is the ROW-based map px = row / ceil(R/nchunk) of mylm_fit_single_pth
// (lmfit.c:86): the hidden-data add / subtract of lmfit.c:890-891,980-981 when nchunk does not divide
// tilesz, i.e. when that map differs from the timeslot ranges the per-chunk LM fits run over.
// in2 and out may be the same vector (the sharded subtract updates r in place): neither is __restrict__.
__global__ void __launch_bounds__(256)
k_cluster_rowmap(const double2 *__restrict__ coh_k, const double2 *__restrict__ in,
                 const double2 *in2, double2 *out,
                 const unsigned char *__restrict__ flag, const double *__restrict__ pp,
                 const int *__restrict__ chunk_poff, int nchunk, const short2 *__restrict__ blpq,
                 long long R, int Nbase, int sign, double beta) {
  for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < R;
       r += (long long)gridDim.x * blockDim.x) {
    const short2 pq = blpq[r % Nbase];
    const int off = chunk_poff[row_chunk(r, R, nchunk)];
    double2 Jp[4], Jq[4], C[4], A[4], m[4];
    load_jones(pp + off, pq.x, Jp);
    load_jones(pp + off, pq.y, Jq);
#pragma unroll
    for (int c = 0; c < 4; c++) C[c] = coh_k[(long long)c * R + r];
    mat_ab(Jp, C, A);
    mat_abh(A, Jq, m);
    const bool fl = flag[r] != 0;
#pragma unroll
    for (int c = 0; c < 4; c++) {
      const long long ix = (long long)c * R + r;
      const double2 mm = fl ? make_double2(0.0, 0.0) : m[c];
      const double2 v = in[ix];
      double2 o;
      if (sign > 0) {
        o = make_double2(beta * v.x + mm.x, beta * v.y + mm.y);
      } else {
        o = make_double2(v.x - mm.x, v.y - mm.y);
        if (in2) {
          const double2 w = in2[ix];
          o.x += (1.0 - beta) * w.x;
          o.y += (1.0 - beta) * w.y;
        }
      }
      out[ix] = o;
    }
  }
}

extern "C" {
#define LINE_GRID 592
void db_launch_line_eval(const double2 *E0, const double2 *E1, const double2 *E2, long long n4,
                         double alpha, int mode, double inv_nu, double *partials, double *out,
                         unsigned int *counter, cudaStream_t st) {
  k_line_eval<<<LINE_GRID, 256, 0, st>>>(E0, E1, E2, n4, alpha, mode, inv_nu, partials, out,
                                         counter);
}
void db_launch_residual_cost(const double2 *x, const double2 *pm, double2 *out, long long n4,
                             int out_mode, int cost_mode, double inv_nu, double *partials,
                             double *cost, unsigned int *counter, cudaStream_t st) {
  k_residual_cost<<<592, 256, 0, st>>>(x, pm, out, n4, out_mode, cost_mode, inv_nu, partials, cost,
                                       counter);
}
void db_launch_axpby(const double2 *x, double2 *y, long long n4, double a, double b,
                     cudaStream_t st) {
  k_axpby<<<592, 256, 0, st>>>(x, y, n4, a, b);
}
void db_launch_cluster_rowmap(const double2 *coh_k, const double2 *in, const double2 *in2,
                               double2 *out, const unsigned char *flag, const double *pp,
                               const int *chunk_poff, int nchunk, const short2 *blpq, long long R,
                               int Nbase, int sign, double beta, cudaStream_t st) {
  k_cluster_rowmap<<<592, 256, 0, st>>>(coh_k, in, in2, out, flag, pp, chunk_poff, nchunk, blpq, R,
                                        Nbase, sign, beta);
}
void db_launch_line_poly(const double2 *E0, const double2 *E1, const double2 *E2, long long n4,
                         double *partials, double *out, unsigned int *counter, cudaStream_t st) {
  k_line_poly<<<192, 256, 0, st>>>(E0, E1, E2, n4, partials, out, counter);
}
void db_launch_line_poly_finish(const double *part, unsigned nparts, double *partials, double *out,
                                unsigned int *counter, cudaStream_t st) {
  k_line_poly_finish<<<192, 256, 0, st>>>(part, nparts, partials, out, counter);
}
void db_launch_sumsq(const double2 *v, long long n4, double *partials, double *out,
                     unsigned int *counter, cudaStream_t st) {
  k_sumsq<<<LINE_GRID, 256, 0, st>>>(v, n4, partials, out, counter);
}
void db_launch_line_residual(const double2 *E0, const double2 *E1, const double2 *E2, double2 *res,
                             long long n4, double alpha, cudaStream_t st) {
  k_line_residual<<<LINE_GRID, 256, 0, st>>>(E0, E1, E2, res, n4, alpha);
}
}
