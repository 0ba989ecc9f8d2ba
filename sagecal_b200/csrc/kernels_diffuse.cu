// Coherencies of the diffuse cluster from a spatial model Z (recalculate_diffuse_coherencies,
// diffuse_predict.c:295-586), every source in the reference's order:
//
//   k_diffuse_station  one CTA per (station q, source): C_Jq[q] = s_coh x Z_q^H, 4 n0^2 complex modes
//                      (shapelet_prod_one_threadfn, :259-271)
//   k_diffuse_predict  one CTA per baseline (p, q): the pair's modes H_pq = Z_p x C_Jq[q] formed in
//                      shared memory (64 KB at n0 = 32; the pair array of all baselines is never
//                      stored), then one warp per row of the baseline: 2 pi sum_modes H coeff(mode),
//                      times the phase and smearing of the source (:72-126, :274-288).  The first
//                      source replaces the row's value, the others add to it.
//
// The products use the separable form of diffuse_math.cuh: O(n0^3 sh) per pair instead of the
// reference's O(n0^4 sh^2) Kronecker sum.  Everything is fp64.
#include "internal.cuh"
#include "coh.h"
#include "diffuse_math.cuh"
#include "problem.h"

#define DIFFUSE_THREADS 256
#define DIFFUSE_WARPS (DIFFUSE_THREADS / 32)

// h = f x g (g^H if herm) by the whole CTA; T, U: [M][N][4] in shared memory.  PLANAR: h[c][l1 + l2 L]
// instead of h[(l1 + l2 L) 4 + c] (the row loop then reads consecutive modes per lane).
template <bool PLANAR>
__device__ void product_cta(int L, int M, int N, const double *Cf, const double2 *f, const double2 *g,
                            int herm, double2 *h, double2 *T, double2 *U) {
  const int MN = M * N;
  for (int l1 = 0; l1 < L; l1++) {
    for (int k = threadIdx.x; k < MN; k += DIFFUSE_THREADS) {
      const int i = k / N, jp = k - i * N;
      diffuse_T(Cf, M, N, l1, f, i, jp, T + 4 * k);
    }
    __syncthreads();
    for (int k = threadIdx.x; k < 4 * MN; k += DIFFUSE_THREADS) {
      const int ij = k >> 2, c = k & 3;
      const int i = ij / N, j = ij - i * N;
      U[k] = diffuse_U(T + 4 * i * N, N, g, j, herm, c);
    }
    __syncthreads();  // (T of l1 + 1 is written after this; U of l1 + 1 after the next barrier)
    for (int k = threadIdx.x; k < 4 * L; k += DIFFUSE_THREADS) {
      const int l2 = k >> 2, c = k & 3;
      const double2 v = diffuse_H(Cf, M, N, l2, U, c);
      if (PLANAR) h[(size_t)c * L * L + l1 + l2 * L] = v;
      else h[((size_t)l1 + (size_t)l2 * L) * 4 + c] = v;
    }
  }
  __syncthreads();
}

__global__ void __launch_bounds__(DIFFUSE_THREADS) k_diffuse_station(DiffuseArgs a) {
  extern __shared__ __align__(16) double2 dsm[];
  const int q = blockIdx.x;
  const DiffuseSource s = a.src[blockIdx.y];
  const int n0 = s.n0, G = a.sh * a.sh;
  double2 *T = dsm, *U = dsm + 4 * n0 * a.sh;
  product_cta<false>(n0, n0, a.sh, a.cf + s.cf1, a.scoh + s.scoh, a.Zt + (size_t)4 * G * q, 1,
                     a.cjq + s.cjq + (size_t)4 * n0 * n0 * q, T, U);
}

__global__ void __launch_bounds__(DIFFUSE_THREADS) k_diffuse_predict(DiffuseArgs a) {
  extern __shared__ __align__(16) double2 dsm[];
  __shared__ double bu[DIFFUSE_WARPS][DIFFUSE_MAX_ORDER], bv[DIFFUSE_WARPS][DIFFUSE_MAX_ORDER];
  const int b = blockIdx.x;
  const int p = a.pairs[b].x, q = a.pairs[b].y;
  const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  const long long r0 = a.rows ? a.row_off[b] : 0;
  const int nrows = a.rows ? (int)(a.row_off[b + 1] - r0) : a.ntime;
  // (the reference forms the pair products for p <= q only; rows of other pairs read zeros, :490)
  const bool have = p >= 0 && q < a.N && p <= q;
  const int G = a.sh * a.sh;
  for (int si = 0; si < a.ns; si++) {
    const DiffuseSource s = a.src[si];
    const int n0 = s.n0, nm = n0 * n0;
    double2 *H = dsm, *T = dsm + 4 * nm, *U = T + 4 * a.sh * n0;
    if (have) {
      product_cta<true>(n0, a.sh, n0, a.cf + s.cf2, a.Zt + (size_t)4 * G * p,
                        a.cjq + s.cjq + (size_t)4 * nm * q, 0, H, T, U);
    } else {
      for (int k = threadIdx.x; k < 4 * nm; k += DIFFUSE_THREADS) H[k] = make_double2(0.0, 0.0);
      __syncthreads();
    }
    for (int k = wp; k < nrows; k += DIFFUSE_WARPS) {
      const long long r = a.rows ? a.rows[r0 + k] : b + (long long)k * a.Nbase;
      const double u = a.u[r], v = a.v[r], w = a.w[r];
      if (lane < 2) shapelet_basis(lane == 0 ? -u * a.freq0 * s.beta : v * a.freq0 * s.beta, n0,
                                   lane == 0 ? bu[wp] : bv[wp]);
      __syncwarp();
      double2 acc[4];
#pragma unroll
      for (int c = 0; c < 4; c++) acc[c] = make_double2(0.0, 0.0);
      for (int ci = lane; ci < nm; ci += 32) {
        const int n2 = ci / n0, n1 = ci - n2 * n0;
        int odd;
        const double av = shapelet_mode_coeff(bu[wp], bv[wp], n1, n2, &odd);
#pragma unroll
        for (int c = 0; c < 4; c++) {
          const double2 m = H[(size_t)c * nm + ci];
          if (odd) {
            acc[c].x = fma(-m.y, av, acc[c].x);
            acc[c].y = fma(m.x, av, acc[c].y);
          } else {
            acc[c].x = fma(m.x, av, acc[c].x);
            acc[c].y = fma(m.y, av, acc[c].y);
          }
        }
      }
#pragma unroll
      for (int c = 0; c < 4; c++) {
        acc[c].x = warp_sum(acc[c].x);
        acc[c].y = warp_sum(acc[c].y);
      }
      __syncwarp();  // bu / bv of this row are read by every lane before the next row writes them
      if (lane < 4) {
        double2 cv = acc[0];
#pragma unroll
        for (int c = 1; c < 4; c++)
          if (lane == c) cv = acc[c];
        cv = make_double2(2.0 * M_PI * cv.x, 2.0 * M_PI * cv.y);
        const double2 ph = diffuse_phase(s.ll, s.mm, s.nn, u, v, w, a.freq0, a.fdelta2);
        cv = cmul(cv, ph);
        double2 *o = a.coh + (long long)lane * a.R + r;
        *o = si == 0 ? cv : cadd(*o, cv);
      }
    }
    __syncthreads();  // H, T and U are rewritten for the next source
  }
}

static size_t station_smem(int n0, int sh) { return sizeof(double2) * 8 * (size_t)n0 * sh; }
static size_t predict_smem(int n0, int sh) {
  return sizeof(double2) * (4 * (size_t)n0 * n0 + 8 * (size_t)n0 * sh);
}

extern "C" void db_launch_diffuse(const DiffuseArgs *a, int max_n0, cudaStream_t st) {
  const size_t s1 = station_smem(max_n0, a->sh), s2 = predict_smem(max_n0, a->sh);
  DB_CHECK(cudaFuncSetAttribute(k_diffuse_station, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)s1));
  DB_CHECK(cudaFuncSetAttribute(k_diffuse_predict, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)s2));
  k_diffuse_station<<<dim3(a->N, a->ns), DIFFUSE_THREADS, s1, st>>>(*a);
  db_count_launch(1);
  // algorithmic bytes: u, v, w read and the cluster's 4 complex written once per row and source
  db_prof_begin(12, (double)a->R * a->ns * (24.0 + 64.0), st);
  k_diffuse_predict<<<a->npairs, DIFFUSE_THREADS, s2, st>>>(*a);
  db_prof_end(st);
  db_count_launch(1);
}
