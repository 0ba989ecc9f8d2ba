// Arithmetic of the diffuse-cluster coherencies (recalculate_diffuse_coherencies,
// diffuse_predict.c:295-586): the shapelet product tensor (host), the product of two 2x2-valued
// shapelet models, and the per-row Fourier-plane value.  Host-callable so that
// oracle/diffuse_math_check.cu runs exactly this code on the CPU against the reference's
// shapelet_product_tensor / shapelet_product_jones / shapelet_contrib_vector (test infrastructure; the
// product runs the products and the rows on the device, kernels_diffuse.cu).
#pragma once
#include <math.h>

#include "coh_math.cuh"

#define DIFFUSE_MAX_ORDER COH_SHAPELET_MAX_N0  // largest L, M, N of a product tensor

#ifdef __CUDA_ARCH__
#define DIFFUSE_UNROLL _Pragma("unroll")
#else
#define DIFFUSE_UNROLL
#endif

// ---- product tensor (shapelet_product_tensor, shapelet.c:640-689; L_mat, :535-626) ----------------
#include <vector>
// B[l*M*N + m + n*M], h = f x g with h: L modes at scale alpha, f: M at beta, g: N at gamma.
// Returns 0, or -1 where the reference's recursion or normalisation leaves the double range (its
// tensor is then inf / nan): the caller refuses such orders.
static inline __host__ int diffuse_product_tensor(int L, int M, int N, double alpha, double beta, double gamma,
                                         double *B) {
  const size_t LMN = (size_t)L * M * N;
  std::vector<double> H(LMN, 0.0);
  std::vector<unsigned char> flag(LMN, 0);
  const double nu = 1.0 / sqrt(1.0 / (alpha * alpha) + 1.0 / (beta * beta) + 1.0 / (gamma * gamma));
  const double a = sqrt(2.0) * nu / alpha, b = sqrt(2.0) * nu / beta, c = sqrt(2.0) * nu / gamma;
  auto at = [&](int l, int m, int n) { return (size_t)l * M * N + (size_t)m * N + n; };
  // L_mat: the recursion in the reference's visiting order, a term counted only once it is set
  for (int l = 0; l < L; l++)
    for (int m = 0; m < M; m++)
      for (int n = 0; n < N; n++) {
        if (!l && !m && !n) { H[at(l, m, n)] = 1.0; flag[at(l, m, n)] = 1; }
        if ((l + m + n) % 2 != 0) { H[at(l, m, n)] = 0.0; flag[at(l, m, n)] = 1; }
        if (n + 1 <= N - 1 && (l + m + n + 1) % 2 == 0) {
          double rhs = 0.0;
          if (n - 1 >= 0 && flag[at(l, m, n - 1)]) rhs += ((double)2 * n) * (c * c - 1.0) * H[at(l, m, n - 1)];
          if (l - 1 >= 0 && flag[at(l - 1, m, n)]) rhs += ((double)2 * l) * (c * a) * H[at(l - 1, m, n)];
          if (m - 1 >= 0 && flag[at(l, m - 1, n)]) rhs += ((double)2 * m) * (c * b) * H[at(l, m - 1, n)];
          if (rhs != 0.0) { H[at(l, m, n + 1)] = rhs; flag[at(l, m, n + 1)] = 1; }
        }
        if (m + 1 <= M - 1 && (l + m + 1 + n) % 2 == 0) {
          double rhs = 0.0;
          if (m - 1 >= 0 && flag[at(l, m - 1, n)]) rhs += ((double)2 * m) * (b * b - 1.0) * H[at(l, m - 1, n)];
          if (n - 1 >= 0 && flag[at(l, m, n - 1)]) rhs += ((double)2 * n) * (b * c) * H[at(l, m, n - 1)];
          if (l - 1 >= 0 && flag[at(l - 1, m, n)]) rhs += ((double)2 * l) * (b * a) * H[at(l - 1, m, n)];
          if (rhs != 0.0) { H[at(l, m + 1, n)] = rhs; flag[at(l, m + 1, n)] = 1; }
        }
        if (l + 1 <= L - 1 && (l + 1 + m + n) % 2 == 0) {
          double rhs = 0.0;
          if (l - 1 >= 0 && flag[at(l - 1, m, n)]) rhs += ((double)2 * l) * (a * a - 1.0) * H[at(l - 1, m, n)];
          if (m - 1 >= 0 && flag[at(l, m - 1, n)]) rhs += ((double)2 * m) * (a * b) * H[at(l, m - 1, n)];
          if (n - 1 >= 0 && flag[at(l, m, n - 1)]) rhs += ((double)2 * n) * (a * c) * H[at(l, m, n - 1)];
          if (rhs != 0.0) { H[at(l + 1, m, n)] = rhs; flag[at(l + 1, m, n)] = 1; }
        }
      }
  const int n0 = L > M ? (L > N ? L : N) : (M > N ? M : N);
  std::vector<double> fact(n0);
  fact[0] = 1.0;
  for (int i = 1; i < n0; i++) fact[i] = (double)i * fact[i - 1];
  for (int l = 0; l < L; l++)
    for (int m = 0; m < M; m++)
      for (int n = 0; n < N; n++) {
        double v = 0.0;
        // shapelet.c:672 with its parentheses: the square root closes after gamma, so H is divided
        // by sqrt(2^(l+m+n) sqrt(pi) l! m! n! alpha beta gamma) in the product's order
        if ((l + m + n) % 2 == 0)
          v = nu * (H[at(l, m, n)] / sqrt((double)(pow(2.0, (double)(l + m + n))) * sqrt(M_PI) *
                                          fact[l] * fact[m] * fact[n] * alpha * beta * gamma));
        B[(size_t)l * M * N + m + (size_t)n * M] = v;
      }
  // rescaled by (L M N)^(1/8) / ||B||_2 (:681-683); the 2-norm accumulates in extended precision
  long double ss = 0.0L;
  for (size_t i = 0; i < LMN; i++) {
    if (!isfinite(B[i])) return -1;
    ss += (long double)B[i] * (long double)B[i];
  }
  const double Bnorm = (double)sqrtl(ss);
  if (!(Bnorm > 0.0) || !isfinite(Bnorm)) return -1;
  const double sc = pow((double)L * M * N, 0.125) / Bnorm;
  for (size_t i = 0; i < LMN; i++) B[i] *= sc;
  return 0;
}

// ---- product of two 2x2-valued shapelet models (shapelet_product_jones, shapelet.c:864-957) -------
// h(l1,l2) = sum_{i,j,i',j'} C[l2][i,j] C[l1][i',j'] F[i,i'] G[j,j'], the reference's Kronecker sum
// (:921-944) regrouped as sum_{i,j} C[l2][i,j] U[i][j], U[i][j] = sum_j' T[i][j'] G[j,j'],
// T[i][j'] = sum_i' C[l1][i',j'] F[i,i'].  C[l][i,j] = Cf[l*M*N + i + j*M]; F[i,i'] = f[i*M + i'],
// G[j,j'] = g[j*N + j'] are 2x2 modes (4 complex, row major), f on the left; herm: G^H for G.
// T and U are [M][N][4]; h[(l1 + l2*L)*4 + c].

// T[i][j'] of output mode l1
__host__ __device__ __forceinline__ void diffuse_T(const double *Cf, int M, int N, int l1, const double2 *f,
                                          int i, int jp, double2 *t) {
  const double *Cl1 = Cf + (size_t)l1 * M * N + (size_t)jp * M;
DIFFUSE_UNROLL
  for (int c = 0; c < 4; c++) t[c] = make_double2(0.0, 0.0);
  for (int ip = 0; ip < M; ip++) {
    const double cc = Cl1[ip];
    const double2 *F = f + 4 * ((size_t)i * M + ip);
DIFFUSE_UNROLL
    for (int c = 0; c < 4; c++) {
      t[c].x = fma(cc, F[c].x, t[c].x);
      t[c].y = fma(cc, F[c].y, t[c].y);
    }
  }
}
// component c = (r, s) of U[i][j] from the row T[i][0..N): sum_j' (T G)_rs, or (T G^H)_rs
__host__ __device__ __forceinline__ double2 diffuse_U(const double2 *Ti, int N, const double2 *g, int j,
                                             int herm, int c) {
  const int r = c >> 1, s = c & 1;
  double2 u = make_double2(0.0, 0.0);
  for (int jp = 0; jp < N; jp++) {
    const double2 *T = Ti + 4 * jp;
    const double2 *G = g + 4 * ((size_t)j * N + jp);
    if (herm) {  // (ambt, shapelet.c:841-846)
      cfmac(u, T[2 * r], G[2 * s]);
      cfmac(u, T[2 * r + 1], G[2 * s + 1]);
    } else {     // (amb, :830-835)
      cfma(u, T[2 * r], G[s]);
      cfma(u, T[2 * r + 1], G[2 + s]);
    }
  }
  return u;
}
// component c of h(l1, l2) from U of l1
__host__ __device__ __forceinline__ double2 diffuse_H(const double *Cf, int M, int N, int l2, const double2 *U,
                                             int c) {
  const double *Cl2 = Cf + (size_t)l2 * M * N;
  double2 s = make_double2(0.0, 0.0);
  for (int i = 0; i < M; i++)
    for (int j = 0; j < N; j++) {
      const double cc = Cl2[i + j * M];
      const double2 v = U[4 * ((size_t)i * N + j) + c];
      s.x = fma(cc, v.x, s.x);
      s.y = fma(cc, v.y, s.y);
    }
  return s;
}

// the whole product on the host; T and U hold 4*M*N complex each
static inline __host__ void diffuse_product_host(int L, int M, int N, const double *Cf, const double2 *f,
                                        const double2 *g, int herm, double2 *h, double2 *T, double2 *U) {
  for (int l1 = 0; l1 < L; l1++) {
    for (int i = 0; i < M; i++)
      for (int jp = 0; jp < N; jp++) diffuse_T(Cf, M, N, l1, f, i, jp, T + 4 * ((size_t)i * N + jp));
    for (int i = 0; i < M; i++)
      for (int j = 0; j < N; j++)
        for (int c = 0; c < 4; c++) U[4 * ((size_t)i * N + j) + c] = diffuse_U(T + 4 * (size_t)i * N, N, g, j, herm, c);
    for (int l2 = 0; l2 < L; l2++)
      for (int c = 0; c < 4; c++) h[((size_t)l1 + (size_t)l2 * L) * 4 + c] = diffuse_H(Cf, M, N, l2, U, c);
  }
}

// ---- one row ------------------------------------------------------------------------------------
// Fourier-plane value of a 2x2-valued model of n0 x n0 modes at (uf, vf) (shapelet_contrib_vector,
// shapelet.c:199-232): 2 pi sum_modes modes[mode] coeff(mode), coeff from
// calculate_uv_mode_vectors_scalar(-uf, vf, beta, n0), odd n1+n2 imaginary.  No eX / eY / eP and no
// projection.
__host__ __device__ __forceinline__ void diffuse_contrib(const double2 *modes, int n0, double beta, double uf,
                                                double vf, double2 *coh) {
  double bu[DIFFUSE_MAX_ORDER], bv[DIFFUSE_MAX_ORDER];
  shapelet_basis(-uf * beta, n0, bu);
  shapelet_basis(vf * beta, n0, bv);
DIFFUSE_UNROLL
  for (int c = 0; c < 4; c++) coh[c] = make_double2(0.0, 0.0);
  for (int n2 = 0; n2 < n0; n2++)
    for (int n1 = 0; n1 < n0; n1++) {
      int odd;
      const double av = shapelet_mode_coeff(bu, bv, n1, n2, &odd);
      const double2 *m = modes + 4 * (n2 * n0 + n1);
DIFFUSE_UNROLL
      for (int c = 0; c < 4; c++) {
        if (odd) {  // m * (i av)
          coh[c].x -= m[c].y * av;
          coh[c].y += m[c].x * av;
        } else {
          coh[c].x += m[c].x * av;
          coh[c].y += m[c].y * av;
        }
      }
    }
DIFFUSE_UNROLL
  for (int c = 0; c < 4; c++) coh[c] = make_double2(2.0 * M_PI * coh[c].x, 2.0 * M_PI * coh[c].y);
}

// phase and |sinc| smearing of a source at (ll, mm, nn) on row (u, v, w) (diffuse_predict.c:86-104):
// the point-source term of source_phase
__host__ __device__ __forceinline__ double2 diffuse_phase(double ll, double mm, double nn, double u, double v,
                                                 double w, double freq0, double fdelta2) {
  DevSource s{};
  s.ll = ll; s.mm = mm; s.nn = nn; s.stype = (double)STYPE_POINT_;
  return source_phase(s, nullptr, u, v, w, freq0, fdelta2);
}
