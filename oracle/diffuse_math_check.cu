// TEST INFRASTRUCTURE ONLY (oracle).  Runs the arithmetic of the product's diffuse-cluster kernels
// (sagecal_b200/csrc/diffuse_math.cuh: product tensor, product of two 2x2-valued shapelet models, row
// value) on the CPU, so that tests/test_oracle_diffuse_math.py can pin it against the compiled
// reference's shapelet_product_tensor, shapelet_product_jones, shapelet_contrib_vector and
// recalculate_diffuse_coherencies without a GPU.  Compiled by nvcc as host code; nothing is launched.
#include <vector>

#include "../sagecal_b200/csrc/diffuse_math.cuh"

extern "C" int check_tensor(int L, int M, int N, double alpha, double beta, double gamma, double *B) {
  return diffuse_product_tensor(L, M, N, alpha, beta, gamma, B);
}

// h (L*L*4 complex) = f (M*M*4) x g (N*N*4), or f x g^H, with the tensor Cf given
extern "C" void check_product(int L, int M, int N, const double *Cf, const double *f, const double *g,
                              int herm, double *h) {
  std::vector<double2> T((size_t)4 * M * N), U((size_t)4 * M * N);
  diffuse_product_host(L, M, N, Cf, reinterpret_cast<const double2 *>(f),
                       reinterpret_cast<const double2 *>(g), herm, reinterpret_cast<double2 *>(h),
                       T.data(), U.data());
}

extern "C" void check_contrib(const double *modes, int n0, double beta, double uf, double vf,
                              double *coh) {
  diffuse_contrib(reinterpret_cast<const double2 *>(modes), n0, beta, uf, vf,
                  reinterpret_cast<double2 *>(coh));
}

// the whole computation of recalculate_diffuse_coherencies for one cluster, in the reference's order
// (diffuse_predict.c:371-572) on this header's arithmetic.  Sources: n0[s], beta[s], lmn[3s..],
// iquv[4s..], modes back to back.  Z: 2N x 2G complex, column major.  out: [R][4] complex, written by
// the first source and accumulated by the others.  Returns -1 where a tensor leaves the double range.
extern "C" int check_pipeline(int N, long long R, const int *sta1, const int *sta2, const double *u,
                              const double *v, const double *w, double freq0, double fdelta, int ns,
                              const int *n0s, const double *betas, const double *lmn,
                              const double *iquv, const double *modes, int sh, double sh_beta,
                              const double *Zin, double *out) {
  const int G = sh * sh;
  const double2 *Z = reinterpret_cast<const double2 *>(Zin);
  double2 *X = reinterpret_cast<double2 *>(out);
  std::vector<double2> Zt((size_t)4 * G * N);
  for (int n = 0; n < N; n++)
    for (int g = 0; g < G; g++)
      for (int c = 0; c < 4; c++)
        Zt[((size_t)n * G + g) * 4 + c] = Z[(size_t)(2 * n + (c & 1)) + (size_t)(2 * g + (c >> 1)) * 2 * N];
  const double *md = modes;
  for (int s = 0; s < ns; s++) {
    const int n0 = n0s[s], nm = n0 * n0;
    const double bimg = betas[s] / (2.0 * M_PI);
    const double *q = iquv + 4 * s;
    const double2 xxyy[4] = {make_double2(q[0] + q[1], 0.0), make_double2(q[2], q[3]),
                             make_double2(q[2], -q[3]), make_double2(q[0] - q[1], 0.0)};
    std::vector<double2> scoh((size_t)4 * nm);
    for (int m = 0; m < nm; m++)
      for (int k = 0; k < 4; k++) scoh[4 * m + k] = make_double2(xxyy[k].x * md[m], xxyy[k].y * md[m]);
    md += nm;
    std::vector<double> cf1((size_t)nm * sh), cf2((size_t)n0 * sh * n0);
    if (diffuse_product_tensor(n0, n0, sh, bimg, bimg, sh_beta, cf1.data())) return -1;
    if (diffuse_product_tensor(n0, sh, n0, bimg, sh_beta, bimg, cf2.data())) return -1;
    const int mx = n0 > sh ? n0 : sh;
    std::vector<double2> T((size_t)4 * mx * mx), U((size_t)4 * mx * mx);
    std::vector<double2> cjq((size_t)4 * nm * N);
    for (int n = 0; n < N; n++)
      diffuse_product_host(n0, n0, sh, cf1.data(), scoh.data(), Zt.data() + (size_t)4 * G * n, 1,
                           cjq.data() + (size_t)4 * nm * n, T.data(), U.data());
    std::vector<double2> H((size_t)4 * nm);
    for (long long r = 0; r < R; r++) {
      const int p = sta1[r], qq = sta2[r];
      double2 coh[4] = {make_double2(0, 0), make_double2(0, 0), make_double2(0, 0), make_double2(0, 0)};
      if (p <= qq) {  // (pair products exist for p <= q only, :498-503)
        diffuse_product_host(n0, sh, n0, cf2.data(), Zt.data() + (size_t)4 * G * p,
                             cjq.data() + (size_t)4 * nm * qq, 0, H.data(), T.data(), U.data());
        diffuse_contrib(H.data(), n0, betas[s], u[r] * freq0, v[r] * freq0, coh);
        const double2 ph = diffuse_phase(lmn[3 * s], lmn[3 * s + 1], lmn[3 * s + 2], u[r], v[r], w[r],
                                         freq0, 0.5 * fdelta);
        for (int c = 0; c < 4; c++) coh[c] = cmul(coh[c], ph);
      }
      for (int c = 0; c < 4; c++) X[4 * r + c] = s == 0 ? coh[c] : cadd(X[4 * r + c], coh[c]);
    }
  }
  return 0;
}
