// TEST INFRASTRUCTURE ONLY (oracle).  Runs the arithmetic of the product's projectback manifold average
// (sagecal_b200/csrc/manifold_math.cuh) on the CPU, step by step as k_manifold_projectback takes it, so
// that tests/test_oracle_manifold_math.py can pin it against the compiled reference's zgesvd-based
// polar factor and calculate_manifold_average_projectback without a GPU.  Compiled by nvcc as host
// code; nothing is launched.
#include <stdlib.h>
#include <vector>

#include "../sagecal_b200/csrc/manifold_math.cuh"

// W = U V^H of the 2x2 complex G, both row-major [00, 01, 10, 11] as interleaved doubles
extern "C" void check_polar(const double *G, double *W) {
  manifold_polar(reinterpret_cast<const double2 *>(G), reinterpret_cast<double2 *>(W));
}

// the whole average on Y [Nf][M][8N] in place; cr [M] (null: 0 for every chunk).  Per chunk: the
// pairwise Grams (summed over the stations in plain order; the kernel sums station groups), the rounds
// on the rotations block by block, then the output station by station.
extern "C" void check_projectback(int N, int M, int Nf, double *Y, int Niter, const int *cr) {
  const int P = Nf * (Nf + 1) / 2;
  const size_t fs = (size_t)4 * N * M;  // block stride in double2
  std::vector<double2> C((size_t)P * 4), R((size_t)Nf * 4), Rn((size_t)Nf * 4);
  double2 *Y2 = reinterpret_cast<double2 *>(Y);
  for (int k = 0; k < M; k++) {
    double2 *Yk = Y2 + (size_t)4 * N * k;
    for (int p = 0; p < P; p++) {
      int f, g;
      manifold_pair(p, Nf, f, g);
      double2 a[4] = {make_double2(0.0, 0.0), make_double2(0.0, 0.0), make_double2(0.0, 0.0),
                      make_double2(0.0, 0.0)};
      for (int i = 0; i < N; i++) manifold_gram_acc(Yk + fs * f + 4 * i, Yk + fs * g + 4 * i, a);
      for (int e = 0; e < 4; e++) C[4 * p + e] = a[e];
    }
    const int c0 = cr ? cr[k] : 0;
    for (int f = 0; f < Nf; f++) manifold_start(C.data(), Nf, f, c0, R.data() + 4 * f);
    for (int it = 0; it < Niter; it++) {
      for (int f = 0; f < Nf; f++) manifold_round(C.data(), Nf, f, R.data(), Rn.data() + 4 * f);
      R = Rn;
    }
    for (int f = 0; f < Nf; f++) manifold_final(C.data(), Nf, f, R.data(), Rn.data() + 4 * f);
    for (int i = 0; i < N; i++) manifold_output(Yk + 4 * i, fs, Nf, R.data(), Rn.data());
  }
}

// the draws of the reference entry point with randomize: rand() % Nf for k = 0..M-1
extern "C" void check_draws(int M, int Nf, int *cr) {
  for (int k = 0; k < M; k++) cr[k] = rand() % Nf;
}
