// The projectback manifold average of the federated stochastic calibration
// (calculate_manifold_average_projectback, manifold_average.c:641-867) on the device.
//
// Y[Nf][Mt][8n]: Nf solutions of Mt chunks, n = N Npoly stations each.  Per chunk k the reference
//   1. projects every block f != cr_k onto block cr_k:   Y_f <- Y_f polar(Y_f^H Y_cr);
//   2. Niter times: J3 = mean_f Y_f, then Y_f <- Y_f polar(Y_f^H J3) for every f;
//   3. forms the fresh mean J3 of the rotated blocks;
//   4. writes J3 polar(J3^H Y_f) into block f, Y_f being the INPUT block (it reloads it).
// Every block stays its input block times a 2x2 unitary R_f, and every Gram it forms is a 2x2 product
// of R's with the pairwise Grams C_fg = Y_f^H Y_g of the input blocks:
//   step 1:  R_cr = I,  R_f = polar(C_f,cr)
//   step 2:  R_f <- R_f polar(R_f^H (sum_g C_fg R_g) / Nf)
//   step 4:  P_f = polar((sum_g R_g^H C_gf) / Nf),  out_f = ((sum_g Y_g R_g) / Nf) P_f
// So k_manifold_projectback reads the chunk twice, whatever Niter is: once for the Grams, once for
// the output, which it writes once.  Each CTA owns one chunk; the Grams are summed over stations in a
// fixed order with no atomics, so the result is the same bit for bit on every run and every rank.
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <atomic>
#include <vector>

#include "../../include/dirac_b200.h"
#include "manifold_math.cuh"
#include "problem.h"

#define MF_THREADS 256
#define MF_TILE_BYTES 32768  // stations of all Nf blocks staged per Gram tile
#define MF_MAX_NF 64         // the pairwise Grams of one chunk must fit in shared memory

struct MfLayout {
  int T;      // stations per tile
  int P;      // pairs f <= g
  int nsg;    // station groups per pair
  int units;  // P * nsg accumulators
  size_t smem;
};

static MfLayout mf_layout(int Nf) {
  MfLayout L;
  L.T = MF_TILE_BYTES / (64 * Nf);
  if (L.T < 1) L.T = 1;
  if (L.T > 64) L.T = 64;
  L.P = Nf * (Nf + 1) / 2;
  L.nsg = L.P >= MF_THREADS ? 1 : MF_THREADS / L.P;
  L.units = L.P * L.nsg;
  // tile [Nf][T][4] | accumulators [units][4], the first P of which end up as C | R [Nf][4] |
  // Rnew [Nf][4]
  L.smem = sizeof(double2) * ((size_t)Nf * L.T * 4 + (size_t)L.units * 4 + (size_t)Nf * 8);
  return L;
}

__global__ void __launch_bounds__(MF_THREADS)
k_manifold_projectback(double *__restrict__ Y, int n, int Mt, int Nf, int Niter,
                       const int *__restrict__ cr, int T, int P, int nsg) {
  extern __shared__ double2 mf_smem[];
  double2 *tile = mf_smem;                       // [Nf][T][4]
  double2 *acc = tile + (size_t)Nf * T * 4;      // [nsg][P][4]
  double2 *C = acc;                              // [P][4], once the station groups are summed
  double2 *R = acc + (size_t)P * nsg * 4;        // [Nf][4]
  double2 *Rn = R + (size_t)Nf * 4;              // [Nf][4]
  const int k = blockIdx.x, tid = threadIdx.x;
  const size_t blk = (size_t)8 * n, fstride = blk * Mt;
  const double2 *Yk = reinterpret_cast<const double2 *>(Y + blk * k);
  const size_t fs2 = fstride / 2;  // block stride in double2
  const int units = P * nsg;

  // ---- pairwise Grams C_fg = sum_i Y_f,i^H Y_g,i, f <= g ----
  for (int u = tid; u < units; u += MF_THREADS)
    for (int e = 0; e < 4; e++) acc[4 * u + e] = make_double2(0.0, 0.0);
  for (int i0 = 0; i0 < n; i0 += T) {
    const int nt = n - i0 < T ? n - i0 : T;
    __syncthreads();
    for (int q = tid; q < Nf * nt * 4; q += MF_THREADS) {
      const int f = q / (nt * 4), r = q - f * nt * 4;
      tile[(size_t)f * T * 4 + r] = Yk[fs2 * f + (size_t)i0 * 4 + r];
    }
    __syncthreads();
    for (int u = tid; u < units; u += MF_THREADS) {
      const int p = u % P, sg = u / P;
      int f, g;
      manifold_pair(p, Nf, f, g);
      double2 a[4] = {make_double2(0.0, 0.0), make_double2(0.0, 0.0), make_double2(0.0, 0.0),
                      make_double2(0.0, 0.0)};
      for (int s = sg; s < nt; s += nsg)
        manifold_gram_acc(tile + ((size_t)f * T + s) * 4, tile + ((size_t)g * T + s) * 4, a);
      for (int e = 0; e < 4; e++) acc[4 * u + e] = cadd(acc[4 * u + e], a[e]);
    }
  }
  __syncthreads();
  for (int p = tid; p < P; p += MF_THREADS) {
    double2 c[4];
    for (int e = 0; e < 4; e++) c[e] = acc[4 * p + e];
    for (int sg = 1; sg < nsg; sg++)
      for (int e = 0; e < 4; e++) c[e] = cadd(c[e], acc[4 * ((size_t)sg * P + p) + e]);
    for (int e = 0; e < 4; e++) C[4 * p + e] = c[e];
  }
  __syncthreads();

  // ---- the Procrustes rounds on the 2x2 rotations, one thread per block ----
  const int c0 = cr ? cr[k] : 0;
  for (int f = tid; f < Nf; f += MF_THREADS) manifold_start(C, Nf, f, c0, R + 4 * f);
  __syncthreads();
  for (int it = 0; it < Niter; it++) {
    for (int f = tid; f < Nf; f += MF_THREADS) manifold_round(C, Nf, f, R, Rn + 4 * f);
    __syncthreads();
    for (int q = tid; q < Nf * 4; q += MF_THREADS) R[q] = Rn[q];
    __syncthreads();
  }
  for (int f = tid; f < Nf; f += MF_THREADS) manifold_final(C, Nf, f, R, Rn + 4 * f);
  __syncthreads();

  // ---- out_f = J3 P_f, one station per thread ----
  double2 *Yw = reinterpret_cast<double2 *>(Y + blk * k);
  for (int i = tid; i < n; i += MF_THREADS) manifold_output(Yw + (size_t)i * 4, fs2, Nf, R, Rn);
}

// Y: device [Nf][Mt][8n]; cr: device [Mt] or null (every chunk projects onto block 0)
int db_manifold_projectback(double *Y, int n, int Mt, int Nf, int Niter, const int *cr,
                            cudaStream_t st) {
  if (Nf > MF_MAX_NF) {
    fprintf(stderr, "dirac_b200: the manifold average takes at most %d solutions, not %d\n",
            MF_MAX_NF, Nf);
    return -1;
  }
  const MfLayout L = mf_layout(Nf);
  // the shared-memory opt-in is per device; two host threads may both make it, which is harmless
  static std::atomic<unsigned long long> attr_set{0};
  int dev = 0;
  DB_CHECK(cudaGetDevice(&dev));
  if (dev >= 64 || !(attr_set.load() >> dev & 1ull)) {
    DB_CHECK(cudaFuncSetAttribute(k_manifold_projectback, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  227 * 1024));
    if (dev < 64) attr_set.fetch_or(1ull << dev);
  }
  db_prof_begin(17, (double)Nf * Mt * 8.0 * n * 8.0 * 3.0, st);
  k_manifold_projectback<<<Mt, MF_THREADS, L.smem, st>>>(Y, n, Mt, Nf, Niter, cr, L.T, L.P, L.nsg);
  db_prof_end(st);
  db_count_launch(1);
  DB_CHECK(cudaGetLastError());
  return 0;
}

static int mf_check(const char *who, int N, int M, int Nf, int Niter) {
  if (N < 1 || M < 1 || Nf < 1 || Niter < 0) {
    fprintf(stderr, "%s: N = %d, M = %d, Nf = %d must be at least 1 and Niter = %d at least 0\n", who,
            N, M, Nf, Niter);
    return -1;
  }
  if (Nf > MF_MAX_NF) {
    fprintf(stderr, "%s: at most %d solutions are averaged, not Nf = %d\n", who, MF_MAX_NF, Nf);
    return -1;
  }
  return 0;
}

// On a device array: Y [Nf][M][8N] device pointer, cr [M] host (null: block 0 for every chunk),
// stream a cudaStream_t or null for the legacy stream.  Returns when the kernel is enqueued.
extern "C" int dirac_b200_manifold_projectback_dev(int N, int M, int Nf, double *Y, int Niter,
                                                   const int *cr, void *stream) {
  if (mf_check("dirac_b200_manifold_projectback_dev", N, M, Nf, Niter)) return -1;
  require_gpu();
  cudaStream_t st = (cudaStream_t)stream;
  int *dcr = nullptr;
  if (cr) {
    for (int k = 0; k < M; k++)
      if (cr[k] < 0 || cr[k] >= Nf) {
        fprintf(stderr, "dirac_b200_manifold_projectback_dev: cr[%d] = %d is outside [0, %d)\n", k,
                cr[k], Nf);
        return -1;
      }
    // stream-ordered: the copy is staged from pageable memory before cudaMemcpyAsync returns, and
    // the buffer is released after the kernel, without a host wait
    DB_CHECK(cudaMallocAsync((void **)&dcr, sizeof(int) * M, st));
    DB_CHECK(cudaMemcpyAsync(dcr, cr, sizeof(int) * M, cudaMemcpyHostToDevice, st));
  }
  const int rv = db_manifold_projectback(Y, N, M, Nf, Niter, dcr, st);
  if (dcr) DB_CHECK(cudaFreeAsync(dcr, st));
  return rv;
}

// The reference's entry point, with its signature: Y [Nf][M][8N] host, in place.  With randomize the
// chunk k projects first onto block rand() % Nf, drawn here for k = 0..M-1 in order: the reference's
// draws with Nt = 1.  With more threads the reference's draws interleave between its threads in an
// order that changes from run to run, so no run of it can be reproduced.  Nt is not used.
extern "C" int calculate_manifold_average_projectback(int N, int M, int Nf, double *Y, int Niter,
                                                      int randomize, int Nt) {
  (void)Nt;
  if (mf_check("calculate_manifold_average_projectback", N, M, Nf, Niter)) return -1;
  std::vector<int> cr(M, 0);
  if (randomize)
    for (int k = 0; k < M; k++) cr[k] = rand() % Nf;
  DeviceScope ds;
  const size_t len = (size_t)Nf * M * 8 * N;
  double *dY = ds.upload(Y, len);
  int *dcr = ds.upload(cr);
  if (db_manifold_projectback(dY, N, M, Nf, Niter, dcr, ds.st)) return -1;
  DB_CHECK(cudaMemcpyAsync(Y, dY, sizeof(double) * len, cudaMemcpyDeviceToHost, ds.st));
  ds.sync();
  return 0;
}
