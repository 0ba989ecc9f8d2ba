// Influence-function kernels of calculate_diagnostics_gpu (influence_function.cu of the reference, in
// fp64 and without atomics: every output element is written by one thread, sums run in a fixed order,
// so results are bit-identical from run to run).  2x2 complex matrices are row major: m[2a+b].
#include "influence.h"

namespace {

__device__ __forceinline__ double2 conjg(double2 a) { return make_double2(a.x, -a.y); }

// Jones of station s of cluster k at row n (the row's hybrid chunk)
__device__ __forceinline__ void jones(const InflArgs &a, int k, long long n, int s, double2 J[4]) {
  const int c = row_chunk(n, a.R, a.clus_nchunk[k]);
  const double2 *pj = reinterpret_cast<const double2 *>(a.p + a.chunk_poff[a.clus_chunk0[k] + c]) + 4 * s;
#pragma unroll
  for (int i = 0; i < 4; i++) J[i] = __ldg(pj + i);
}

// One thread per (baseline b, cluster k), over the timeslots: the off-diagonal blocks of the
// Hessian, kernel_hessian's kron(-C^T, R^H) as stored at (q, p), i.e. [2a+c][2b+d] = -C_ab conj(R_cd),
// and its conjugate transpose at (p, q); AdV's column b at station p's split rows, (1+j) times the
// column sums of kron(conj(C) J_q^T, I2); S_b = sum_t conj(J_q) C^T over every row.
__global__ void __launch_bounds__(128) k_infl_baseline(InflArgs a) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  const int k = blockIdx.y;
  if (b >= a.Nbase) return;
  const int p = a.sta1[b], q = a.sta2[b];
  const int n4 = 4 * a.N;
  const double2 z = make_double2(0.0, 0.0);
  double2 G[16], S[4], adv0 = z, adv1 = z;
#pragma unroll
  for (int i = 0; i < 16; i++) G[i] = z;
#pragma unroll
  for (int i = 0; i < 4; i++) S[i] = z;
  const double2 *ck = a.coh + (size_t)k * 4 * a.R;
  for (int t = 0; t < a.T; t++) {
    const long long n = (long long)t * a.Nbase + b;
    double2 C[4], J[4];
#pragma unroll
    for (int i = 0; i < 4; i++) C[i] = ck[4 * n + i];
    jones(a, k, n, q, J);
    // conj(J) C^T: [x][y] = sum_m conj(J_xm) C_ym
#pragma unroll
    for (int x = 0; x < 2; x++)
#pragma unroll
      for (int y = 0; y < 2; y++)
        S[2 * x + y] = cadd(S[2 * x + y], cadd(cmulc(C[2 * y], J[2 * x]), cmulc(C[2 * y + 1], J[2 * x + 1])));
    if (a.flag[n]) continue;
    double2 Rv[4];
#pragma unroll
    for (int i = 0; i < 4; i++) Rv[i] = a.res[4 * n + i];
#pragma unroll
    for (int ia = 0; ia < 2; ia++)
#pragma unroll
      for (int ib = 0; ib < 2; ib++)
#pragma unroll
        for (int ic = 0; ic < 2; ic++)
#pragma unroll
          for (int id = 0; id < 2; id++) {
            const double2 v = cmulc(C[2 * ia + ib], Rv[2 * ic + id]);
            double2 &g = G[4 * (2 * ia + ic) + 2 * ib + id];
            g = make_double2(g.x - v.x, g.y - v.y);
          }
    // A = conj(C) J_q^T: A_xy = sum_m conj(C_xm) J_ym; column sums A_0y + A_1y
#pragma unroll
    for (int y = 0; y < 2; y++) {
      double2 s = z;
#pragma unroll
      for (int x = 0; x < 2; x++)
        s = cadd(s, cadd(cmulc(J[2 * y], C[2 * x]), cmulc(J[2 * y + 1], C[2 * x + 1])));
      if (y == 0) adv0 = cadd(adv0, s); else adv1 = cadd(adv1, s);
    }
  }
  double2 *Hk = a.H + (size_t)k * n4 * n4;
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) {
      Hk[(size_t)(4 * p + j) * n4 + 4 * q + i] = G[4 * i + j];
      Hk[(size_t)(4 * q + i) * n4 + 4 * p + j] = conjg(G[4 * i + j]);
    }
  double2 *Ak = a.AdV + ((size_t)k * a.Nbase + b) * n4;
  const double2 v0 = make_double2(adv0.x - adv0.y, adv0.x + adv0.y);  // (1+j) adv0
  const double2 v1 = make_double2(adv1.x - adv1.y, adv1.x + adv1.y);
  Ak[2 * p] = v0;
  Ak[2 * p + 1] = v0;
  Ak[2 * a.N + 2 * p] = v1;
  Ak[2 * a.N + 2 * p + 1] = v1;
  double2 *Sk = a.S + ((size_t)k * a.Nbase + b) * 4;
#pragma unroll
  for (int i = 0; i < 4; i++) Sk[i] = S[i];
}

// One CTA per (station s, cluster k): the diagonal block kron(D, I2) of s, D summed over the unflagged
// rows of its baselines: (C J_q^H)(C J_q^H)^H where s is sta1, (J_p C)^H (J_p C) where s is sta2.
// Strided per-thread sums, then a fixed-order tree.
#define INFL_ST_THREADS 128
__global__ void __launch_bounds__(INFL_ST_THREADS) k_infl_station(InflArgs a) {
  const int s = blockIdx.x, k = blockIdx.y;
  const int e0 = a.st_off[s], nb = a.st_off[s + 1] - e0;
  const double2 z = make_double2(0.0, 0.0);
  double2 D[4] = {z, z, z, z};
  const double2 *ck = a.coh + (size_t)k * 4 * a.R;
  const long long items = (long long)nb * a.T;
  for (long long it = threadIdx.x; it < items; it += INFL_ST_THREADS) {
    const int e = a.st_bl[e0 + (int)(it % nb)];
    const int b = e >> 1, side = e & 1;
    const long long n = (it / nb) * a.Nbase + b;
    if (a.flag[n]) continue;
    double2 C[4], J[4], A[4];
#pragma unroll
    for (int i = 0; i < 4; i++) C[i] = ck[4 * n + i];
    if (side == 0) {
      jones(a, k, n, a.sta2[b], J);
      // A = C J^H: A_xy = sum_m C_xm conj(J_ym); D = A A^H: D_xy = sum_m A_xm conj(A_ym)
#pragma unroll
      for (int x = 0; x < 2; x++)
#pragma unroll
        for (int y = 0; y < 2; y++)
          A[2 * x + y] = cadd(cmulc(C[2 * x], J[2 * y]), cmulc(C[2 * x + 1], J[2 * y + 1]));
#pragma unroll
      for (int x = 0; x < 2; x++)
#pragma unroll
        for (int y = 0; y < 2; y++)
          D[2 * x + y] = cadd(D[2 * x + y], cadd(cmulc(A[2 * x], A[2 * y]), cmulc(A[2 * x + 1], A[2 * y + 1])));
    } else {
      jones(a, k, n, a.sta1[b], J);
      // A = J C: A_xy = sum_m J_xm C_my; D = A^H A: D_xy = sum_m conj(A_mx) A_my
#pragma unroll
      for (int x = 0; x < 2; x++)
#pragma unroll
        for (int y = 0; y < 2; y++)
          A[2 * x + y] = cadd(cmul(J[2 * x], C[y]), cmul(J[2 * x + 1], C[2 + y]));
#pragma unroll
      for (int x = 0; x < 2; x++)
#pragma unroll
        for (int y = 0; y < 2; y++)
          D[2 * x + y] = cadd(D[2 * x + y], cadd(cmulc(A[y], A[x]), cmulc(A[2 + y], A[2 + x])));
    }
  }
  __shared__ double2 sh[4][INFL_ST_THREADS];
#pragma unroll
  for (int i = 0; i < 4; i++) sh[i][threadIdx.x] = D[i];
  __syncthreads();
  for (int w = INFL_ST_THREADS / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w)
#pragma unroll
      for (int i = 0; i < 4; i++) sh[i][threadIdx.x] = cadd(sh[i][threadIdx.x], sh[i][threadIdx.x + w]);
    __syncthreads();
  }
  if (threadIdx.x < 16) {
    const int r = threadIdx.x & 3, c = threadIdx.x >> 2;  // element (r, c) of the 4x4 block
    const int n4 = 4 * a.N;
    const double2 v = ((r & 1) == (c & 1)) ? sh[2 * (r >> 1) + (c >> 1)][0] : z;
    a.H[(size_t)k * n4 * n4 + (size_t)(4 * s + c) * n4 + 4 * s + r] = v;
  }
}

__global__ void k_infl_condition(InflArgs a, const double *hadd) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x, k = blockIdx.y;
  const int n4 = 4 * a.N;
  if (i >= n4) return;
  double2 *h = a.H + (size_t)k * n4 * n4 + (size_t)i * n4 + i;
  double v = h->x;
  // diagnostics.c:712 compares the C integer abs of the float: (int)v == 0, i.e. -1 < v < 1
  if (v > -1.0 && v < 1.0) v = 1.0;
  if (hadd) v += hadd[k];
  h->x = v;
}

// dR_c[b][bl] = sum_k (kron(S_kb^T, I2) x_k(b, bl))_c, x_k(b, bl) the split rows of station sta1[b]
// in column bl of X_k.  Threads along b: the writes of a warp are contiguous.
__global__ void __launch_bounds__(256) k_infl_dr(InflArgs a) {
  const int b = blockIdx.x * 32 + threadIdx.x;
  const int bl = blockIdx.y * 8 + threadIdx.y;
  if (b >= a.Nbase || bl >= a.Nbase) return;
  const int s = a.sta1[b];
  const int n4 = 4 * a.N;
  const double2 z = make_double2(0.0, 0.0);
  double2 o0 = z, o1 = z, o2 = z, o3 = z;
  for (int k = 0; k < a.M; k++) {
    const double2 *Sk = a.S + ((size_t)k * a.Nbase + b) * 4;
    const double2 S00 = Sk[0], S01 = Sk[1], S10 = Sk[2], S11 = Sk[3];
    const double2 *xc = a.X + ((size_t)k * a.Nbase + bl) * n4;
    const double2 j0 = xc[2 * s], j1 = xc[2 * s + 1], j2 = xc[2 * a.N + 2 * s], j3 = xc[2 * a.N + 2 * s + 1];
    o0 = cadd(o0, cadd(cmul(S00, j0), cmul(S10, j2)));
    o1 = cadd(o1, cadd(cmul(S00, j1), cmul(S10, j3)));
    o2 = cadd(o2, cadd(cmul(S01, j0), cmul(S11, j2)));
    o3 = cadd(o3, cadd(cmul(S01, j1), cmul(S11, j3)));
  }
  const size_t nn = (size_t)a.Nbase * a.Nbase, at = (size_t)bl * a.Nbase + b;
  a.dR[at] = o0;
  a.dR[nn + at] = o1;
  a.dR[2 * nn + at] = o2;
  a.dR[3 * nn + at] = o3;
}

// find_eigenvalues' layout (diagnostics.c:975-988): E_c the eigenvalues of correlation c as
// interleaved doubles; x[8b+2c] = E_c[b], x[8b+2c+1] = E_c[Nbase+b], in every timeslot
__global__ void k_infl_eigs(const double2 *W, double2 *x, int Nbase, long long R) {
  const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= R) return;
  const int b = (int)(n % Nbase);
#pragma unroll
  for (int c = 0; c < 4; c++) {
    const double *E = reinterpret_cast<const double *>(W + (size_t)c * Nbase);
    x[4 * n + c] = make_double2(E[b], E[Nbase + b]);
  }
}

}  // namespace

extern "C" void db_launch_infl_assemble(const InflArgs *a, cudaStream_t st) {
  const size_t n4 = 4 * (size_t)a->N;
  DB_CHECK(cudaMemsetAsync(a->H, 0, sizeof(double2) * n4 * n4 * a->M, st));
  DB_CHECK(cudaMemsetAsync(a->AdV, 0, sizeof(double2) * n4 * a->Nbase * a->M, st));
  k_infl_baseline<<<dim3((a->Nbase + 127) / 128, a->M), 128, 0, st>>>(*a);
  k_infl_station<<<dim3(a->N, a->M), INFL_ST_THREADS, 0, st>>>(*a);
  DB_CHECK(cudaGetLastError());
}

extern "C" void db_launch_infl_condition(const InflArgs *a, const double *hadd, cudaStream_t st) {
  k_infl_condition<<<dim3((4 * a->N + 127) / 128, a->M), 128, 0, st>>>(*a, hadd);
  DB_CHECK(cudaGetLastError());
}

extern "C" void db_launch_infl_dr(const InflArgs *a, cudaStream_t st) {
  k_infl_dr<<<dim3((a->Nbase + 31) / 32, (a->Nbase + 7) / 8), dim3(32, 8), 0, st>>>(*a);
  DB_CHECK(cudaGetLastError());
}

extern "C" void db_launch_infl_eigs(const double2 *W, double2 *x, int Nbase, int T, cudaStream_t st) {
  const long long R = (long long)Nbase * T;
  k_infl_eigs<<<(unsigned)((R + 255) / 256), 256, 0, st>>>(W, x, Nbase, R);
  DB_CHECK(cudaGetLastError());
}
