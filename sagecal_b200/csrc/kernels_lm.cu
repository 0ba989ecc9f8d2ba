// Normal-equation assembly and small dense helpers of the per-cluster LM solver.
//
// The reference forms the dense n x 8N Jacobian (jacobian_threadfn, lmfit.c:392-474) and calls
// dgemm for J^T J (clmfit.c:307).  J has 16 non-zeros per row-octet and, for fixed Jones, J^T J
// depends on the data only through the per-baseline Gram tensor Th = sum_t conj(c) c^T of the
// coherencies (k_coh_gram).  With X = C Jq^H, Y = Jp C (V = Jp X = Y Jq^H):
//   block (p,q)[(i,l),(j,l')] = R( sum_t conj(X_lj) Y_il' ) S ,  sum_t conj(X_lj) Y_il'
//                             = sum_ab Jq_ja Jp_ib Th[(l,a),(b,l')]
//   block (p,p)[(i,l),(i,l')] = R( conj(Hp_ll') ),  Hp_ll' = sum_ab (Jq^H Jq)_ab Th[(l',b),(l,a)]
//   block (q,q)[(j,l),(j,l')] = R( conj(Hq_ll') ),  Hq_ll' = sum_ab (Jp^H Jp)_ab Th[(a,l),(b,l')]
// where R(z) = [[zr,-zi],[zi,zr]], S = diag(1,-1); parameter order per station is
// [Re J00, Im J00, Re J01, Im J01, Re J10, Im J10, Re J11, Im J11] (lmfit.c:90-97,460-467).
// See DESIGN.md for the derivation.
#include "internal.cuh"

// Hermitian 4x4 Gram tensor access from its packed form (k_coh_gram): index u = 2a+b
struct Gram {
  double d[4];
  double2 o[6];  // (0,1)(0,2)(0,3)(1,2)(1,3)(2,3)
  __device__ __forceinline__ double2 at(int u, int v) const {
    if (u == v) return make_double2(d[u], 0.0);
    int lo = u < v ? u : v, hi = u < v ? v : u;
    int idx = (lo == 0) ? (hi - 1) : (lo == 1 ? (hi + 1) : 5);
    double2 z = o[idx];
    return (u < v) ? z : make_double2(z.x, -z.y);
  }
};


// Baseline index of the station pair p < q (the canonical order problem.cu builds blpq in)
__device__ __forceinline__ long long pair_baseline(int p, int q, int N) {
  return (long long)p * (2 * N - p - 1) / 2 + (q - p - 1);
}

__device__ __forceinline__ Gram load_gram(const double *T, long long b) {
  Gram G;
  const double2 *Tb = reinterpret_cast<const double2 *>(T + b * 16);
  const double2 t0 = __ldg(Tb), t1 = __ldg(Tb + 1);
  G.d[0] = t0.x; G.d[1] = t0.y; G.d[2] = t1.x; G.d[3] = t1.y;
#pragma unroll
  for (int z = 0; z < 6; z++) G.o[z] = __ldg(Tb + 2 + z);
  return G;
}

// system y of an assembly launch (one system, or matrix y of a batch over b.list)
struct AsmSys {
  const double *T, *J;
  double *A, *H;
  double mu;
};
__device__ __forceinline__ AsmSys asm_sys(const AssembleArgs &a, int y) {
  AsmSys s;
  if (a.list) {
    const int k = a.list[y];
    s.T = a.T + (long long)a.tix[k] * a.Nbase * 16;
    s.J = a.pblk + a.poff[k];
  } else {
    s.T = a.T;
    s.J = a.pblk;
  }
  s.A = a.JTJ + (long long)y * a.stride;
  s.H = a.Hst + (long long)y * 4 * a.N;
  s.mu = a.mu_dev ? a.mu_dev[y] : a.mu;
  return s;
}

// Station sums of the diagonal blocks: one warp per station s walks its N-1 baselines (lane-strided)
// and reduces with a fixed shuffle tree, so the sums do not depend on scheduling.
//   s = p of (s,o):  Hp_ll' = sum_ab (Jo^H Jo)_ab Th[(l',b),(l,a)]
//   s = q of (o,s):  Hq_ll' = sum_ab (Jo^H Jo)_ab Th[(a,l),(b,l')]
// Hst[s] = (H00, H11, Re H01, Im H01); blockIdx.y: matrix of the batch.
__global__ void __launch_bounds__(256)
k_station_sums(AssembleArgs a) {
  const AsmSys S = asm_sys(a, blockIdx.y);
  const int s = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (s >= a.N) return;
  double h0 = 0.0, h1 = 0.0, h2 = 0.0, h3 = 0.0;
  for (int o = lane; o < a.N; o += 32) {
    if (o == s) continue;
    const bool sp = s < o;
    const Gram G = load_gram(S.T, sp ? pair_baseline(s, o, a.N) : pair_baseline(o, s, a.N));
    double2 Jo[4], Qo[4];
    load_jones(S.J, o, Jo);
    mat_ahb(Jo, Jo, Qo);
    double2 h[4];
#pragma unroll
    for (int l = 0; l < 2; l++)
#pragma unroll
      for (int lp = 0; lp < 2; lp++) {
        double2 z = make_double2(0.0, 0.0);
#pragma unroll
        for (int aa = 0; aa < 2; aa++)
#pragma unroll
          for (int bb = 0; bb < 2; bb++)
            cfma(z, Qo[2 * aa + bb], sp ? G.at(2 * lp + bb, 2 * l + aa) : G.at(2 * aa + l, 2 * bb + lp));
        h[2 * l + lp] = z;
      }
    h0 += h[0].x;
    h1 += h[3].x;
    h2 += h[1].x;
    h3 += h[1].y;
  }
  h0 = warp_sum(h0);
  h1 = warp_sum(h1);
  h2 = warp_sum(h2);
  h3 = warp_sum(h3);
  if (lane == 0) {
    S.H[4 * s] = h0;
    S.H[4 * s + 1] = h1;
    S.H[4 * s + 2] = h2;
    S.H[4 * s + 3] = h3;
  }
}

// J^T J (+ mu I) by output tiles.  Memory row R = 8P + r holds, from column 8Q on, the 8x8 block of
// the station pair (P,Q).  A warp owns station P and a group of 8 stations Q: lane t computes the 2x2
// sub-blocks (i,l) x (j,lp) = (0..3) x (t & 3) of the pair (P, Q0 + t/4) and stores them as double2,
// so each store of the warp is one contiguous 512-byte row segment.  A CTA (8 warps) covers 64
// stations Q of one station P; blockIdx.z: matrix of the batch.
//
// `lower`: only the Q groups that reach Q >= P are written, i.e. the lower triangle of the
// column-major matrix that dpotrf(LOWER) and the blocked triangular solves read (plus a few blocks
// of the other triangle in the diagonal group, written with their true values).
//
// Off-diagonal block (p,q), p < q: [(i,l),(j,l')] = R(z) S = [[zr, zi],[zi, -zr]] with
// z = sum_ab Jq_ja Jp_ib Th[(l,a),(b,l')]; the 2x2 is symmetric, so block (q,p) holds the same 2x2
// at the transposed sub-block.  Diagonal block: the station sums (k_station_sums) plus mu.
__global__ void __launch_bounds__(256)
k_assemble_tiles(AssembleArgs a) {
  const int P = blockIdx.x;
  const int qcta = blockIdx.y * 64;
  if (a.lower && qcta + 64 <= P) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = qcta + 8 * warp;
  if (q0 >= a.N || (a.lower && q0 + 8 <= P)) return;
  const AsmSys S = asm_sys(a, blockIdx.z);
  const int Q = q0 + (lane >> 2);
  const int jl = lane & 3, j = jl >> 1, lp = jl & 1;
  const long long ld = 8ll * a.N;
  if (Q == P) {
    const double h00 = S.H[4 * P], h11 = S.H[4 * P + 1], hr = S.H[4 * P + 2], hi = S.H[4 * P + 3];
    // 4x4 block of polarisation row i = column j; the blocks i != j are zero
    const double blk[4][4] = {{h00, 0.0, hr, hi}, {0.0, h00, -hi, hr}, {hr, -hi, h11, 0.0},
                              {hi, hr, 0.0, h11}};
#pragma unroll
    for (int il = 0; il < 4; il++) {
      const int i = il >> 1, l = il & 1;
      double2 v0 = make_double2(0.0, 0.0), v1 = v0;
      if (i == j) {  // (lane-dependent lp selects between static indices: no local memory)
        const double m = (l == lp) ? S.mu : 0.0;
        v0 = lp ? make_double2(blk[2 * l][2], blk[2 * l][3]) : make_double2(blk[2 * l][0], blk[2 * l][1]);
        v1 = lp ? make_double2(blk[2 * l + 1][2], blk[2 * l + 1][3])
                : make_double2(blk[2 * l + 1][0], blk[2 * l + 1][1]);
        v0.x += m;
        v1.y += m;
      }
      const long long r0 = 8ll * P + 2 * il;
      *reinterpret_cast<double2 *>(S.A + r0 * ld + 8ll * Q + 2 * jl) = v0;
      *reinterpret_cast<double2 *>(S.A + (r0 + 1) * ld + 8ll * Q + 2 * jl) = v1;
    }
    return;
  }
  if (Q < a.N) {
    const bool pq = P < Q;  // the pair's baseline is (P,Q); otherwise (Q,P) and its block transposed
    const Gram G = load_gram(S.T, pq ? pair_baseline(P, Q, a.N) : pair_baseline(Q, P, a.N));
    double2 JP[4], JQ[4];
    load_jones(S.J, P, JP);
    load_jones(S.J, Q, JQ);
    const double2 Jj[2] = {j ? JQ[2] : JQ[0], j ? JQ[3] : JQ[1]};  // JQ[2j + x]
#pragma unroll
    for (int il = 0; il < 4; il++) {
      const int i = il >> 1, l = il & 1;
      double2 z = make_double2(0.0, 0.0);
#pragma unroll
      for (int aa = 0; aa < 2; aa++)
#pragma unroll
        for (int bb = 0; bb < 2; bb++) {
          if (pq)  // baseline (p,q) = (P,Q), sub-block (i,l) x (j,lp)
            cfma(z, cmul(Jj[aa], JP[2 * i + bb]),
                 lp ? G.at(2 * l + aa, 2 * bb + 1) : G.at(2 * l + aa, 2 * bb));
          else     // baseline (p,q) = (Q,P), sub-block (j,lp) x (i,l)
            cfma(z, cmul(JP[2 * i + aa], Jj[bb]), lp ? G.at(2 + aa, 2 * bb + l) : G.at(aa, 2 * bb + l));
        }
      const long long r0 = 8ll * P + 2 * il;
      *reinterpret_cast<double2 *>(S.A + r0 * ld + 8ll * Q + 2 * jl) = z;
      *reinterpret_cast<double2 *>(S.A + (r0 + 1) * ld + 8ll * Q + 2 * jl) = make_double2(z.y, -z.x);
    }
  }
}

// per matrix of the batch: mu0 = tau * max_i (J^T J)_ii (clmfit.c:342-352) -> mu[y]; the diagonal is
// (h00 x4, h11 x4) per station, so the maximum runs over the station sums
__global__ void __launch_bounds__(128)
k_batch_mu0(const double *__restrict__ Hst, double *__restrict__ mu, int N, double tau) {
  __shared__ double sv[4];
  const double *H = Hst + (long long)blockIdx.x * 4 * N;
  double mx = 0.0;
  for (int s = threadIdx.x; s < N; s += blockDim.x) {
    const double a = H[4 * s], b = H[4 * s + 1];
    if (fabs(a) > fabs(mx)) mx = a;
    if (fabs(b) > fabs(mx)) mx = b;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double other = __shfl_xor_sync(0xffffffffu, mx, o);
    if (fabs(other) > fabs(mx)) mx = other;
  }
  if ((threadIdx.x & 31) == 0) sv[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < 4; i++)
      if (fabs(sv[i]) > fabs(mx)) mx = sv[i];
    mu[blockIdx.x] = tau * mx;
  }
}

// A_ii += mu  (cudakernel_diagmu, mderiv.cu:936; my_daxpys on the diagonal, clmfit.c:363)
__global__ void k_copy_add_diag(const double *__restrict__ A0, double *__restrict__ A, int n,
                                double mu) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long nn = (long long)n * n;
  if (i < nn) {
    double v = A0[i];
    if (i / n == i % n) v += mu;
    A[i] = v;
  }
}

__global__ void k_extract_diag(const double *__restrict__ A, double *__restrict__ dst, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = A[(long long)i * n + i];
}

// pnew = p + dp ; sc[0] = |dp|^2 ; sc[1] = dp . J^T e   (clmfit.c:440-449,487-497), one CTA
// zero (optional): accumulator of the trial pass that follows, cleared here instead of by a memset
__global__ void __launch_bounds__(512)
k_lm_step(const double *__restrict__ p, const double *__restrict__ Dp,
          const double *__restrict__ jte, double *__restrict__ pnew, double *__restrict__ sc,
          double *__restrict__ zero, int n) {
  __shared__ double s0[16], s1[16];
  double a = 0.0, b = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const double dp = Dp[i];
    pnew[i] = p[i] + dp;
    if (zero) zero[i] = 0.0;
    a = fma(dp, dp, a);
    b = fma(dp, jte[i], b);
  }
  a = warp_sum(a);
  b = warp_sum(b);
  if ((threadIdx.x & 31) == 0) {
    s0[threadIdx.x >> 5] = a;
    s1[threadIdx.x >> 5] = b;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double ta = 0.0, tb = 0.0;
    for (int i = 0; i < (int)(blockDim.x >> 5); i++) {
      ta += s0[i];
      tb += s1[i];
    }
    sc[0] = ta;
    sc[1] = tb;
  }
}

// g <- g - y/2 - rho/2 (p - bz): J^T e of a pass -> (minus half) the gradient of the consensus-
// augmented cost ||e||^2 + y^T (p - bz) + rho/2 |p - bz|^2
__global__ void k_lm_aug_rhs(double *__restrict__ g, const double *__restrict__ p,
                             const double *__restrict__ y, const double *__restrict__ bz, double rho,
                             int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) g[i] = g[i] - 0.5 * y[i] - 0.5 * rho * (p[i] - bz[i]);
}

extern "C" {
void db_launch_lm_aug_rhs(double *jte, const double *p, const double *y, const double *bz,
                          double rho, int n, cudaStream_t st) {
  k_lm_aug_rhs<<<(n + 255) / 256, 256, 0, st>>>(jte, p, y, bz, rho, n);
}
void db_launch_lm_step(const double *p, const double *Dp, const double *jte, double *pnew,
                       double *sc, double *zero, int n, cudaStream_t st) {
  k_lm_step<<<1, 512, 0, st>>>(p, Dp, jte, pnew, sc, zero, n);
}
void db_launch_extract_diag(const double *A, double *dst, int n, cudaStream_t st) {
  k_extract_diag<<<(n + 127) / 128, 128, 0, st>>>(A, dst, n);
}
void db_launch_station_sums(const AssembleArgs *a, int nb, cudaStream_t st) {
  k_station_sums<<<dim3((a->N + 7) / 8, nb), 256, 0, st>>>(*a);
}
void db_launch_assemble_tiles(const AssembleArgs *a, int nb, cudaStream_t st) {
  k_assemble_tiles<<<dim3(a->N, (a->N + 63) / 64, nb), 256, 0, st>>>(*a);
}
void db_launch_batch_mu0(const double *Hst, double *mu, int N, double tau, int nb, cudaStream_t st) {
  k_batch_mu0<<<nb, 128, 0, st>>>(Hst, mu, N, tau);
}
void db_launch_copy_add_diag(const double *A0, double *A, int n, double mu, cudaStream_t st) {
  long long nn = (long long)n * n;
  k_copy_add_diag<<<(unsigned)((nn + 255) / 256), 256, 0, st>>>(A0, A, n, mu);
}
}
