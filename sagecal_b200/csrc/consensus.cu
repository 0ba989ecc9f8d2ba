// Consensus (ADMM) calibration over frequency subbands, one subband per GPU (BASELINE.json config 5).
//
// The reference runs a master process that gathers Y_f + rho J_f from every slave, forms
// z = sum_f B_f (x) (Y_f + rho J_f), Z = Bi z, and sends B_f Z back (sagecal_master.cpp:844-877,
// sagecal_slave.cpp:831-878, consensus_poly.c:636-700).  Here there is no master: every rank owns one
// subband, the sum over subbands is ONE all-reduce of Npoly*8*N*Mt doubles (1.5 MB at 62 stations,
// 128 clusters, Npoly 3) on the library's stream, and every rank applies the replicated Bi and its
// own basis row B_f itself.  Per cluster k the two steps collapse into Npoly weights
// c_k[p] = sum_p' Bi_k[p][p'] B_f[p'] (host, tiny), so B_f Z of cluster k is sum_p c_k[p] z_p.
//
// The basis and the pseudo-inverse are plain host arithmetic (no GPU needed): they restate
// setup_polynomials (consensus_poly.c:38-190) and find_prod_inverse_full (:380-545) and are pinned
// against the compiled reference by the CPU tests.
#include <math.h>
#include <stdio.h>
#include <string.h>
#include <vector>

#include "../../include/dirac_b200.h"
#include "problem.h"

// ---- basis functions in frequency (consensus_poly.c:38-190); B[f*Npoly + p] -----------------------
extern "C" int dirac_b200_consensus_basis(double *B, int Npoly, int Nf, const double *freqs,
                                          double freq0, int type) {
  if (type == 0 || type == 1) {
    const double invf = 1.0 / freq0;
    for (int f = 0; f < Nf; f++) {
      B[f * Npoly] = 1.0;
      const double frat = (freqs[f] - freq0) * invf;
      for (int p = 1; p < Npoly; p++) B[f * Npoly + p] = B[f * Npoly + p - 1] * frat;
    }
    if (type == 1) {  // every basis function normalised over the subbands
      for (int p = 0; p < Npoly; p++) {
        double s = 0.0;
        for (int f = 0; f < Nf; f++) s += B[f * Npoly + p] * B[f * Npoly + p];
        const double sc = s > 0.0 ? 1.0 / sqrt(s) : 0.0;
        for (int f = 0; f < Nf; f++) B[f * Npoly + p] *= sc;
      }
    }
    return 0;
  }
  if (type == 2) {  // Bernstein polynomials on [fmin, fmax]
    double fmax = freqs[0], fmin = freqs[0];
    {
      // the reference picks the extremes by |value| (idamax / idamin); frequencies are positive
      double amax = fabs(freqs[0]), amin = fabs(freqs[0]);
      for (int f = 1; f < Nf; f++) {
        if (fabs(freqs[f]) > amax) { amax = fabs(freqs[f]); fmax = freqs[f]; }
        if (fabs(freqs[f]) < amin) { amin = fabs(freqs[f]); fmin = freqs[f]; }
      }
    }
    std::vector<double> fact(Npoly), px((size_t)Npoly * Nf), p1x((size_t)Npoly * Nf);
    fact[0] = 1.0;
    for (int i = 1; i < Npoly; i++) fact[i] = fact[i - 1] * (double)i;
    const double invf = 1.0 / (fmax - fmin);
    for (int f = 0; f < Nf; f++) {
      const double frat = (freqs[f] - fmin) * invf;
      px[f] = 1.0;
      p1x[f] = 1.0;
      if (Npoly > 1) {
        px[f + Nf] = frat;
        p1x[f + Nf] = 1.0 - frat;
      }
    }
    for (int j = 2; j < Npoly; j++)
      for (int f = 0; f < Nf; f++) {
        px[j * Nf + f] = px[(j - 1) * Nf + f] * px[Nf + f];
        p1x[j * Nf + f] = p1x[(j - 1) * Nf + f] * p1x[Nf + f];
      }
    for (int j = 0; j < Npoly; j++) {
      const double c = fact[Npoly - 1] / (fact[Npoly - j - 1] * fact[j]);
      for (int f = 0; f < Nf; f++) B[f * Npoly + j] = c * px[j * Nf + f] * p1x[(Npoly - j - 1) * Nf + f];
    }
    return 0;
  }
  if (type == 3) {  // [1, (f-f0)/f0, (f0/f-1), ((f-f0)/f0)^2, ...]
    const double invf = 1.0 / freq0;
    for (int f = 0; f < Nf; f++) {
      B[f * Npoly] = 1.0;
      double frat = (freqs[f] - freq0) * invf, last = frat;
      for (int p = 1; p < Npoly; p += 2) { B[f * Npoly + p] = last; last *= frat; }
      frat = freq0 / freqs[f] - 1.0;
      last = frat;
      for (int p = 2; p < Npoly; p += 2) { B[f * Npoly + p] = last; last *= frat; }
    }
    return 0;
  }
  return -1;
}

// symmetric eigen-decomposition by cyclic Jacobi rotations (n <= ~16): A = V diag(w) V^T
static void jacobi_eig(std::vector<double> &A, int n, std::vector<double> &V, std::vector<double> &w) {
  V.assign((size_t)n * n, 0.0);
  for (int i = 0; i < n; i++) V[i * n + i] = 1.0;
  for (int sweep = 0; sweep < 60; sweep++) {
    double off = 0.0;
    for (int i = 0; i < n; i++)
      for (int j = i + 1; j < n; j++) off += A[i * n + j] * A[i * n + j];
    if (off < 1e-300) break;
    for (int p = 0; p < n; p++)
      for (int q = p + 1; q < n; q++) {
        const double apq = A[p * n + q];
        if (fabs(apq) < 1e-300) continue;
        const double theta = (A[q * n + q] - A[p * n + p]) / (2.0 * apq);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < n; k++) {
          const double akp = A[k * n + p], akq = A[k * n + q];
          A[k * n + p] = c * akp - s * akq;
          A[k * n + q] = s * akp + c * akq;
        }
        for (int k = 0; k < n; k++) {
          const double apk = A[p * n + k], aqk = A[q * n + k];
          A[p * n + k] = c * apk - s * aqk;
          A[q * n + k] = s * apk + c * aqk;
        }
        for (int k = 0; k < n; k++) {
          const double vkp = V[k * n + p], vkq = V[k * n + q];
          V[k * n + p] = c * vkp - s * vkq;
          V[k * n + q] = s * vkp + c * vkq;
        }
      }
  }
  w.resize(n);
  for (int i = 0; i < n; i++) w[i] = A[i * n + i];
}

// Bi[k] = pinv( sum_f rho[k + f*M] B_f B_f^T ), singular values <= 1e-12 dropped
// (find_prod_inverse_full / sum_inv_threadfn, consensus_poly.c:380-545; the matrix is symmetric PSD,
// so its SVD pseudo-inverse is the eigen pseudo-inverse)
extern "C" int dirac_b200_consensus_prod_inverse(const double *B, double *Bi, int Npoly, int Nf,
                                                 int M, const double *rho) {
  const int n = Npoly;
  std::vector<double> A((size_t)n * n), V, w;
  for (int k = 0; k < M; k++) {
    std::fill(A.begin(), A.end(), 0.0);
    for (int f = 0; f < Nf; f++) {
      const double r = rho[k + (size_t)f * M];
      for (int i = 0; i < n; i++)
        for (int j = 0; j < n; j++) A[i * n + j] += r * B[f * n + i] * B[f * n + j];
    }
    jacobi_eig(A, n, V, w);
    double *out = Bi + (size_t)k * n * n;
    for (int i = 0; i < n; i++)
      for (int j = 0; j < n; j++) {
        double s = 0.0;
        for (int e = 0; e < n; e++)
          if (w[e] > 1e-12) s += V[i * n + e] * V[j * n + e] / w[e];
        out[i * n + j] = s;
      }
  }
  return 0;
}

// Bi[k] = (sum_f rho[k + f*M] B_f B_f^T + alpha_k I)^-1 as find_prod_inverse_full_fed
// (consensus_poly.c:381-451, 546-600) forms it: every singular value s > 1e-12 becomes 1/(s + alpha_k),
// every other one 1/alpha_k (so a singular sum with alpha_k = 0 gives inf, as the reference's does)
extern "C" int dirac_b200_consensus_prod_inverse_fed(const double *B, double *Bi, int Npoly, int Nf,
                                                     int M, const double *rho, const double *alpha) {
  const int n = Npoly;
  std::vector<double> A((size_t)n * n), V, w;
  for (int k = 0; k < M; k++) {
    std::fill(A.begin(), A.end(), 0.0);
    for (int f = 0; f < Nf; f++) {
      const double r = rho[k + (size_t)f * M];
      for (int i = 0; i < n; i++)
        for (int j = 0; j < n; j++) A[i * n + j] += r * B[f * n + i] * B[f * n + j];
    }
    jacobi_eig(A, n, V, w);
    double *out = Bi + (size_t)k * n * n;
    for (int i = 0; i < n; i++)
      for (int j = 0; j < n; j++) {
        double s = 0.0;
        for (int e = 0; e < n; e++)
          s += V[i * n + e] * V[j * n + e] * (w[e] > 1e-12 ? 1.0 / (w[e] + alpha[k]) : 1.0 / alpha[k]);
        out[i * n + j] = s;
      }
  }
  return 0;
}

// ---- the ADMM step of the spectral consensus over bands (minibatch_consensus_mode.cpp:524-601) ------
// z = B_b Z of every chunk, as the driver sums it (:526-531): z[ci] = sum_p Bb[p] Z[ci][p]
void db_consensus_bz(const double *Z, const double *Bb, int N, int Mt, int Npoly, double *z) {
  const size_t n8 = (size_t)8 * N;
  for (int ci = 0; ci < Mt; ci++) {
    double *zc = z + n8 * ci;
    memset(zc, 0, sizeof(double) * n8);
    for (int p = 0; p < Npoly; p++) {
      const double *Zp = Z + n8 * ((size_t)ci * Npoly + p);
      const double bp = Bb[p];
      for (size_t i = 0; i < n8; i++) zc[i] += bp * Zp[i];
    }
  }
}

// The host lines that run after the bands of one minibatch are fitted, decision for decision, with
// the driver's quirks (DESIGN.md 7): res_0 / res_1 become (previous + sum over bands) / nsolbw, a
// running mixture; a band is flagged when its cost after the fit exceeds 1.5 res_1 (a cost that is not
// > 0 counts as CLM_DBL_MAX); good bands get Y_b += rho_b J_b; the sum z = sum_b B_b (x) Y_b always
// holds band 0, flagged or not; Z = Bi z (update_global_z_multi, consensus_poly.c:706-832); good
// bands get Y_b -= rho_b B_b Z.
extern "C" int dirac_b200_consensus_bands_update(int N, int Mt, int nsolbw, int Npoly,
                                                 const double *res_00, const double *res_01,
                                                 const double *pfreq, const double *B,
                                                 const double *Bi, const double *rhok, double *res_0,
                                                 double *res_1, double *Y, double *Z, int *fband) {
  if (N < 1 || Mt < 1 || nsolbw < 1 || Npoly < 1) {
    fprintf(stderr, "dirac_b200_consensus_bands_update: N = %d, Mt = %d, nsolbw = %d, Npoly = %d; "
                    "each must be at least 1\n", N, Mt, nsolbw, Npoly);
    return -1;
  }
  const size_t n8 = (size_t)8 * N, m = n8 * Mt;
  const double res_ratio = 1.5, clm_dbl_max = 1e12;  // minibatch_consensus_mode.cpp:262, CLM_DBL_MAX
  std::vector<double> resband(nsolbw);
  for (int b = 0; b < nsolbw; b++) {
    *res_0 += res_00[b];
    *res_1 += res_01[b];
    resband[b] = res_00[b] > 0.0 && res_01[b] > 0.0 ? res_01[b] : clm_dbl_max;
  }
  *res_0 /= (double)nsolbw;
  *res_1 /= (double)nsolbw;
  for (int b = 0; b < nsolbw; b++) fband[b] = resband[b] > res_ratio * *res_1 ? 1 : 0;
  // Y_b <- Y_b + rho_b J_b for the good bands
  for (int b = 0; b < nsolbw; b++) {
    if (fband[b]) continue;
    for (int ci = 0; ci < Mt; ci++) {
      const double r = rhok[(size_t)b * Mt + ci];
      const double *J = pfreq + (size_t)b * m + n8 * ci;
      double *y = Y + (size_t)b * m + n8 * ci;
      for (size_t i = 0; i < n8; i++) y[i] += r * J[i];
    }
  }
  // z[p] = sum_b B_b[p] Y_b, laid out [Npoly][Mt][8N]: band 0 unconditionally (:569-572), the others
  // when good
  std::vector<double> z((size_t)Npoly * m);
  for (int p = 0; p < Npoly; p++)
    for (size_t i = 0; i < m; i++) z[(size_t)p * m + i] = B[p] * Y[i];
  for (int b = 1; b < nsolbw; b++) {
    if (fband[b]) continue;
    for (int p = 0; p < Npoly; p++) {
      const double bp = B[(size_t)b * Npoly + p];
      const double *y = Y + (size_t)b * m;
      double *zp = z.data() + (size_t)p * m;
      for (size_t i = 0; i < m; i++) zp[i] += bp * y[i];
    }
  }
  // Z[ci][p] = sum_q Bi[ci][p][q] z[q][ci], Z laid out [Mt][Npoly][8N]
  for (int ci = 0; ci < Mt; ci++)
    for (int p = 0; p < Npoly; p++) {
      double *Zp = Z + n8 * ((size_t)ci * Npoly + p);
      const double *bi = Bi + ((size_t)ci * Npoly + p) * Npoly;
      for (size_t i = 0; i < n8; i++) {
        double s = 0.0;
        for (int q = 0; q < Npoly; q++) s += bi[q] * z[(size_t)q * m + n8 * ci + i];
        Zp[i] = s;
      }
    }
  // Y_b <- Y_b - rho_b B_b Z for the good bands
  std::vector<double> bz(m);
  for (int b = 0; b < nsolbw; b++) {
    if (fband[b]) continue;
    db_consensus_bz(Z, B + (size_t)b * Npoly, N, Mt, Npoly, bz.data());
    for (int ci = 0; ci < Mt; ci++) {
      const double r = rhok[(size_t)b * Mt + ci];
      double *y = Y + (size_t)b * m + n8 * ci;
      for (size_t i = 0; i < n8; i++) y[i] += -r * bz[n8 * ci + i];
    }
  }
  return 0;
}

// The federated slave's step after the bands of one minibatch (sagecal_stochastic_slave.cpp:731-852),
// decision for decision, with one MS per rank.  Where it differs from the in-process step above
// (DESIGN.md 7): res_0 / res_1 are the plain mean over the bands of this minibatch; z starts from zero
// when band 0 is flagged; from ADMM iteration 1 on, z[p][ci] += alpha_k Zavg[ci][p] - X[ci][p].
extern "C" int dirac_b200_federated_bands_update(int N, int Mt, int nsolbw, int Npoly, int admm,
                                                 const double *res_00, const double *res_01,
                                                 const double *pfreq, const double *B,
                                                 const double *Bi, const double *rhok,
                                                 const double *alphak, const double *Zavg,
                                                 const double *X, double *res_0, double *res_1,
                                                 double *Y, double *Z, int *fband) {
  if (N < 1 || Mt < 1 || nsolbw < 1 || Npoly < 1 || admm < 0) {
    fprintf(stderr, "dirac_b200_federated_bands_update: N = %d, Mt = %d, nsolbw = %d, Npoly = %d "
                    "must be at least 1 and admm = %d at least 0\n", N, Mt, nsolbw, Npoly, admm);
    return -1;
  }
  const size_t n8 = (size_t)8 * N, m = n8 * Mt;
  const double res_ratio = 1.5, clm_dbl_max = 1e12;  // sagecal_stochastic_slave.cpp res_ratio, CLM_DBL_MAX
  std::vector<double> resband(nsolbw);
  double r0 = 0.0, r1 = 0.0;
  for (int b = 0; b < nsolbw; b++) {
    r0 += res_00[b];
    r1 += res_01[b];
    resband[b] = res_00[b] > 0.0 && res_01[b] > 0.0 ? res_01[b] : clm_dbl_max;
  }
  r0 /= (double)nsolbw;
  r1 /= (double)nsolbw;
  *res_0 = r0;
  *res_1 = r1;
  for (int b = 0; b < nsolbw; b++) fband[b] = resband[b] > res_ratio * r1 ? 1 : 0;
  // Y_b <- Y_b + rho_b J_b for the good bands
  for (int b = 0; b < nsolbw; b++) {
    if (fband[b]) continue;
    for (int ci = 0; ci < Mt; ci++) {
      const double r = rhok[(size_t)b * Mt + ci];
      const double *J = pfreq + (size_t)b * m + n8 * ci;
      double *y = Y + (size_t)b * m + n8 * ci;
      for (size_t i = 0; i < n8; i++) y[i] += r * J[i];
    }
  }
  // z[p] = sum over the good bands of B_b[p] Y_b, laid out [Npoly][Mt][8N] (:783-797)
  std::vector<double> z((size_t)Npoly * m, 0.0);
  if (!fband[0])
    for (int p = 0; p < Npoly; p++)
      for (size_t i = 0; i < m; i++) z[(size_t)p * m + i] = B[p] * Y[i];
  for (int b = 1; b < nsolbw; b++) {
    if (fband[b]) continue;
    for (int p = 0; p < Npoly; p++) {
      const double bp = B[(size_t)b * Npoly + p];
      const double *y = Y + (size_t)b * m;
      double *zp = z.data() + (size_t)p * m;
      for (size_t i = 0; i < m; i++) zp[i] += bp * y[i];
    }
  }
  // the federated-averaging term, Zavg and X laid out [Mt][Npoly][8N] like Z (:805-826)
  if (admm > 0)
    for (int ci = 0; ci < Mt; ci++)
      for (int p = 0; p < Npoly; p++) {
        const double *za = Zavg + n8 * ((size_t)ci * Npoly + p);
        const double *x = X + n8 * ((size_t)ci * Npoly + p);
        double *zp = z.data() + (size_t)p * m + n8 * ci;
        for (size_t i = 0; i < n8; i++) zp[i] += alphak[ci] * za[i];
        for (size_t i = 0; i < n8; i++) zp[i] += -x[i];
      }
  // Z[ci][p] = sum_q Bi[ci][p][q] z[q][ci]
  for (int ci = 0; ci < Mt; ci++)
    for (int p = 0; p < Npoly; p++) {
      double *Zp = Z + n8 * ((size_t)ci * Npoly + p);
      const double *bi = Bi + ((size_t)ci * Npoly + p) * Npoly;
      for (size_t i = 0; i < n8; i++) {
        double s = 0.0;
        for (int q = 0; q < Npoly; q++) s += bi[q] * z[(size_t)q * m + n8 * ci + i];
        Zp[i] = s;
      }
    }
  // Y_b <- Y_b - rho_b B_b Z for the good bands
  std::vector<double> bz(m);
  for (int b = 0; b < nsolbw; b++) {
    if (fband[b]) continue;
    db_consensus_bz(Z, B + (size_t)b * Npoly, N, Mt, Npoly, bz.data());
    for (int ci = 0; ci < Mt; ci++) {
      const double r = rhok[(size_t)b * Mt + ci];
      double *y = Y + (size_t)b * m + n8 * ci;
      for (size_t i = 0; i < n8; i++) y[i] += -r * bz[n8 * ci + i];
    }
  }
  return 0;
}

// ---- device side of one exchange ---------------------------------------------------------------------
// Y <- Y + rho_k J ; z[p][i] = B_f[p] Y[i]
__global__ void __launch_bounds__(256)
k_consensus_form(const double *__restrict__ J, double *__restrict__ Y, double *__restrict__ z,
                 const double *__restrict__ rho_i, const double *__restrict__ Bf, int m, int Npoly) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
    const double y = fma(rho_i[i], J[i], Y[i]);
    Y[i] = y;
    for (int p = 0; p < Npoly; p++) z[(size_t)p * m + i] = Bf[p] * y;
  }
}
// BZ[i] = sum_p c[i's cluster][p] z[p][i] ; Y <- Y - rho BZ ; partial sums of |J-BZ|^2 and |BZ-BZold|^2
__global__ void __launch_bounds__(256)
k_consensus_apply(const double *__restrict__ z, const double *__restrict__ cw,
                  const int *__restrict__ clus_of, const double *__restrict__ rho_i,
                  const double *__restrict__ J, double *__restrict__ Y, double *__restrict__ BZ,
                  int m, int Npoly, double *acc) {
  double pr = 0.0, du = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
    const double *c = cw + (size_t)clus_of[i] * Npoly;
    double bz = 0.0;
    for (int p = 0; p < Npoly; p++) bz = fma(c[p], z[(size_t)p * m + i], bz);
    const double old = BZ[i];
    BZ[i] = bz;
    Y[i] = fma(-rho_i[i], bz, Y[i]);
    pr = fma(J[i] - bz, J[i] - bz, pr);
    du = fma(bz - old, bz - old, du);
  }
  pr = warp_sum(pr);
  du = warp_sum(du);
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(acc, pr);
    atomicAdd(acc + 1, du);
  }
}

// One consensus exchange for this rank's subband.  J, Y, BZ: host vectors of npar doubles (the layout
// of pp); rho[M]; Bf[Npoly] = this subband's row of the basis; Bi[M][Npoly][Npoly].  On return
// Y = Y_in + rho (J - B_f Z), BZ = B_f Z; *primal = ||J - B_f Z||, *dual = ||B_f Z - B_f Z_old||.
extern "C" int dirac_b200_consensus_step(dirac_b200_problem *pr, const double *J, double *Y,
                                         double *BZ, const double *rho, const double *Bf,
                                         const double *Bi, int Npoly, double *primal, double *dual) {
  DevProblem &d = pr->d;
  const int m = (int)d.npar;
  const int N8 = 8 * d.N;
  // per-parameter cluster index and rho; per-cluster weights c_k = Bi_k B_f
  std::vector<int> clus_of(m);
  std::vector<double> rho_i(m), cw((size_t)d.M * Npoly);
  for (int k = 0; k < d.M; k++) {
    for (int ck = 0; ck < d.h_clus[k].nchunk; ck++) {
      const int off = d.h_chunk_poff[d.h_clus[k].chunk0 + ck];
      for (int i = 0; i < N8; i++) {
        clus_of[off + i] = k;
        rho_i[off + i] = rho[k];
      }
    }
    for (int p = 0; p < Npoly; p++) {
      double s = 0.0;
      for (int q = 0; q < Npoly; q++) s += Bi[(size_t)k * Npoly * Npoly + p * Npoly + q] * Bf[q];
      cw[(size_t)k * Npoly + p] = s;
    }
  }
  double *dJ = (double *)db_malloc(sizeof(double) * ((size_t)m * (3 + Npoly) + 8));
  double *dY = dJ + m, *dBZ = dY + m, *dz = dBZ + m, *dacc = dz + (size_t)m * Npoly;
  double *drho = (double *)db_malloc(sizeof(double) * ((size_t)m + d.M * Npoly + Npoly));
  double *dcw = drho + m, *dBf = dcw + (size_t)d.M * Npoly;
  int *dclus = (int *)db_malloc(sizeof(int) * (size_t)m);
  cudaStream_t st = d.stream;
  DB_CHECK(cudaMemcpyAsync(dJ, J, sizeof(double) * m, cudaMemcpyHostToDevice, st));
  DB_CHECK(cudaMemcpyAsync(dY, Y, sizeof(double) * m, cudaMemcpyHostToDevice, st));
  DB_CHECK(cudaMemcpyAsync(dBZ, BZ, sizeof(double) * m, cudaMemcpyHostToDevice, st));
  DB_CHECK(cudaMemcpyAsync(drho, rho_i.data(), sizeof(double) * m, cudaMemcpyHostToDevice, st));
  DB_CHECK(cudaMemcpyAsync(dcw, cw.data(), sizeof(double) * d.M * Npoly, cudaMemcpyHostToDevice, st));
  DB_CHECK(cudaMemcpyAsync(dBf, Bf, sizeof(double) * Npoly, cudaMemcpyHostToDevice, st));
  DB_CHECK(cudaMemcpyAsync(dclus, clus_of.data(), sizeof(int) * m, cudaMemcpyHostToDevice, st));
  DB_CHECK(cudaMemsetAsync(dacc, 0, 2 * sizeof(double), st));
  const int grid = (m + 255) / 256 < 592 ? (m + 255) / 256 : 592;
  k_consensus_form<<<grid, 256, 0, st>>>(dJ, dY, dz, drho, dBf, m, Npoly);
  // the sum over subbands: ONE all-reduce of Npoly*8*N*Mt doubles (sagecal_master.cpp:844-850)
  db_allreduce_world(pr, dz, (long long)m * Npoly);
  k_consensus_apply<<<grid, 256, 0, st>>>(dz, dcw, dclus, drho, dJ, dY, dBZ, m, Npoly, dacc);
  db_count_launch(2);
  double hacc[2];
  DB_CHECK(cudaMemcpyAsync(Y, dY, sizeof(double) * m, cudaMemcpyDeviceToHost, st));
  DB_CHECK(cudaMemcpyAsync(BZ, dBZ, sizeof(double) * m, cudaMemcpyDeviceToHost, st));
  DB_CHECK(cudaMemcpyAsync(hacc, dacc, 2 * sizeof(double), cudaMemcpyDeviceToHost, st));
  db_stream_sync(st);
  DB_CHECK(cudaGetLastError());
  if (primal) *primal = sqrt(hacc[0]);
  if (dual) *dual = sqrt(hacc[1]);
  db_free(dJ);
  db_free(drho);
  db_free(dclus);
  return 0;
}

// ---- the J-update of one ADMM iteration ---------------------------------------------------------------
// replaces sagefit_visibilities_admm (Dirac.h:1521, admm_solve.c:221-420): the SAGE sweep over the
// clusters with the consensus terms in every cluster's cost.  The reference solves each cluster's
// sub-problem with its Riemannian trust-region solver (rtr_solve_nocuda_robust_admm); this library
// solves the same augmented cost with its Levenberg-Marquardt (Gauss-Newton system with rho/2 on the
// diagonal and y/2 + rho/2 (p - bz) in the right-hand side), so iterates differ from the reference's
// while the fixed point of the ADMM iteration is the same.  No LBFGS stage (the reference has none).
extern "C" int dirac_b200_sagefit_admm(dirac_b200_problem *pr, double *pp, double *x_out,
                                       const double *Y, const double *BZ, const double *admm_rho,
                                       int max_emiter, int max_iter, int linsolv, int randomize,
                                       double *res_0, double *res_1) {
  DevProblem &d = pr->d;
  const size_t m = (size_t)d.npar;
  pr->aug_dev = (double *)db_malloc(sizeof(double) * 2 * m);
  DB_CHECK(cudaMemcpyAsync(pr->aug_dev, Y, sizeof(double) * m, cudaMemcpyHostToDevice, d.stream));
  DB_CHECK(cudaMemcpyAsync(pr->aug_dev + m, BZ, sizeof(double) * m, cudaMemcpyHostToDevice, d.stream));
  pr->aug_y_host = Y;
  pr->aug_bz_host = BZ;
  pr->aug_rho = admm_rho;
  double nu = 0.0;
  const int rv = dirac_b200_sagefit(pr, pp, x_out, max_emiter, max_iter, 0, 0, linsolv, SM_LM_LBFGS,
                                    2.0, 30.0, randomize, &nu, res_0, res_1);
  db_stream_sync(d.stream);
  db_free(pr->aug_dev);
  pr->aug_dev = nullptr;
  pr->aug_y_host = pr->aug_bz_host = pr->aug_rho = nullptr;
  return rv;
}

// The J-update as the reference does it (admm_solve.c:221-420): every cluster visit is the robust
// Riemannian trust-region solver on the consensus-augmented cost (rtr_solve_nocuda_robust_admm: the
// flow of solver_mode 5 in Euclidean space, rtr_algo.h), whatever solver_mode the caller names; no
// LBFGS stage; mean nu as in the robust modes.
extern "C" int dirac_b200_sagefit_admm_rtr(dirac_b200_problem *pr, double *pp, double *x_out,
                                           const double *Y, const double *BZ,
                                           const double *admm_rho, int max_emiter, int max_iter,
                                           double nulow, double nuhigh, int randomize,
                                           double *mean_nu, double *res_0, double *res_1) {
  pr->aug_y_host = Y;
  pr->aug_bz_host = BZ;
  pr->aug_rho = admm_rho;
  const int rv = dirac_b200_sagefit(pr, pp, x_out, max_emiter, max_iter, 0, 0, 0, 7 /* SM_RTR_ADMM_ */,
                                    nulow, nuhigh, randomize, mean_nu, res_0, res_1);
  db_stream_sync(pr->d.stream);
  pr->aug_y_host = pr->aug_bz_host = pr->aug_rho = nullptr;
  return rv;
}

extern "C" int sagefit_visibilities_admm(double *u, double *v, double *w, double *x, int N, int Nbase,
                                         int tilesz, baseline_t *barr, clus_source_t *carr,
                                         double *coh, int M, int Mt, double freq0, double fdelta,
                                         double *pp, double *Y, double *BZ, double uvmin, int Nt,
                                         int max_emiter, int max_iter, int max_lbfgs, int lbfgs_m,
                                         int gpu_threads, int linsolv, int solver_mode, double nulow,
                                         double nuhigh, int randomize, double *admm_rho,
                                         double *mean_nu, double *res_0, double *res_1) {
  (void)u; (void)v; (void)w; (void)freq0; (void)fdelta; (void)uvmin; (void)Nt; (void)max_lbfgs;
  (void)lbfgs_m; (void)gpu_threads; (void)solver_mode;
  dirac_b200_problem *pr = dirac_b200_create(N, Nbase, tilesz, barr, carr, M, Mt, coh, x);
  int rv;
  if (db_opt(DB_OPT_ADMM_LM)) {  // this library's LM on the augmented cost (round-2 default until RTR)
    rv = dirac_b200_sagefit_admm(pr, pp, x, Y, BZ, admm_rho, max_emiter, max_iter, linsolv, randomize,
                                 res_0, res_1);
    *mean_nu = nulow;
  } else {
    rv = dirac_b200_sagefit_admm_rtr(pr, pp, x, Y, BZ, admm_rho, max_emiter, max_iter, nulow, nuhigh,
                                     randomize, mean_nu, res_0, res_1);
  }
  dirac_b200_destroy(pr);
  return rv;
}
extern "C" int sagefit_visibilities_admm_dual_pt_flt(
    double *u, double *v, double *w, double *x, int N, int Nbase, int tilesz, baseline_t *barr,
    clus_source_t *carr, double *coh, int M, int Mt, double freq0, double fdelta, double *pp,
    double *Y, double *BZ, double uvmin, int Nt, int max_emiter, int max_iter, int max_lbfgs,
    int lbfgs_m, int gpu_threads, int linsolv, int solver_mode, double nulow, double nuhigh,
    int randomize, double *admm_rho, double *mean_nu, double *res_0, double *res_1) {
  return sagefit_visibilities_admm(u, v, w, x, N, Nbase, tilesz, barr, carr, coh, M, Mt, freq0, fdelta,
                                   pp, Y, BZ, uvmin, Nt, max_emiter, max_iter, max_lbfgs, lbfgs_m,
                                   gpu_threads, linsolv, solver_mode, nulow, nuhigh, randomize,
                                   admm_rho, mean_nu, res_0, res_1);
}
