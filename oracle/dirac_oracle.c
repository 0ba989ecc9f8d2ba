/* TEST INFRASTRUCTURE ONLY — CPU restatement ("oracle") of the Dirac calibration hot path.
 * See dirac_oracle.h.  Pinned against the compiled reference by tests/test_oracle_vs_ref.py.
 * Citations are reference file:line (relative to /root/reference/src/lib). */
#include "dirac_oracle.h"

#include <float.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

typedef double complex cplx;

static void *xcalloc(size_t n, size_t s) {
  void *p = calloc(n ? n : 1, s);
  if (!p) {
    fprintf(stderr, "%s: %d: no free memory\n", __FILE__, __LINE__);
    exit(1);
  }
  return p;
}

/* ---- index helpers (Dirac/baseline_utils.c:438-466, :206-227) -------------------------------- */
void orc_generate_baselines(int Nbase, int tilesz, int N, int *sta1, int *sta2) {
  for (int t = 0; t < tilesz; t++) {
    int a = 0, b = 1;
    for (int cj = 0; cj < Nbase; cj++) {
      sta1[t * Nbase + cj] = a;
      sta2[t * Nbase + cj] = b;
      if (b < N - 1) {
        b++;
      } else if (a < N - 2) {
        a++;
        b = a + 1;
      } else {
        a = 0;
        b = 1;
      }
    }
  }
}

void orc_preset_flags_and_data(int n, const double *flag, unsigned char *bflag, double *x) {
  for (int ci = 0; ci < n; ci++) {
    if (flag[ci] > 0.0) {
      bflag[ci] = 1;
      for (int c = 0; c < 8; c++) x[8 * ci + c] = 0.0;
    } else {
      bflag[ci] = 0;
    }
  }
}

/* ---- 2x2 products (Dirac/lmfit.c:37-58) -------------------------------------------------------- */
static void amb(const cplx *a, const cplx *b, cplx *c) {
  c[0] = a[0] * b[0] + a[1] * b[2];
  c[1] = a[0] * b[1] + a[1] * b[3];
  c[2] = a[2] * b[0] + a[3] * b[2];
  c[3] = a[2] * b[1] + a[3] * b[3];
}
static void ambt(const cplx *a, const cplx *b, cplx *c) {
  c[0] = a[0] * conj(b[0]) + a[1] * conj(b[1]);
  c[1] = a[0] * conj(b[2]) + a[1] * conj(b[3]);
  c[2] = a[2] * conj(b[0]) + a[3] * conj(b[1]);
  c[3] = a[2] * conj(b[2]) + a[3] * conj(b[3]);
}
static void jones_of(const double *pblk, int sta, cplx *G) {
  const double *s = pblk + 8 * sta;
  G[0] = s[0] + _Complex_I * s[1];
  G[1] = s[2] + _Complex_I * s[3];
  G[2] = s[4] + _Complex_I * s[5];
  G[3] = s[6] + _Complex_I * s[7];
}
static void model_row(const cplx *G1, const cplx *C, const cplx *G2, cplx *T2) {
  cplx T1[4];
  amb(G1, C, T1);
  ambt(T1, G2, T2);
}

/* chunk of a row in the predict path: row / ceil(Nbase1/nchunk)  (Dirac/lmfit.c:86,655) */
static int predict_chunk(long row, long Nbase1, int nchunk) {
  return (int)(row / ((Nbase1 + nchunk - 1) / nchunk));
}

/* ---- minimize_viz_full_pth (Dirac/lmfit.c:611-688) ------------------------------------------- */
void orc_predict_full(const orc_problem *P, const double *pp, double *out) {
  const long R = (long)P->Nbase * P->tilesz;
  const int M = P->M;
  for (long r = 0; r < R; r++) {
    double *o = out + 8 * r;
    memset(o, 0, 8 * sizeof(double));
    if (P->flag[r]) continue;
    for (int k = 0; k < M; k++) {
      int px = predict_chunk(r, R, P->nchunk[k]);
      const double *pblk = pp + P->chunk_off[P->chunk0[k] + px];
      cplx G1[4], G2[4], T2[4];
      jones_of(pblk, P->sta1[r], G1);
      jones_of(pblk, P->sta2[r], G2);
      model_row(G1, P->coh + 4 * ((size_t)M * r + k), G2, T2);
      for (int c = 0; c < 4; c++) {
        o[2 * c] += creal(T2[c]);
        o[2 * c + 1] += cimag(T2[c]);
      }
    }
  }
}

/* ---- mylm_fit_single_pth: one cluster, hybrid aware (Dirac/lmfit.c:64-124) -------------------- */
void orc_predict_cluster(const orc_problem *P, int k, const double *pp, double *out) {
  const long R = (long)P->Nbase * P->tilesz;
  for (long r = 0; r < R; r++) {
    double *o = out + 8 * r;
    memset(o, 0, 8 * sizeof(double));
    if (P->flag[r]) continue;
    int px = predict_chunk(r, R, P->nchunk[k]);
    const double *pblk = pp + P->chunk_off[P->chunk0[k] + px];
    cplx G1[4], G2[4], T2[4];
    jones_of(pblk, P->sta1[r], G1);
    jones_of(pblk, P->sta2[r], G2);
    model_row(G1, P->coh + 4 * ((size_t)P->M * r + k), G2, T2);
    for (int c = 0; c < 4; c++) {
      o[2 * c] = creal(T2[c]);
      o[2 * c + 1] = cimag(T2[c]);
    }
  }
}

/* ---- mylm_fit_single_pth0: one cluster, tiles [t0,t0+ntiles), one parameter block
 * (Dirac/lmfit.c:233-296,300-384); out has 8*ntiles*Nbase values ------------------------------ */
void orc_predict_chunk(const orc_problem *P, int k, int t0, int ntiles, const double *pblk,
                       double *out) {
  const long r0 = (long)t0 * P->Nbase, nr = (long)ntiles * P->Nbase;
  for (long i = 0; i < nr; i++) {
    long r = r0 + i;
    double *o = out + 8 * i;
    memset(o, 0, 8 * sizeof(double));
    if (P->flag[r]) continue;
    cplx G1[4], G2[4], T2[4];
    jones_of(pblk, P->sta1[r], G1);
    jones_of(pblk, P->sta2[r], G2);
    model_row(G1, P->coh + 4 * ((size_t)P->M * r + k), G2, T2);
    for (int c = 0; c < 4; c++) {
      o[2 * c] = creal(T2[c]);
      o[2 * c + 1] = cimag(T2[c]);
    }
  }
}

/* ---- cost_func / robust_cost_func (Dirac/robust_lbfgs.c:674-694,707-726,67-85) ---------------- */
double orc_cost(const orc_problem *P, const double *pp, const double *x, int robust, double nu) {
  const long n = 8l * P->Nbase * P->tilesz;
  double *f = (double *)xcalloc(n, sizeof(double));
  orc_predict_full(P, pp, f);
  double s = 0.0;
  if (!robust) {
    for (long i = 0; i < n; i++) {
      double e = x[i] - f[i];
      s += e * e;
    }
  } else {
    const double inv_nu = 1.0 / nu;
    for (long i = 0; i < n; i++) {
      double e = x[i] - f[i];
      s += log(1.0 + e * e * inv_nu);
    }
  }
  free(f);
  return s;
}

/* ---- func_grad / func_grad_robust (Dirac/robust_lbfgs.c:569-669,322-416) ----------------------
 * The reference loops per PARAMETER over all rows (cpu_calc_deriv, :424-560; _robust :155-316).
 * Here the same sum is accumulated row by row: for each row and cluster the 16 parameters of its
 * two stations receive sum_i r_i * d f_i / d theta, with
 *   Gaussian: g += -2 Re(conj(x) . dV),  x = model - data              (:536-554)
 *   robust  : g += +2 sum_i x_i dV_i/(nu + x_i^2)                      (:286-299)
 * and the chunk of a row taken per TILE: (row/Nbase)/ceil(tilesz/nchunk) (:464-470, SURVEY 3.5-3) */
void orc_grad(const orc_problem *P, const double *pp, const double *x, double *g, int robust,
              double nu) {
  const long R = (long)P->Nbase * P->tilesz;
  const long n = 8 * R;
  const int M = P->M, N = P->N;
  double *f = (double *)xcalloc(n, sizeof(double));
  orc_predict_full(P, pp, f);
  for (long i = 0; i < n; i++) f[i] -= x[i]; /* x <- model - data (:599) */
  memset(g, 0, sizeof(double) * 8 * N * P->Mt);
  for (long r = 0; r < R; r++) {
    if (P->flag[r]) continue;
    const double *xr = f + 8 * r;
    double wr[8];
    for (int c = 0; c < 8; c++) wr[c] = robust ? xr[c] / (nu + xr[c] * xr[c]) : xr[c];
    const int s1 = P->sta1[r], s2 = P->sta2[r];
    const int ttile = (int)(r / P->Nbase);
    for (int k = 0; k < M; k++) {
      const int nchunk = P->nchunk[k];
      const int tilesperchunk = (P->tilesz + nchunk - 1) / nchunk;
      const int tpchunk = ttile / tilesperchunk;
      const int off = P->chunk_off[P->chunk0[k]] + tpchunk * 8 * N; /* pstart + tpchunk*8N (:476) */
      const double *pblk = pp + off;
      cplx G1[4], G2[4], E[4], T2[4];
      jones_of(pblk, s1, G1);
      jones_of(pblk, s2, G2);
      const cplx *C = P->coh + 4 * ((size_t)M * r + k);
      for (int stoff = 0; stoff < 8; stoff++) {
        /* d/d(parameter stoff of station s1): G1 -> unit matrix E (:497-512) */
        memset(E, 0, sizeof(E));
        E[stoff / 2] = (stoff & 1) ? _Complex_I : 1.0;
        model_row(E, C, G2, T2);
        double d = 0.0;
        for (int c = 0; c < 4; c++) d += wr[2 * c] * creal(T2[c]) + wr[2 * c + 1] * cimag(T2[c]);
        g[off + 8 * s1 + stoff] += (robust ? 2.0 : -2.0) * d;
        /* d/d(parameter stoff of station s2) (:513-527) */
        model_row(G1, C, E, T2);
        d = 0.0;
        for (int c = 0; c < 4; c++) d += wr[2 * c] * creal(T2[c]) + wr[2 * c + 1] * cimag(T2[c]);
        g[off + 8 * s2 + stoff] += (robust ? 2.0 : -2.0) * d;
      }
    }
  }
  free(f);
}

/* ---- normal equations of one cluster / tile range --------------------------------------------
 * Row-wise restatement of jacobian_threadfn (Dirac/lmfit.c:392-474) followed by
 * J^T J = dgemm, J^T e = dgemv (Dirac/clmfit.c:307-315); optional row weights wt (sqrt weights of
 * the robust LM, Dirac/robustlm.c:2298-2316: J <- wt.J, e <- wt.e).  xd, wt: 8*ntiles*Nbase values
 * of the tile range.  JTJ is 8N x 8N (symmetric), JTe 8N.  returns ||wt.e||^2. */
double orc_normal_eq(const orc_problem *P, int k, int t0, int ntiles, const double *pblk,
                     const double *xd, const double *wt, double *JTJ, double *JTe) {
  const int N = P->N, n8 = 8 * N;
  const long r0 = (long)t0 * P->Nbase, nr = (long)ntiles * P->Nbase;
  memset(JTJ, 0, sizeof(double) * n8 * n8);
  memset(JTe, 0, sizeof(double) * n8);
  double cost = 0.0;
  for (long i = 0; i < nr; i++) {
    const long r = r0 + i;
    double e[8];
    cplx G1[4], G2[4], T2[4], E[4];
    const int s1 = P->sta1[r], s2 = P->sta2[r];
    const cplx *C = P->coh + 4 * ((size_t)P->M * r + k);
    jones_of(pblk, s1, G1);
    jones_of(pblk, s2, G2);
    if (P->flag[r]) {
      for (int c = 0; c < 8; c++) {
        double w = wt ? wt[8 * i + c] : 1.0;
        e[c] = w * xd[8 * i + c];
        cost += e[c] * e[c];
      }
      continue; /* Jacobian rows of flagged data are zero (:413) */
    }
    model_row(G1, C, G2, T2);
    for (int c = 0; c < 4; c++) {
      double w0 = wt ? wt[8 * i + 2 * c] : 1.0, w1 = wt ? wt[8 * i + 2 * c + 1] : 1.0;
      e[2 * c] = w0 * (xd[8 * i + 2 * c] - creal(T2[c]));
      e[2 * c + 1] = w1 * (xd[8 * i + 2 * c + 1] - cimag(T2[c]));
      cost += e[2 * c] * e[2 * c] + e[2 * c + 1] * e[2 * c + 1];
    }
    double A[8][16]; /* local Jacobian: columns 0..7 station s1, 8..15 station s2 */
    for (int stoff = 0; stoff < 8; stoff++) {
      memset(E, 0, sizeof(E));
      E[stoff / 2] = (stoff & 1) ? _Complex_I : 1.0;
      model_row(E, C, G2, T2);
      for (int c = 0; c < 4; c++) {
        A[2 * c][stoff] = creal(T2[c]);
        A[2 * c + 1][stoff] = cimag(T2[c]);
      }
      model_row(G1, C, E, T2);
      for (int c = 0; c < 4; c++) {
        A[2 * c][8 + stoff] = creal(T2[c]);
        A[2 * c + 1][8 + stoff] = cimag(T2[c]);
      }
    }
    if (wt)
      for (int c = 0; c < 8; c++)
        for (int a = 0; a < 16; a++) A[c][a] *= wt[8 * i + c];
    int col[16];
    for (int a = 0; a < 8; a++) {
      col[a] = 8 * s1 + a;
      col[8 + a] = 8 * s2 + a;
    }
    for (int a = 0; a < 16; a++) {
      double je = 0.0;
      for (int c = 0; c < 8; c++) je += A[c][a] * e[c];
      JTe[col[a]] += je;
      for (int b = 0; b < 16; b++) {
        double s = 0.0;
        for (int c = 0; c < 8; c++) s += A[c][a] * A[c][b];
        JTJ[(size_t)col[a] * n8 + col[b]] += s;
      }
    }
  }
  return cost;
}

/* ---- normal equations of ONE ordered subset with the reference's own pairing -------------------
 * oslevmar / osrlevmar (Dirac/clmfit.c:1313-1413, robustlm.c:2835-2935) split the n data of a chunk
 * into Nsubsets pieces of Npersubset = ceil(n/Nsubsets) reals AND its tiles into pieces of
 * Ntpersubset = ceil(ntiles/Nsubsets) tiles.  Subset l gets the Jacobian of ITS TILES, cut (or
 * zero padded: jacf memsets Nos[l] rows first, lmfit.c:524) to Nos[l] rows, the residual slice
 * ed[edI[l] .. edI[l]+Nos[l]) and, in the robust variant, the weights wtd[edI[l] + row].  The two
 * offsets coincide only when ntiles is a multiple of Nsubsets (or < 10); otherwise row i of J meets
 * the residual / weight of data index edI[l] + i, which belongs to another tile, baseline and even
 * polarisation component.  Reproduced literally.
 * e_full: the chunk's residual as the LM holds it (weighted in the robust variant), wt: the chunk's
 * sqrt-weights or NULL. */
void orc_normal_eq_os(const orc_problem *P, int k, int t0, int ntiles, const double *pblk,
                      const double *e_full, const double *wt, int l, double *JTJ, double *JTe) {
  const int N = P->N, n8 = 8 * N;
  const long n = 8l * ntiles * P->Nbase;
  int Nsubsets = 10;
  if (ntiles < Nsubsets) Nsubsets = ntiles;
  const long Nper = (n + Nsubsets - 1) / Nsubsets;
  const int Ntper = (ntiles + Nsubsets - 1) / Nsubsets;
  const long kl = (long)l * Nper;
  const int tl = l * Ntper;
  long Nos;
  int tileI;
  if (tl + Ntper < ntiles) {
    Nos = Nper;
    tileI = Ntper;
  } else {
    Nos = n - kl;
    tileI = ntiles - tl;
  }
  memset(JTJ, 0, sizeof(double) * n8 * n8);
  memset(JTe, 0, sizeof(double) * n8);
  long nJ = (tileI > 0) ? 8l * P->Nbase * tileI : 0;
  if (Nos < nJ) nJ = Nos;
  for (long i0 = 0; i0 < nJ; i0 += 8) {
    const long r = (long)(t0 + tl) * P->Nbase + i0 / 8;
    if (P->flag[r]) continue; /* Jacobian rows of flagged data are zero */
    cplx G1[4], G2[4], T2[4], E[4];
    const int s1 = P->sta1[r], s2 = P->sta2[r];
    const cplx *C = P->coh + 4 * ((size_t)P->M * r + k);
    jones_of(pblk, s1, G1);
    jones_of(pblk, s2, G2);
    double A[8][16];
    for (int stoff = 0; stoff < 8; stoff++) {
      memset(E, 0, sizeof(E));
      E[stoff / 2] = (stoff & 1) ? _Complex_I : 1.0;
      model_row(E, C, G2, T2);
      for (int c = 0; c < 4; c++) {
        A[2 * c][stoff] = creal(T2[c]);
        A[2 * c + 1][stoff] = cimag(T2[c]);
      }
      model_row(G1, C, E, T2);
      for (int c = 0; c < 4; c++) {
        A[2 * c][8 + stoff] = creal(T2[c]);
        A[2 * c + 1][8 + stoff] = cimag(T2[c]);
      }
    }
    int col[16];
    for (int a = 0; a < 8; a++) {
      col[a] = 8 * s1 + a;
      col[8 + a] = 8 * s2 + a;
    }
    const int nc = (nJ - i0 < 8) ? (int)(nJ - i0) : 8; /* the cut may fall inside a row */
    for (int c = 0; c < nc; c++) {
      const long g = kl + i0 + c; /* the data index this Jacobian row is paired with */
      const double w = wt ? wt[g] : 1.0;
      const double eg = e_full[g];
      for (int a = 0; a < 16; a++) {
        const double ja = w * A[c][a];
        JTe[col[a]] += ja * eg;
        for (int b = 0; b < 16; b++) JTJ[(size_t)col[a] * n8 + col[b]] += ja * (w * A[c][b]);
      }
    }
  }
}

/* ---- dense symmetric solvers ------------------------------------------------------------------ */
/* Cholesky A = L L^T in place (lower), returns 0 or the failing pivot index+1 (dpotrf) */
static int chol_factor(double *A, int n) {
  for (int j = 0; j < n; j++) {
    double d = A[(size_t)j * n + j];
    for (int k = 0; k < j; k++) d -= A[(size_t)j * n + k] * A[(size_t)j * n + k];
    if (!(d > 0.0)) return j + 1;
    d = sqrt(d);
    A[(size_t)j * n + j] = d;
    for (int i = j + 1; i < n; i++) {
      double s = A[(size_t)i * n + j];
      for (int k = 0; k < j; k++) s -= A[(size_t)i * n + k] * A[(size_t)j * n + k];
      A[(size_t)i * n + j] = s / d;
    }
  }
  return 0;
}
static void chol_solve(const double *L, int n, double *b) {
  for (int i = 0; i < n; i++) {
    double s = b[i];
    for (int k = 0; k < i; k++) s -= L[(size_t)i * n + k] * b[k];
    b[i] = s / L[(size_t)i * n + i];
  }
  for (int i = n - 1; i >= 0; i--) {
    double s = b[i];
    for (int k = i + 1; k < n; k++) s -= L[(size_t)k * n + i] * b[k];
    b[i] = s / L[(size_t)i * n + i];
  }
}
/* Householder QR solve of the square system (dgels), A destroyed; returns 0 if solved */
static int qr_solve(double *A, int n, double *b) {
  for (int k = 0; k < n; k++) {
    double nrm = 0.0;
    for (int i = k; i < n; i++) nrm += A[(size_t)i * n + k] * A[(size_t)i * n + k];
    nrm = sqrt(nrm);
    if (nrm == 0.0) return k + 1;
    double alpha = (A[(size_t)k * n + k] > 0.0) ? -nrm : nrm;
    double v0 = A[(size_t)k * n + k] - alpha;
    A[(size_t)k * n + k] = v0;
    double vnorm2 = 0.0;
    for (int i = k; i < n; i++) vnorm2 += A[(size_t)i * n + k] * A[(size_t)i * n + k];
    if (vnorm2 > 0.0) {
      for (int j = k + 1; j < n; j++) {
        double s = 0.0;
        for (int i = k; i < n; i++) s += A[(size_t)i * n + k] * A[(size_t)i * n + j];
        s = 2.0 * s / vnorm2;
        for (int i = k; i < n; i++) A[(size_t)i * n + j] -= s * A[(size_t)i * n + k];
      }
      double s = 0.0;
      for (int i = k; i < n; i++) s += A[(size_t)i * n + k] * b[i];
      s = 2.0 * s / vnorm2;
      for (int i = k; i < n; i++) b[i] -= s * A[(size_t)i * n + k];
    }
    A[(size_t)k * n + k] = alpha;
    for (int i = k + 1; i < n; i++) A[(size_t)i * n + k] = 0.0;
  }
  for (int i = n - 1; i >= 0; i--) {
    double s = b[i];
    for (int j = i + 1; j < n; j++) s -= A[(size_t)i * n + j] * b[j];
    if (A[(size_t)i * n + i] == 0.0) return i + 1;
    b[i] = s / A[(size_t)i * n + i];
  }
  return 0;
}

static double nrm2sq(const double *v, long n) {
  double s = 0.0;
  for (long i = 0; i < n; i++) s += v[i] * v[i];
  return s;
}

/* weighted residual e = wt.(xd - f(p)) over the tile range, returns ||e||^2 */
static double chunk_residual(const orc_problem *P, int k, int t0, int ntiles, const double *p,
                             const double *xd, const double *wt, double *e) {
  const long n = 8l * ntiles * P->Nbase;
  orc_predict_chunk(P, k, t0, ntiles, p, e);
  for (long i = 0; i < n; i++) {
    e[i] = xd[i] - e[i];
    if (wt) e[i] *= wt[i];
  }
  return nrm2sq(e, n);
}

/* ---- the LM core shared by clevmar / oslevmar / rlevmar / osrlevmar -----------------------------
 * One call = the "iteration loop" of Dirac/clmfit.c:241-540 (os=0) or :1281-1640 (os=1) with
 * optional sqrt-weights wt (Dirac/robustlm.c:2233-2420).  State that the robust driver carries
 * across its IRLS rounds (nu_damp, mu) is passed by pointer.  e_last receives the residual of the
 * last function evaluation (the reference's `ed`, which a rejected trial overwrites,
 * Dirac/clmfit.c:478 "note: e is updated"). */
typedef struct {
  double init_eL2, eL2, jacTe_inf, Dp_L2, mu;
  int k, stop;
} lm_out;

/* Number of LM accept/reject decisions taken at rounding level since the last reset.  The OS
 * variants reject trial steps along a subset's gradient until the step is ~1e-15 |p|; whether the
 * last of them counts as an improvement is rounding noise, yet it resets mu and nu and so steers
 * everything after it (the compiled reference and this restatement part ways on such cases).  Parity
 * to 1e-5 is only defined for runs in which this counter stays 0. */
static long g_noise_decisions = 0;
long orc_noise_decisions(int reset) {
  long v = g_noise_decisions;
  if (reset) g_noise_decisions = 0;
  return v;
}

static void lm_core(const orc_problem *P, int k, int t0, int ntiles, double *p, const double *xd,
                    const double *wt, int itmax, const double *opts, int linsolv, int os,
                    int os_shift, int *nu_damp, double *e_last, lm_out *out) {
  const int n8 = 8 * P->N;
  const long n = 8l * ntiles * P->Nbase;
  const double tau = opts[0], eps1 = opts[1], eps2 = opts[2], eps2_sq = opts[2] * opts[2],
               eps3 = opts[3];
  double *JTJ0 = (double *)xcalloc((size_t)n8 * n8, sizeof(double));
  double *JTJ = (double *)xcalloc((size_t)n8 * n8, sizeof(double));
  double *JTe = (double *)xcalloc(n8, sizeof(double));
  double *Dp = (double *)xcalloc(n8, sizeof(double));
  double *pnew = (double *)xcalloc(n8, sizeof(double));
  double p_eL2 = chunk_residual(P, k, t0, ntiles, p, xd, wt, e_last);
  const double init_p_eL2 = p_eL2;
  int stop = 0, nu = *nu_damp, nu2, kiter;
  double mu = 0.0, Dp_L2 = DBL_MAX, jacTe_inf = 0.0;
  if (!isfinite(p_eL2)) stop = 7;
  int Nsubsets = 10, s0 = 0, sn = ntiles;
  if (ntiles < Nsubsets) Nsubsets = ntiles;
  const int max_os_iter = os ? (int)ceil(0.1 * (double)Nsubsets) : 1;
  for (kiter = 0; kiter < itmax && !stop; ++kiter) {
    if (p_eL2 <= eps3) {
      stop = 6;
      break;
    }
    for (int ositer = 0; ositer < max_os_iter; ositer++) {
      if (os) {
        /* subset l with the reference's pairing of Jacobian rows, residual and weights; e_last is
         * the residual of the last function evaluation, i.e. at p here (every exit of the damping
         * loop that continues the iteration is an accepted step) */
        int l = (os_shift + kiter + ositer) % Nsubsets;
        orc_normal_eq_os(P, k, t0, ntiles, p, e_last, wt, l, JTJ0, JTe);
      } else {
        /* J^T J and J^T e; e is the current (weighted) residual */
        const long off = 8l * s0 * P->Nbase;
        orc_normal_eq(P, k, t0 + s0, sn, p, xd + off, wt ? wt + off : NULL, JTJ0, JTe);
      }
      jacTe_inf = 0.0;
      for (int i = 0; i < n8; i++)
        if (fabs(JTe[i]) > jacTe_inf) jacTe_inf = fabs(JTe[i]);
      const double p_L2 = nrm2sq(p, n8);
      if (jacTe_inf <= eps1) {
        Dp_L2 = 0.0;
        stop = 1;
        break;
      }
      if (kiter == 0) {
        double mx = 0.0; /* idamax on the diagonal, value kept signed (clmfit.c:342-352) */
        for (int i = 0; i < n8; i++)
          if (fabs(JTJ0[(size_t)i * n8 + i]) > fabs(mx)) mx = JTJ0[(size_t)i * n8 + i];
        mu = tau * mx;
      }
      while (1) {
        memcpy(JTJ, JTJ0, sizeof(double) * n8 * n8);
        for (int i = 0; i < n8; i++) JTJ[(size_t)i * n8 + i] += mu;
        memcpy(Dp, JTe, sizeof(double) * n8);
        int issolved;
        if (linsolv == 0) {
          issolved = (chol_factor(JTJ, n8) == 0);
          if (issolved) chol_solve(JTJ, n8, Dp);
        } else {
          issolved = (qr_solve(JTJ, n8, Dp) == 0);
        }
        if (issolved) {
          for (int i = 0; i < n8; i++) pnew[i] = p[i] + Dp[i];
          Dp_L2 = nrm2sq(Dp, n8);
          if (Dp_L2 <= eps2_sq * p_L2) {
            stop = 2;
            break;
          }
          if (Dp_L2 >= (p_L2 + eps2) / (1e-12 * 1e-12)) {
            stop = 4;
            break;
          }
          const double pDp_eL2 = chunk_residual(P, k, t0, ntiles, pnew, xd, wt, e_last);
          if (!isfinite(pDp_eL2)) {
            stop = 7;
            break;
          }
          double dL = 0.0;
          for (int i = 0; i < n8; i++) dL += Dp[i] * (mu * Dp[i] + JTe[i]);
          const double dF = p_eL2 - pDp_eL2;
          /* accept / reject decided at rounding level: the sums behind dF differ by ~1e-14 ||e||^2
           * between implementations (summation order), so below that the branch is noise */
          if (fabs(dF) <= 1e-11 * p_eL2) g_noise_decisions++;
          if (dL > 0.0 && dF > 0.0) {
            double tmp = (2.0 * dF / dL - 1.0);
            tmp = 1.0 - tmp * tmp * tmp;
            mu = mu * ((tmp >= 0.3333333334) ? tmp : 0.3333333334);
            nu = 2;
            memcpy(p, pnew, sizeof(double) * n8);
            p_eL2 = pDp_eL2;
            break;
          }
        }
        mu *= (double)nu;
        nu2 = nu << 1;
        if (nu2 <= nu) {
          stop = 5;
          break;
        }
        nu = nu2;
      }
      if (stop) break;
    }
  }
  if (kiter >= itmax) stop = 3;
  (void)n;
  *nu_damp = nu;
  out->init_eL2 = init_p_eL2;
  out->eL2 = p_eL2;
  out->jacTe_inf = jacTe_inf;
  out->Dp_L2 = Dp_L2;
  out->mu = mu;
  out->k = kiter;
  out->stop = stop;
  free(JTJ0); free(JTJ); free(JTe); free(Dp); free(pnew);
}

static void fill_info(double *info, const lm_out *o) {
  if (!info) return;
  info[0] = o->init_eL2; info[1] = o->eL2; info[2] = o->jacTe_inf; info[3] = o->Dp_L2;
  info[4] = o->mu; info[5] = (double)o->k; info[6] = (double)o->stop;
  info[7] = info[8] = info[9] = 0.0;
}

/* clevmar_der_single_nocuda (Dirac/clmfit.c:29) / oslevmar_der_single_nocuda (:1074) */
int orc_lm_chunk(const orc_problem *P, int k, int t0, int ntiles, double *pblk, const double *xd,
                 int itmax, const double *opts, int linsolv, int os, double *info) {
  static const double defopts[4] = {1e-3, 1e-17, 1e-17, 1e-17};
  const long n = 8l * ntiles * P->Nbase;
  double *e = (double *)xcalloc(n, sizeof(double));
  int nu = 2;
  lm_out o;
  lm_core(P, k, t0, ntiles, pblk, xd, NULL, itmax, opts ? opts : defopts, linsolv, os, 0, &nu, e,
          &o);
  fill_info(info, &o);
  free(e);
  return 0;
}

/* digamma (Dirac/updatenu.c:36-49) */
static double digamma_(double x) {
  double result = 0.0, xx, xx2, xx4;
  for (; x < 7.0; ++x) result -= 1.0 / x;
  x -= 0.5;
  xx = 1.0 / x;
  xx2 = xx * xx;
  xx4 = xx2 * xx2;
  result += log(x) + (1. / 24.) * xx2 - (7.0 / 960.0) * xx4 + (31.0 / 8064.0) * xx4 * xx2 -
            (127.0 / 30720.0) * xx4 * xx4;
  return result;
}

/* update_w_and_nu (Dirac/updatenu.c:137-262): w <- sqrt((nu0+1)/(nu0+e^2)), returns the nu of a
 * 30-point grid on [nulow,nuhigh) minimising psi((nu+1)/2)-ln((nu+1)/2)-psi(nu/2)+ln(nu/2)
 * - mean(w - ln w) + 1  (the reference takes idamin = smallest |value|) */
double orc_update_w_and_nu(double nu0, double *w, const double *ed, int n, double nulow,
                           double nuhigh) {
  const int Nd = 30;
  double sumq = 0.0;
  for (int i = 0; i < n; i++) {
    w[i] = (nu0 + 1.0) / (nu0 + ed[i] * ed[i]);
    sumq += fabs(w[i] - log(w[i]));
  }
  sumq /= (double)n;
  for (int i = 0; i < n; i++) w[i] = sqrt(w[i]);
  const double deltanu = (nuhigh - nulow) / (double)Nd;
  int best = 0;
  double bestv = 0.0;
  for (int ci = 0; ci < Nd; ci++) {
    double thisnu = nulow + (double)ci * deltanu;
    double q = digamma_(thisnu * 0.5 + 0.5) - log((thisnu + 1.0) * 0.5);
    q += -digamma_(thisnu * 0.5) + log(thisnu * 0.5);
    q += -sumq + 1.0;
    if (ci == 0 || fabs(q) < bestv) {
      bestv = fabs(q);
      best = ci;
    }
  }
  return nulow + (double)best * deltanu;
}

/* rlevmar_der_single_nocuda (Dirac/robustlm.c:2008) / osrlevmar_der_single_nocuda (:2607):
 * three IRLS rounds of weighted LM with Student's-t weights and nu re-estimated in between */
int orc_rlm_chunk(const orc_problem *P, int k, int t0, int ntiles, double *pblk, const double *xd,
                  int itmax, int linsolv, int os, double nulow, double nuhigh, double *robust_nu,
                  double *info) {
  static const double defopts[4] = {1e-3, 1e-17, 1e-17, 1e-17}; /* opts == NULL (lmfit.c:917) */
  const int wt_itmax = 3;
  const long n = 8l * ntiles * P->Nbase;
  double *wt = (double *)xcalloc(n, sizeof(double));
  double *e = (double *)xcalloc(n, sizeof(double));
  for (long i = 0; i < n; i++) wt[i] = 1.0;
  double nu_t = *robust_nu;
  int nu = 2;
  lm_out o;
  memset(&o, 0, sizeof(o));
  for (int nw = 0; nw < wt_itmax; nw++) {
    lm_core(P, k, t0, ntiles, pblk, xd, wt, itmax, defopts, linsolv, os, nw, &nu, e, &o);
    if (nw > 0 && nw < wt_itmax - 1) {
      /* unweighted residual at the current p (robustlm.c:2538-2545) */
      chunk_residual(P, k, t0, ntiles, pblk, xd, NULL, e);
    }
    if (nw < wt_itmax - 1) {
      double lambda = 0.0;
      for (long i = 0; i < n; i++) lambda += fabs(wt[i]);
      nu_t = orc_update_w_and_nu(nu_t, wt, e, (int)n, nulow, nuhigh);
      const double wt_sum = lambda / (double)n;
      for (long i = 0; i < n; i++) wt[i] *= wt_sum;
    }
  }
  *robust_nu = nu_t;
  fill_info(info, &o);
  free(wt);
  free(e);
  return 0;
}

/* ---- LBFGS (Dirac/lbfgs.c:33-111,116-205,211-290,298-430,479-640) ----------------------------- */
typedef struct {
  const orc_problem *P;
  const double *x;
  int robust;
  double nu;
  long long ncost;  /* cost evaluations so far */
  double margin;    /* smallest decision margin so far, in units of its rounding noise */
} lb_ctx;
static double lb_cost(lb_ctx *c, const double *p) {
  c->ncost++;
  return orc_cost(c->P, p, c->x, c->robust, c->nu);
}
/* One comparison lhs <op> rhs of the line search: its margin |lhs - rhs| over `noise`, the change of
 * lhs - rhs that rounding of the costs behind it can cause (costs known to eps |cost|, a central
 * difference of two costs to eps (|p01| + |p02|) / (2 step)).  The smallest margin of a run says how
 * far every decision was from flipping under a cost computed another way (the product's quartic). */
static void lb_decide(lb_ctx *c, double lhs, double rhs, double noise) {
  if (noise > 0.0 && fabs(lhs - rhs) / noise < c->margin) c->margin = fabs(lhs - rhs) / noise;
}
#define LB_EPS DBL_EPSILON
static double cost_noise(double a, double b) { return LB_EPS * (fabs(a) + fabs(b)); }
static double diff_noise(double p01, double p02, double step) {
  return LB_EPS * (fabs(p01) + fabs(p02)) / (2.0 * step);
}
static double vdot(const double *a, const double *b, int m) {
  double s = 0.0;
  for (int i = 0; i < m; i++) s += a[i] * b[i];
  return s;
}
static void vaxpy(double *y, const double *x, double a, int m) {
  for (int i = 0; i < m; i++) y[i] += a * x[i];
}

void orc_mult_hessian(int m, double *pk, const double *gk, const double *s, const double *y,
                      const double *rho, int M, int ii) {
  double *alphai = (double *)xcalloc(M, sizeof(double));
  int *idx = (int *)xcalloc(M, sizeof(int));
  if (M > 0) {
    ii = (ii > 0) ? ii - 1 : M - 1;
    for (int ci = 0; ci < M - ii - 1; ci++) idx[ci] = ii + ci + 1;
    for (int ci = M - ii - 1; ci < M; ci++) idx[ci] = ci - M + ii + 1;
  }
  memcpy(pk, gk, sizeof(double) * m);
  for (int ci = 0; ci < M; ci++) {
    int j = idx[M - ci - 1];
    alphai[M - ci - 1] = rho[j] * vdot(s + (size_t)m * j, pk, m);
    vaxpy(pk, y + (size_t)m * j, -alphai[M - ci - 1], m);
  }
  if (M > 0) {
    int j = idx[M - 1];
    double gamma = vdot(s + (size_t)m * j, y + (size_t)m * j, m) /
                   vdot(y + (size_t)m * j, y + (size_t)m * j, m);
    for (int i = 0; i < m; i++) pk[i] *= gamma;
  }
  for (int ci = 0; ci < M; ci++) {
    int j = idx[ci];
    double beta = rho[j] * vdot(y + (size_t)m * j, pk, m);
    vaxpy(pk, s + (size_t)m * j, alphai[ci] - beta, m);
  }
  free(alphai);
  free(idx);
}

static double cubic_interp(lb_ctx *c, const double *xk, const double *pk, double a, double b,
                           double *xp, int m, double step) {
  double f0, f1, f0d, f1d, p01, p02, z0, fz0, aa, cc;
  memcpy(xp, xk, sizeof(double) * m);
  vaxpy(xp, pk, a, m);
  f0 = lb_cost(c, xp);
  vaxpy(xp, pk, step, m);
  p01 = lb_cost(c, xp);
  vaxpy(xp, pk, -2.0 * step, m);
  p02 = lb_cost(c, xp);
  f0d = (p01 - p02) / (2.0 * step);
  const double d0 = diff_noise(p01, p02, step);
  vaxpy(xp, pk, -a + step + b, m);
  f1 = lb_cost(c, xp);
  vaxpy(xp, pk, step, m);
  p01 = lb_cost(c, xp);
  vaxpy(xp, pk, -2.0 * step, m);
  p02 = lb_cost(c, xp);
  f1d = (p01 - p02) / (2.0 * step);
  const double d1 = diff_noise(p01, p02, step);
  aa = 3.0 * (f0 - f1) / (b - a) + (f1d - f0d);
  p01 = aa * aa - f0d * f1d;
  const double na = 3.0 * cost_noise(f0, f1) / fabs(b - a) + d0 + d1;
  lb_decide(c, p01, 0.0, 2.0 * fabs(aa) * na + fabs(f1d) * d0 + fabs(f0d) * d1);
  if (p01 > 0.0) {
    const double nd = 2.0 * fabs(aa) * na + fabs(f1d) * d0 + fabs(f0d) * d1;
    cc = sqrt(p01);
    const double num = f1d + cc - aa, den = f1d - f0d + 2.0 * cc, ncc = nd / (2.0 * cc);
    z0 = b - num * (b - a) / den;
    const double nz = fabs(b - a) * ((d1 + ncc + na) / fabs(den) + fabs(num) * (d0 + d1 + 2.0 * ncc) /
                                     (den * den));
    aa = (a > b) ? a : b;
    cc = (a < b) ? a : b;
    lb_decide(c, z0, aa, nz);
    if (!(z0 > aa)) lb_decide(c, z0, cc, nz);
    if (z0 > aa || z0 < cc) {
      fz0 = f0 + f1;
    } else {
      vaxpy(xp, pk, -b + step + a + z0 * (b - a), m);
      fz0 = lb_cost(c, xp);
    }
    lb_decide(c, f0, f1, cost_noise(f0, f1));
    if (f0 < f1) lb_decide(c, f0, fz0, cost_noise(f0, fz0));
    if (f0 < f1 && f0 < fz0) return a;
    lb_decide(c, f1, fz0, cost_noise(f1, fz0));
    if (f1 < fz0) return b;
    return z0;
  }
  lb_decide(c, f0, f1, cost_noise(f0, f1));
  return (f0 < f1) ? a : b;
}

static double ls_zoom(lb_ctx *c, const double *xk, const double *pk, double a, double b, double *xp,
                      double phi_0, double gphi_0, double n0, double sigma, double rho, double t2,
                      double t3, int m, double step) {
  double alphaj = 0.0, phi_j, phi_aj, gphi_j, p01, p02, aj = a, bj = b, alphak = 1.0;
  int ci = 0, found = 0;
  while (ci < 10) {
    p01 = aj + t2 * (bj - aj);
    p02 = bj - t3 * (bj - aj);
    alphaj = cubic_interp(c, xk, pk, p01, p02, xp, m, step);
    memcpy(xp, xk, sizeof(double) * m);
    vaxpy(xp, pk, alphaj, m);
    phi_j = lb_cost(c, xp);
    vaxpy(xp, pk, -alphaj + aj, m);
    phi_aj = lb_cost(c, xp);
    lb_decide(c, phi_j, phi_0 + rho * alphaj * gphi_0,
              cost_noise(phi_j, phi_0) + rho * fabs(alphaj) * n0);
    if (!(phi_j > phi_0 + rho * alphaj * gphi_0)) lb_decide(c, phi_j, phi_aj, cost_noise(phi_j, phi_aj));
    if ((phi_j > phi_0 + rho * alphaj * gphi_0) || phi_j >= phi_aj) {
      bj = alphaj;
    } else {
      vaxpy(xp, pk, -aj + alphaj + step, m);
      p01 = lb_cost(c, xp);
      vaxpy(xp, pk, -2.0 * step, m);
      p02 = lb_cost(c, xp);
      gphi_j = (p01 - p02) / (2.0 * step);
      const double nj = diff_noise(p01, p02, step);
      lb_decide(c, (aj - alphaj) * gphi_j, step, fabs(aj - alphaj) * nj);
      if ((aj - alphaj) * gphi_j <= step) {
        alphak = alphaj;
        found = 1;
        break;
      }
      lb_decide(c, fabs(gphi_j), -sigma * gphi_0, nj + sigma * n0);
      if (fabs(gphi_j) <= -sigma * gphi_0) {
        alphak = alphaj;
        found = 1;
        break;
      }
      lb_decide(c, gphi_j * (bj - aj), 0.0, fabs(bj - aj) * nj);
      if (gphi_j * (bj - aj) >= 0) bj = aj;
      aj = alphaj;
    }
    ci++;
  }
  if (!found) alphak = alphaj;
  return alphak;
}

static double linesearch(lb_ctx *c, const double *xk, const double *pk, double alpha1, double sigma,
                         double rho, double t1, double t2, double t3, int m, double step) {
  double *xp = (double *)xcalloc(m, sizeof(double));
  double alphai, alphai1, phi_0, phi_alphai, phi_alphai1, p01, p02, gphi_0, gphi_i, alphak = 1.0, mu,
                                                                                    tol;
  phi_0 = lb_cost(c, xk);
  tol = (0.01 * phi_0 < 1e-6) ? 0.01 * phi_0 : 1e-6;
  memcpy(xp, xk, sizeof(double) * m);
  vaxpy(xp, pk, step, m);
  p01 = lb_cost(c, xp);
  vaxpy(xp, pk, -2.0 * step, m);
  p02 = lb_cost(c, xp);
  gphi_0 = (p01 - p02) / (2.0 * step);
  const double n0 = diff_noise(p01, p02, step);
  mu = (tol - phi_0) / (rho * gphi_0);
  const double nmu = fabs(mu) * (n0 / fabs(gphi_0) + cost_noise(tol, phi_0) / fabs(tol - phi_0));
  if (!isnormal(mu)) {
    free(xp);
    return mu;
  }
  int ci = 1;
  alphai = alpha1;
  alphai1 = 0.0;
  phi_alphai1 = phi_0;
  while (ci < 10) {
    memcpy(xp, xk, sizeof(double) * m);
    vaxpy(xp, pk, alphai, m);
    phi_alphai = lb_cost(c, xp);
    lb_decide(c, phi_alphai, tol, cost_noise(phi_alphai, tol));
    if (phi_alphai < tol) {
      alphak = alphai;
      break;
    }
    lb_decide(c, phi_alphai, phi_0 + alphai * gphi_0,
              cost_noise(phi_alphai, phi_0) + fabs(alphai) * n0);
    if (!(phi_alphai > phi_0 + alphai * gphi_0) && ci > 1)
      lb_decide(c, phi_alphai, phi_alphai1, cost_noise(phi_alphai, phi_alphai1));
    if ((phi_alphai > phi_0 + alphai * gphi_0) || (ci > 1 && phi_alphai >= phi_alphai1)) {
      alphak = ls_zoom(c, xk, pk, alphai1, alphai, xp, phi_0, gphi_0, n0, sigma, rho, t2, t3, m,
                       step);
      break;
    }
    vaxpy(xp, pk, step, m);
    p01 = lb_cost(c, xp);
    vaxpy(xp, pk, -2.0 * step, m);
    p02 = lb_cost(c, xp);
    gphi_i = (p01 - p02) / (2.0 * step);
    const double ni = diff_noise(p01, p02, step);
    lb_decide(c, fabs(gphi_i), -sigma * gphi_0, ni + sigma * n0);
    if (fabs(gphi_i) <= -sigma * gphi_0) {
      alphak = alphai;
      break;
    }
    lb_decide(c, gphi_i, 0.0, ni);
    if (gphi_i >= 0) {
      alphak = ls_zoom(c, xk, pk, alphai, alphai1, xp, phi_0, gphi_0, n0, sigma, rho, t2, t3, m,
                       step);
      break;
    }
    lb_decide(c, mu, 2.0 * alphai - alphai1, nmu);
    if (mu <= (2.0 * alphai - alphai1)) {
      alphai1 = alphai;
      alphai = mu;
    } else {
      p01 = 2.0 * alphai - alphai1;
      double hi = alphai + t1 * (alphai - alphai1);
      p02 = (mu < hi) ? mu : hi;
      alphai = cubic_interp(c, xk, pk, p01, p02, xp, m, step);
    }
    phi_alphai1 = phi_alphai;
    ci++;
  }
  free(xp);
  return alphak;
}

static double g_lbfgs_margin = HUGE_VAL;
double orc_lbfgs_last_margin(void) { return g_lbfgs_margin; }

void orc_lbfgs_traced(const orc_problem *P, double *pp, const double *x, int itmax, int M,
                      int robust, double nu, orc_lbfgs_trace *tr) {
  const int m = 8 * P->N * P->Mt;
  lb_ctx ctx = {P, x, robust, nu, 0, HUGE_VAL};
  if (tr) tr->niter = 0;
  if (M < 1) M = 1;
  double *gk = (double *)xcalloc(m, sizeof(double)), *xk1 = (double *)xcalloc(m, sizeof(double));
  double *xk = (double *)xcalloc(m, sizeof(double)), *pk = (double *)xcalloc(m, sizeof(double));
  double *s = (double *)xcalloc((size_t)m * M, sizeof(double));
  double *y = (double *)xcalloc((size_t)m * M, sizeof(double));
  double *rho = (double *)xcalloc(M, sizeof(double));
  memcpy(xk, pp, sizeof(double) * m);
  orc_grad(P, xk, x, gk, robust, nu);
  double gradnrm = sqrt(vdot(gk, gk, m));
  double step;
  int ck, ci = 0, cm = 0;
  if (gradnrm < 1e-17) {
    ck = itmax;
    step = 0.0;
  } else {
    ck = 0;
    double t = 1e-3 / gradnrm;
    if (t > 1e-6) t = 1e-6;
    step = (t > 1e-9) ? t : 1e-9;
  }
  while (ck < itmax && isnormal(gradnrm) && gradnrm > 1e-17) {
    const long long ncost0 = ctx.ncost;
    orc_mult_hessian(m, pk, gk, s, y, rho, ck < M ? ck : M, ci);
    for (int i = 0; i < m; i++) pk[i] = -pk[i];
    double alphak = linesearch(&ctx, xk, pk, 10.0, 0.1, 0.01, 9, 0.1, 0.5, m, step);
    if (!isnormal(alphak) || fabs(alphak) < 1e-12) break;
    memcpy(xk1, xk, sizeof(double) * m);
    vaxpy(xk1, pk, alphak, m);
    for (int i = 0; i < m; i++) {
      s[cm + i] = xk1[i] - xk[i];
      y[cm + i] = -gk[i];
    }
    orc_grad(P, xk1, x, gk, robust, nu);
    gradnrm = sqrt(vdot(gk, gk, m));
    vaxpy(y + cm, gk, 1.0, m);
    rho[ci] = 1.0 / vdot(y + cm, s + cm, m);
    memcpy(xk, xk1, sizeof(double) * m);
    if (tr) {
      tr->alphak[ck] = alphak;
      tr->ncost[ck] = ctx.ncost - ncost0;
      tr->slot[ck] = ci;
      tr->gnorm[ck] = gradnrm;
      memcpy(tr->iterates + (size_t)m * ck, xk, sizeof(double) * m);
      tr->niter = ck + 1;
    }
    ck++;
    if (cm < (M - 1) * m) {
      cm += m;
      ci++;
    } else {
      cm = ci = 0;
    }
  }
  memcpy(pp, xk, sizeof(double) * m);
  free(gk); free(xk1); free(xk); free(pk); free(s); free(y); free(rho);
  g_lbfgs_margin = ctx.margin;
  if (tr) tr->margin = ctx.margin;
}

void orc_lbfgs(const orc_problem *P, double *pp, const double *x, int itmax, int M, int robust,
               double nu) {
  orc_lbfgs_traced(P, pp, x, itmax, M, robust, nu, NULL);
}

/* ---- RTR / RSD / NSD: the per-row evaluators (Dirac/rtr_solve.c, Dirac/rtr_solve_robust.c) -------
 * The reference keeps the Jones of one (cluster, chunk) as a 2N x 2 complex matrix
 * (rtr_solve.c:1224-1243); here they stay in the API's parameter layout (station s: J[a][m] at
 * 8s + 2(2a+m)), a permutation of it.  y: hidden data of the chunk (row t0*Nbase first), wt: one
 * weight per row or NULL (= 1).  The control flow on top of these sums is rtr_algo.h (shared with
 * the product, instantiated with these evaluators by oracle/rtr_harness.cpp) and is pinned against
 * the compiled reference by tests/test_oracle_rtr.py. */
static void atmb(const cplx *a, const cplx *b, cplx *c) { /* a^H b, rtr_solve.c:58-64 */
  c[0] = conj(a[0]) * b[0] + conj(a[2]) * b[2];
  c[1] = conj(a[0]) * b[1] + conj(a[2]) * b[3];
  c[2] = conj(a[1]) * b[0] + conj(a[3]) * b[2];
  c[3] = conj(a[1]) * b[1] + conj(a[3]) * b[3];
}
static void rtr_acc(double *vec, int sta, const cplx *T, double w) {
  for (int i = 0; i < 4; i++) {
    vec[8 * sta + 2 * i] += w * creal(T[i]);
    vec[8 * sta + 2 * i + 1] += w * cimag(T[i]);
  }
}
/* cost (threadfn_fns_f, rtr_solve.c:188-241, rtr_solve_robust.c:72-130) and, if vec != NULL, the
 * unscaled station sums of the gradient (eta == NULL: threadfn_fns_fgrad, rtr_solve.c:453-526,
 * rtr_solve_robust.c:519-612) or of the Hessian-vector product (threadfn_fns_fhess,
 * rtr_solve.c:643-761, rtr_solve_robust.c:722-860) */
double orc_rtr_raw(const orc_problem *P, int k, int t0, int ntiles, const double *y,
                   const double *wt, const double *x, const double *eta, double *vec) {
  const int N = P->N, M = P->M;
  const long nrow = (long)ntiles * P->Nbase, boff = (long)t0 * P->Nbase;
  double fcost = 0.0;
  if (vec) memset(vec, 0, sizeof(double) * 8 * N);
  for (long ci = 0; ci < nrow; ci++) {
    if (P->flag[ci + boff]) continue;
    const int s1 = P->sta1[ci + boff], s2 = P->sta2[ci + boff];
    const double w = wt ? wt[ci] : 1.0;
    cplx G1[4], G2[4], C[4], T1[4], T2[4], res[4];
    jones_of(x, s1, G1);
    jones_of(x, s2, G2);
    for (int c = 0; c < 4; c++) C[c] = P->coh[4 * M * (ci + boff) + 4 * k + c];
    amb(G1, C, T1);
    ambt(T1, G2, T2);
    double e2 = 0.0;
    for (int c = 0; c < 4; c++) {
      res[c] = (y[8 * ci + 2 * c] + _Complex_I * y[8 * ci + 2 * c + 1]) - T2[c];
      e2 += creal(res[c]) * creal(res[c]) + cimag(res[c]) * cimag(res[c]);
    }
    fcost += w * e2;
    if (!vec) continue;
    if (!eta) {
      amb(res, G2, T1);  /* res G2 C^H */
      ambt(T1, C, T2);
      rtr_acc(vec, s1, T2, w);
      atmb(res, G1, T1); /* res^H G1 C */
      amb(T1, C, T2);
      rtr_acc(vec, s2, T2, w);
    } else {
      cplx E1[4], E2[4], res1[4];
      jones_of(eta, s1, E1);
      jones_of(eta, s2, E2);
      amb(G1, C, T1);
      ambt(T1, E2, res1);
      amb(E1, C, T1);
      ambt(T1, G2, T2);
      for (int c = 0; c < 4; c++) res1[c] += T2[c];
      amb(res, E2, T1); /* (res E2 - res1 G2) C^H */
      amb(res1, G2, T2);
      for (int c = 0; c < 4; c++) T1[c] -= T2[c];
      ambt(T1, C, T2);
      rtr_acc(vec, s1, T2, w);
      atmb(res, E1, T1); /* (res^H E1 - res1^H G1) C */
      atmb(res1, G1, T2);
      for (int c = 0; c < 4; c++) T1[c] -= T2[c];
      amb(T1, C, T2);
      rtr_acc(vec, s2, T2, w);
    }
  }
  return fcost;
}
/* unflagged rows per station (threadfn_fns_fcount, rtr_solve.c:71-91) */
void orc_rtr_counts(const orc_problem *P, int t0, int ntiles, double *cnt) {
  const long nrow = (long)ntiles * P->Nbase, boff = (long)t0 * P->Nbase;
  for (int i = 0; i < P->N; i++) cnt[i] = 0.0;
  for (long ci = 0; ci < nrow; ci++)
    if (!P->flag[ci + boff]) {
      cnt[P->sta1[ci + boff]] += 1.0;
      cnt[P->sta2[ci + boff]] += 1.0;
    }
}
/* row weights (nu+2)/(nu + max_c |res_c|^2) at x (threadfn_fns_fupdate_weights,
 * rtr_solve_robust.c:209-262); returns sum(log w - w) over the unflagged rows divided by ALL rows
 * (:271-287,360-370; flagged rows keep their weight and are never read) */
double orc_rtr_weights(const orc_problem *P, int k, int t0, int ntiles, const double *y,
                       const double *x, double nu, double *wt) {
  const int M = P->M;
  const long nrow = (long)ntiles * P->Nbase, boff = (long)t0 * P->Nbase;
  double s = 0.0;
  for (long ci = 0; ci < nrow; ci++) {
    if (P->flag[ci + boff]) continue;
    cplx G1[4], G2[4], C[4], T2[4];
    jones_of(x, P->sta1[ci + boff], G1);
    jones_of(x, P->sta2[ci + boff], G2);
    for (int c = 0; c < 4; c++) C[c] = P->coh[4 * M * (ci + boff) + 4 * k + c];
    model_row(G1, C, G2, T2);
    double mx = 0.0;
    for (int c = 0; c < 4; c++) {
      const double er = y[8 * ci + 2 * c] - creal(T2[c]), ei = y[8 * ci + 2 * c + 1] - cimag(T2[c]);
      const double e2 = er * er + ei * ei;
      if (e2 > mx) mx = e2;
    }
    const double w = (nu + 2.0) / (nu + mx);
    if (wt) wt[ci] = w;
    s += log(w) - w;
  }
  return s / (double)nrow;
}

/* solver of one (cluster, chunk) for solver_mode 4-6, registered by oracle/rtr_harness.cpp */
static orc_rtr_solver_fn g_rtr_solver = 0;
void orc_set_rtr_solver(orc_rtr_solver_fn fn) { g_rtr_solver = fn; }

/* ---- sagefit_visibilities (Dirac/lmfit.c:778-1053), randomize=0 ------------------------------- */
static int robust_mode(int sm) { return sm == 2 || sm == 3 || sm == 5 || sm == 6; }

int orc_sagefit(const orc_problem *P, double *x, double *pp, int max_emiter, int max_iter,
                int max_lbfgs, int lbfgs_m, int linsolv, int solver_mode, double nulow,
                double nuhigh, double *mean_nu, double *res_0, double *res_1) {
  const int N = P->N, M = P->M, Nbase = P->Nbase, tilesz = P->tilesz;
  const long n = 8l * Nbase * tilesz;
  const double opts[5] = {1e-3, 1e-15, 1e-15, 1e-20, -1e-6}; /* lmfit.c:801 */
  double info[10];
  double *xsub = (double *)xcalloc(n, sizeof(double));
  double *xdummy = (double *)xcalloc(n, sizeof(double));
  double *nerr = (double *)xcalloc(M, sizeof(double));
  double *nuM = (double *)xcalloc(M, sizeof(double));
  double robust_nu0 = nulow;
  double rtr_nu = nulow; /* lmdata.robust_nu of the RTR / NSD visits (lmfit.c:938-957) */
  if (solver_mode < 0 || solver_mode > 6 || (solver_mode > 3 && !g_rtr_solver)) {
    fprintf(stderr, "oracle: solver_mode %d not available (4-6 need oracle/librtr_harness.so)\n",
            solver_mode);
    exit(1);
  }
  for (int i = 0; i < 10; i++) info[i] = 0.0;
  orc_predict_full(P, pp, xsub);
  for (long i = 0; i < n; i++) xdummy[i] = x[i] - xsub[i];
  *res_0 = sqrt(nrm2sq(xdummy, n)) / (double)n;
  for (int ci = 0; ci < max_emiter; ci++) {
    for (int cj = 0; cj < M; cj++) {
      const int this_itermax = max_iter; /* weighted_iter only flips when randomize (lmfit.c:1007) */
      if (this_itermax <= 0) continue;
      orc_predict_cluster(P, cj, pp, xsub);
      for (long i = 0; i < n; i++) xdummy[i] += xsub[i];
      const int nchunk = P->nchunk[cj];
      const int tilechunk = (tilesz + nchunk - 1) / nchunk;
      int tcj = 0;
      double init_res = 0.0, final_res = 0.0;
      for (int ck = 0; ck < nchunk; ck++) {
        int ntiles = (tcj + tilechunk < tilesz) ? tilechunk : tilesz - tcj;
        double *pblk = pp + P->chunk_off[P->chunk0[cj] + ck];
        const double *xd = xdummy + 8l * tcj * Nbase;
        const int last = (ci == max_emiter - 1);
        if (solver_mode == 1) {
          orc_lm_chunk(P, cj, tcj, ntiles, pblk, xd, this_itermax, opts, linsolv, 0, info);
        } else if (solver_mode == 0) {
          orc_lm_chunk(P, cj, tcj, ntiles, pblk, xd, this_itermax, opts, linsolv, last ? 0 : 1,
                       info);
        } else if (solver_mode == 4) { /* lmfit.c:934-937 */
          g_rtr_solver(P, cj, tcj, ntiles, xd, 4, pblk, this_itermax + 5, this_itermax + 10, nulow,
                       nuhigh, &rtr_nu, info);
        } else if (solver_mode == 5 || solver_mode == 6) { /* lmfit.c:938-957 */
          if (!ci) rtr_nu = robust_nu0;
          if (solver_mode == 5)
            g_rtr_solver(P, cj, tcj, ntiles, xd, 5, pblk, this_itermax + 5, this_itermax + 10,
                         nulow, nuhigh, &rtr_nu, info);
          else
            g_rtr_solver(P, cj, tcj, ntiles, xd, 6, pblk, this_itermax + 15, 0, nulow, nuhigh,
                         &rtr_nu, info);
          if (last) nuM[cj] += rtr_nu;
        } else if (last) {
          double nu = robust_nu0;
          orc_rlm_chunk(P, cj, tcj, ntiles, pblk, xd, this_itermax, linsolv, solver_mode == 3,
                        nulow, nuhigh, &nu, info);
          nuM[cj] += nu;
        } else {
          orc_lm_chunk(P, cj, tcj, ntiles, pblk, xd, this_itermax, opts, linsolv, 1, info);
        }
        init_res += info[0];
        final_res += info[1];
        tcj += tilechunk;
      }
      nerr[cj] = (init_res > 0.0) ? (init_res - final_res) / init_res : 0.0;
      if (nerr[cj] < 0.0) nerr[cj] = 0.0;
      orc_predict_cluster(P, cj, pp, xsub);
      for (long i = 0; i < n; i++) xdummy[i] -= xsub[i];
      if (robust_mode(solver_mode) && ci == max_emiter - 1) nuM[cj] /= (double)nchunk;
    }
    double tot = 0.0;
    for (int cj = 0; cj < M; cj++) tot += fabs(nerr[cj]);
    if (tot > 0.0)
      for (int cj = 0; cj < M; cj++) nerr[cj] /= tot;
  }
  if (robust_mode(solver_mode)) {
    double s = 0.0;
    for (int cj = 0; cj < M; cj++) s += fabs(nuM[cj]);
    robust_nu0 = s / (double)M;
    if (robust_nu0 < nulow) robust_nu0 = nulow;
    else if (robust_nu0 > nuhigh) robust_nu0 = nuhigh;
  }
  if (max_lbfgs > 0) {
    if (robust_mode(solver_mode)) {
      if (lbfgs_m > 0) orc_lbfgs(P, pp, x, max_lbfgs, lbfgs_m, 1, robust_nu0);
    } else {
      orc_lbfgs(P, pp, x, max_lbfgs, lbfgs_m, 0, 0.0);
    }
  }
  orc_predict_full(P, pp, xsub);
  for (long i = 0; i < n; i++) x[i] -= xsub[i];
  *mean_nu = robust_nu0;
  *res_1 = sqrt(nrm2sq(x, n)) / (double)n;
  free(xsub); free(xdummy); free(nerr); free(nuM);
  return (*res_1 > *res_0) ? -1 : 0;
}

/* ---- bfgsfit_visibilities (Dirac/lmfit.c:1127-1212) ------------------------------------------- */
int orc_bfgsfit(const orc_problem *P, double *x, double *pp, int max_lbfgs, int lbfgs_m,
                int solver_mode, double mean_nu, double *res_0, double *res_1) {
  const long n = 8l * P->Nbase * P->tilesz;
  double *xsub = (double *)xcalloc(n, sizeof(double));
  orc_predict_full(P, pp, xsub);
  double s = 0.0;
  for (long i = 0; i < n; i++) s += (x[i] - xsub[i]) * (x[i] - xsub[i]);
  *res_0 = sqrt(s) / (double)n;
  if (max_lbfgs > 0)
    orc_lbfgs(P, pp, x, max_lbfgs, lbfgs_m, robust_mode(solver_mode), mean_nu);
  orc_predict_full(P, pp, xsub);
  for (long i = 0; i < n; i++) x[i] -= xsub[i];
  *res_1 = sqrt(nrm2sq(x, n)) / (double)n;
  free(xsub);
  return (*res_1 > *res_0) ? -1 : 0;
}

/* ---- coherencies from the sky model (Radio/predict.c:345-497, Radio/residual.c:1067-1248) ----- */
static cplx source_term(const orc_sky *S, int s, double u, double v, double w, double freq,
                        double fdelta2) {
  const double G = 2.0 * M_PI * (u * S->ll[s] + v * S->mm[s] + w * S->nn[s]);
  double fac = 1.0;
  if (G != 0.0) {
    double sm = G * fdelta2;
    fac = fabs(sin(sm) / sm);
  }
  cplx ph = (cos(G * freq) + _Complex_I * sin(G * freq)) * fac;
  const int st = S->stype[s];
  if (st != 0) {
    const double *g = S->gauss + 8 * (size_t)s;
    const double uf = u * freq, vf = v * freq, wf = w * freq;
    double up = uf, vp = vf;
    if (!(st == 1 && g[7] == 0.0)) { /* projection (Radio/predict.c:38-46,66-67,82-83) */
      up = uf * g[3] - vf * g[5] * g[4] + wf * g[6] * g[4];
      vp = uf * g[4] + vf * g[5] * g[3] - wf * g[6] * g[3];
    }
    if (st == 1) {
      const double ut = g[0] * (cos(g[2]) * up - sin(g[2]) * vp);
      const double vt = g[1] * (sin(g[2]) * up + cos(g[2]) * vp);
      ph *= exp(-2.0 * M_PI * M_PI * (ut * ut + vt * vt));
    } else if (st == 2) {
      ph *= j1(sqrt(up * up + vp * vp) * g[0] * 2.0 * M_PI);
    } else if (st == 3) {
      ph *= j0(sqrt(up * up + vp * vp) * g[0] * 2.0 * M_PI);
    } else {
      fprintf(stderr, "oracle: source type %d not restated\n", st);
      exit(1);
    }
  }
  return ph;
}

void orc_coherencies(const orc_sky *S, const double *u, const double *v, const double *w, int nrow,
                     double freq0, double fdelta, double uvmin, double uvmax, unsigned char *flag,
                     cplx *coh) {
  const int M = S->M;
  for (int r = 0; r < nrow; r++) {
    for (int k = 0; k < M; k++) {
      cplx C[4] = {0, 0, 0, 0};
      for (int s = S->src0[k]; s < S->src0[k + 1]; s++) {
        cplx ph = source_term(S, s, u[r], v[r], w[r], freq0, fdelta * 0.5);
        C[0] += ph * S->sI[s] + ph * S->sQ[s];
        C[1] += ph * S->sU[s] + _Complex_I * (ph * S->sV[s]);
        C[2] += ph * S->sU[s] - _Complex_I * (ph * S->sV[s]);
        C[3] += ph * S->sI[s] - ph * S->sQ[s];
      }
      memcpy(coh + 4 * ((size_t)M * r + k), C, sizeof(C));
    }
    if (flag && !flag[r]) { /* uv cut (Radio/predict.c:488-493) */
      double uvdist = sqrt(u[r] * u[r] + v[r] * v[r]) * freq0;
      if (uvdist < uvmin || uvdist > uvmax) flag[r] = 2;
    }
  }
}

static double spec_flux(double s0, double tempfr) {
  if (s0 > 0.0) return exp(log(s0) + tempfr);
  return (s0 == 0.0) ? 0.0 : -exp(log(-s0) + tempfr);
}

void orc_predict_multifreq(const orc_sky *S, const double *u, const double *v, const double *w,
                           int nrow, const double *freqs, int Nchan, double fdelta, int add_to_data,
                           double *x) {
  if (add_to_data == 1) memset(x, 0, sizeof(double) * 8 * (size_t)nrow * Nchan); /* SIMUL_ONLY */
  const double fd2 = (fdelta / (double)Nchan) * 0.5;
  for (int r = 0; r < nrow; r++)
    for (int k = 0; k < S->M; k++)
      for (int cf = 0; cf < Nchan; cf++) {
        const double f = freqs[cf];
        cplx C[4] = {0, 0, 0, 0};
        for (int s = S->src0[k]; s < S->src0[k + 1]; s++) {
          cplx ph = source_term(S, s, u[r], v[r], w[r], f, fd2);
          double fI = S->sI[s], fQ = S->sQ[s], fU = S->sU[s], fV = S->sV[s];
          if (S->spec_idx[s] != 0.0) {
            double fr = log(f / S->f0[s]), fr1 = fr * fr, fr2 = fr1 * fr;
            double tf = S->spec_idx[s] * fr + S->spec_idx1[s] * fr1 + S->spec_idx2[s] * fr2;
            fI = spec_flux(S->sI0[s], tf);
            fQ = spec_flux(S->sQ0[s], tf);
            fU = spec_flux(S->sU0[s], tf);
            fV = spec_flux(S->sV0[s], tf);
          }
          C[0] += ph * fI + ph * fQ;
          C[1] += ph * fU + _Complex_I * (ph * fV);
          C[2] += ph * fU - _Complex_I * (ph * fV);
          C[3] += ph * fI - ph * fQ;
        }
        double *o = x + 8 * (size_t)r + (size_t)cf * nrow * 8;
        for (int c = 0; c < 4; c++) {
          o[2 * c] += creal(C[c]);
          o[2 * c + 1] += cimag(C[c]);
        }
      }
}
