// Minibatch (stochastic) LBFGS of the reference, restated decision for decision, templated on the
// function object that supplies cost and gradient (lbfgs_fit_minibatch, linesearch_backtrack,
// mult_hessian: lbfgs.c:717-930, 444-474, 33-111).  The product instantiates it with the multi-channel
// device evaluator and, through lbfgs_fit_robust_wrapper_minibatch, with the row windows of a resident
// interval (sagefit's stochastic stage, minibatch.cu; pinned on the CPU by
// tests/test_oracle_minibatch_window.py); oracle/minibatch_harness.cpp instantiates it with the oracle's
// per-row cost / gradient to pin the control flow against the compiled reference without a GPU (test
// infrastructure, not shipped).
//
// F concept:  double cost(const double *p);   void grad(const double *p, double *g);
#pragma once
#include <math.h>
#include <string.h>
#include <vector>

#include "../../include/dirac_b200.h"

namespace minibatch {

// ---- persistent state ---------------------------------------------------------------------------------
// The reference declares persistent_data_t twice (Dirac.h:86-110 CPU build, :196-226 GPU build); the
// two layouts agree only up to `Nt`.  This library touches nothing beyond that common prefix, so a
// caller compiled against either header can hand its struct in: the running averages of the on-line
// gradient variance and the iteration count live behind the curvature pairs in the `s` allocation.
inline double *pt_running_avg(persistent_data_t *pt) {
  return pt->s + (size_t)pt->m * pt->lbfgs_m;
}
inline double *pt_running_avg_sq(persistent_data_t *pt) {
  return pt->s + (size_t)pt->m * (pt->lbfgs_m + 1);
}
inline double *pt_niter(persistent_data_t *pt) {
  return pt->s + (size_t)pt->m * (pt->lbfgs_m + 2);
}

inline double ddot(int m, const double *a, const double *b) {
  double s = 0.0;
  for (int i = 0; i < m; i++) s += a[i] * b[i];
  return s;
}

// pk = H_k gk by the two-loop recursion over the M stored pairs, the newest at slot ii-1
// (mult_hessian, lbfgs.c:33-111)
inline void mult_hessian(int m, double *pk, const double *gk, const double *s, const double *y,
                         const double *rho, int M, int ii) {
  std::vector<double> alphai(M > 0 ? M : 1);
  std::vector<int> idx(M > 0 ? M : 1);
  if (M > 0) {
    ii = ii > 0 ? ii - 1 : M - 1;
    for (int ci = 0; ci < M - ii - 1; ci++) idx[ci] = ii + ci + 1;
    for (int ci = M - ii - 1; ci < M; ci++) idx[ci] = ci - M + ii + 1;
  }
  memcpy(pk, gk, sizeof(double) * m);
  for (int ci = 0; ci < M; ci++) {
    const int j = idx[M - ci - 1];
    alphai[M - ci - 1] = rho[j] * ddot(m, s + (size_t)m * j, pk);
    for (int i = 0; i < m; i++) pk[i] -= alphai[M - ci - 1] * y[(size_t)m * j + i];
  }
  if (M > 0) {
    const int j = idx[M - 1];
    const double gamma = ddot(m, s + (size_t)m * j, y + (size_t)m * j) /
                         ddot(m, y + (size_t)m * j, y + (size_t)m * j);
    for (int i = 0; i < m; i++) pk[i] *= gamma;
  }
  for (int ci = 0; ci < M; ci++) {
    const int j = idx[ci];
    const double beta = rho[j] * ddot(m, y + (size_t)m * j, pk);
    for (int i = 0; i < m; i++) pk[i] += (alphai[ci] - beta) * s[(size_t)m * j + i];
  }
}

// Armijo backtracking (linesearch_backtrack, lbfgs.c:444-474)
template <class FN>
double linesearch_backtrack(FN &F, const double *xk, const double *pk,
                                   const double *gk, int m, double alpha0) {
  const double c = 1e-4;
  double alphak = alpha0;
  std::vector<double> xk1(m);
  for (int i = 0; i < m; i++) xk1[i] = xk[i] + alphak * pk[i];
  double fnew = F.cost(xk1.data());
  const double fold = F.cost(xk);
  const double product = c * ddot(m, pk, gk);
  int ci = 0;
  while (ci < 15 && (isnan(fnew) || fnew > fold + alphak * product)) {
    alphak *= 0.5;
    for (int i = 0; i < m; i++) xk1[i] = xk[i] + alphak * pk[i];
    fnew = F.cost(xk1.data());
    ci++;
  }
  return alphak;
}

// lbfgs_fit_minibatch (lbfgs.c:717-930)
template <class FN>
void lbfgs_fit_minibatch(FN &F, double *p, int m, int itmax, int M,
                                persistent_data_t *indata) {
  const double CLM_STOP_THRESH_ = 1e-17, CLM_EPSILON_ = 1e-12;
  std::vector<double> gk(m), xk1(m), xk(p, p + m), pk(m);
  double *s = indata->s, *y = indata->y, *rho = indata->rho;
  double *running_avg = pt_running_avg(indata), *running_avg_sq = pt_running_avg_sq(indata);
  double *niter = pt_niter(indata);
  double alphabar = 1.0;
  F.grad(xk.data(), gk.data());
  double gradnrm = sqrt(ddot(m, gk.data(), gk.data()));
  int ck = gradnrm < CLM_STOP_THRESH_ ? itmax : 0;
  int ci = indata->vacant;
  size_t cm = (size_t)m * ci;
  while (ck < itmax && isnormal(gradnrm) && gradnrm > CLM_STOP_THRESH_) {
    *niter += 1.0;
    const int nit = (int)*niter;
    const bool batch_changed = (nit > 1 && ck == 0);
    if (batch_changed) {
      // running mean / variance of the gradient over the minibatches -> step size cap
      double asum = 0.0;
      for (int i = 0; i < m; i++) {
        const double g_min_rold = gk[i] - running_avg[i];
        running_avg[i] += g_min_rold / (double)nit;
        const double g_min_rnew = gk[i] - running_avg[i];
        running_avg_sq[i] += g_min_rold * g_min_rnew;
      }
      for (int i = 0; i < m; i++) asum += fabs(running_avg_sq[i]);
      alphabar = 10.0 / (1.0 + asum / ((double)(nit - 1) * gradnrm));
    }
    mult_hessian(m, pk.data(), gk.data(), s, y, rho, indata->nfilled < M ? indata->nfilled : M, ci);
    for (int i = 0; i < m; i++) pk[i] = -pk[i];
    const double alphak = linesearch_backtrack(F, xk.data(), pk.data(), gk.data(), m, alphabar);
    if (!isnormal(alphak) || fabs(alphak) < CLM_EPSILON_) break;
    for (int i = 0; i < m; i++) xk1[i] = xk[i] + alphak * pk[i];
    if (!batch_changed)
      for (int i = 0; i < m; i++) {
        s[cm + i] = xk1[i] - xk[i];
        y[cm + i] = -gk[i];
      }
    F.grad(xk1.data(), gk.data());
    gradnrm = sqrt(ddot(m, gk.data(), gk.data()));
    if (!isnormal(gradnrm) || gradnrm < CLM_STOP_THRESH_) break;
    if (!batch_changed) {
      for (int i = 0; i < m; i++) y[cm + i] += gk[i];
      const double lm0 = 1e-6;
      if (gradnrm > 1e3 * lm0)
        for (int i = 0; i < m; i++) y[cm + i] += lm0 * s[cm + i];
      rho[ci] = 1.0 / ddot(m, y + cm, s + cm);
    }
    xk = xk1;
    ck++;
    if (!batch_changed) {
      indata->nfilled = (indata->nfilled < M ? indata->nfilled + 1 : M);
      if (cm < (size_t)(M - 1) * m) {
        cm += m;
        ci++;
        indata->vacant++;
      } else {
        cm = 0;
        ci = 0;
        indata->vacant = 0;
      }
    }
  }
  memcpy(p, xk.data(), sizeof(double) * m);
}

// Batch table of the stochastic stage of sagefit (lbfgs_persist_init, lbfgs.c:954-1010, with the
// n rows of the interval): window i is the rows [i b, i b + len_i), b = ceil(n / nbatch),
// len_i = min(b, n - i b).  len_i <= 0 (fewer rows than windows) is an empty window.
inline void batch_window(long long n, int nbatch, int i, long long *off, long long *len) {
  const long long b = (n + nbatch - 1) / nbatch;
  *off = (long long)i * b;
  *len = (n - *off < b) ? n - *off : b;
}

// lbfgs_fit_robust_wrapper_minibatch (robust_batchmode_lbfgs.c:859-930): (itmax + 4) / 4 epochs over
// the 5 row windows of the interval in order, 4 minibatch iterations per window, one persistent state
// (curvature pairs, gradient running averages) created for this call and carried through all of them.
// FW: the F concept plus  void set_window(long long row0, long long nrows);
template <class FW>
void lbfgs_fit_robust_wrapper_minibatch(FW &F, double *p, int m, long long nrows, int itmax,
                                        int M) {
  const int Nbatch = 5, Niterperbatch = 4;
  std::vector<double> s((size_t)m * (M + 2) + 8, 0.0), y((size_t)m * M + 1, 0.0), rho(M + 1, 0.0);
  persistent_data_t pt;
  memset(&pt, 0, sizeof(pt));
  pt.s = s.data();
  pt.y = y.data();
  pt.rho = rho.data();
  pt.m = m;
  pt.lbfgs_m = M;
  const int Nloops = (itmax + Niterperbatch) / Niterperbatch;
  for (int nl = 0; nl < Nloops; nl++)
    for (int ci = 0; ci < Nbatch; ci++) {
      long long off, len;
      batch_window(nrows, Nbatch, ci, &off, &len);
      F.set_window(off, len);
      lbfgs_fit_minibatch(F, p, m, Niterperbatch, M, &pt);
    }
}


}  // namespace minibatch
