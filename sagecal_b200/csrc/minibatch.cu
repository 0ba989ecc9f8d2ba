// Multi-channel minibatch (stochastic) robust LBFGS: bfgsfit_minibatch_visibilities /
// bfgsfit_minibatch_consensus and the persistent state that carries the curvature pairs and the
// on-line gradient variance from one minibatch to the next (SURVEY.md 8f-3).
//
// Replaces (reference file:line)
//   bfgsfit_minibatch_visibilities / _consensus     robust_batchmode_lbfgs.c:1446-1577
//   robust_cost_func_multifreq / robust_grad_func_multifreq   robust_batchmode_lbfgs.c:1096-1445
//   lbfgs_fit_minibatch, linesearch_backtrack, mult_hessian   lbfgs.c:717-930, 444-474, 33-111
//   lbfgs_persist_init / _clear / _reset             lbfgs.c:954-1045
//
// Data flow: the reference's data and coherencies are [channel][row][...] arrays with ONE set of Jones
// for all channels of the minibatch.  Every channel becomes a resident single-channel problem (the same
// layout and kernels as the full-batch path: k_stream_all for the Student's-t cost, k_grad_tma_split
// for its gradient), cost and gradient are the sums over the channels, the iterate, the curvature
// pairs and the two-loop recursion (2 M dot products over 8 N Mt doubles) stay on the host like the
// reference's.  Control flow: restated decision for decision; the line search is the reference's
// Armijo backtracking (no numerical differentiation here, unlike the full-batch Fletcher search).
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

#include "../../include/dirac_b200.h"
#include "problem.h"
#include "minibatch_algo.h"

// ---- persistent state (layout: minibatch_algo.h) ------------------------------------------------------
using minibatch::pt_niter;
using minibatch::pt_running_avg;
using minibatch::pt_running_avg_sq;
extern "C" int lbfgs_persist_init(persistent_data_t *pt, int Nminibatch, int m, int n, int lbfgs_m,
                                  int Nt) {
  (void)Nminibatch; (void)n;  // the reference's offsets[] / lengths[] tables are never read by its
                              // minibatch drivers (robust_batchmode_lbfgs.c:1493-1495 "not used here")
  const size_t ns = (size_t)m * (lbfgs_m + 2) + 8;
  pt->s = (double *)calloc(ns, sizeof(double));
  pt->y = (double *)calloc((size_t)m * lbfgs_m + 1, sizeof(double));
  pt->rho = (double *)calloc((size_t)lbfgs_m + 1, sizeof(double));
  if (!pt->s || !pt->y || !pt->rho) {
    fprintf(stderr, "%s: %d: no free memory\n", __FILE__, __LINE__);
    exit(1);
  }
  pt->m = m;
  pt->lbfgs_m = lbfgs_m;
  pt->nfilled = 0;
  pt->vacant = 0;
  pt->Nt = Nt;
  return 0;
}
extern "C" int lbfgs_persist_clear(persistent_data_t *pt) {
  free(pt->s);
  free(pt->y);
  free(pt->rho);
  pt->s = pt->y = pt->rho = nullptr;
  return 0;
}
extern "C" int lbfgs_persist_reset(persistent_data_t *pt) {
  memset(pt->s, 0, sizeof(double) * ((size_t)pt->m * (pt->lbfgs_m + 2) + 8));
  memset(pt->y, 0, sizeof(double) * (size_t)pt->m * pt->lbfgs_m);
  memset(pt->rho, 0, sizeof(double) * (size_t)pt->lbfgs_m);
  pt->nfilled = 0;
  pt->vacant = 0;
  return 0;
}

// ---- multi-channel cost / gradient on the device -------------------------------------------------------
struct MultiChan {
  std::vector<dirac_b200_problem *> ch;
  int m, Mt, N;
  double nu;
  const double *y, *z, *rho;  // consensus terms (null: none)
  std::vector<double> gtmp;

  // robust_cost_func_multifreq (robust_batchmode_lbfgs.c:1096-1139)
  double cost(const double *p) {
    double f = 0.0;
    for (auto *pr : ch) f += dirac_b200_predict(pr, p, nullptr, 0, 2, nu);
    if (y && z && rho) {
      for (int ci = 0; ci < Mt; ci++) {
        double a = 0.0, b = 0.0;
        for (int i = 8 * N * ci; i < 8 * N * (ci + 1); i++) {
          const double xp = p[i] - z[i];
          a += xp * y[i];
          b += xp * xp;
        }
        f += a + rho[ci] * 0.5 * b;
      }
    }
    return f;
  }
  // robust_grad_func_multifreq (robust_batchmode_lbfgs.c:1300-1445): sum over the channels of the
  // single-channel Student's-t gradient WITH THE REFERENCE'S SIGN: cpu_calc_deriv_multifreq
  // accumulates -2 sum xr dV / (nu + xr^2) with xr = model - data (:1291), the full-batch
  // cpu_calc_deriv_robust +2 (robust_lbfgs.c:299, the true gradient, which dirac_b200_grad returns).
  // The minibatch LBFGS therefore starts uphill (first step: 2^-15 of the gradient after 15 failed
  // halvings) and only turns once the curvature pairs have negative y^T s; reproduced as is
  // (DESIGN.md 7.8).  The consensus terms enter as the reference writes them (:1420-1438).
  void grad(const double *p, double *g) {
    memset(g, 0, sizeof(double) * m);
    for (auto *pr : ch) {
      dirac_b200_grad(pr, p, gtmp.data(), 1, nu);
      for (int i = 0; i < m; i++) g[i] -= gtmp[i];
    }
    if (y && z && rho)
      for (int ci = 0; ci < Mt; ci++)
        for (int i = 8 * N * ci; i < 8 * N * (ci + 1); i++) g[i] += -y[i] - rho[ci] * (p[i] - z[i]);
  }
};

// ---- the stochastic closing stage of sagefit (lbfgs_m < 0, robust modes) ------------------------------
// Cost and gradient of one row window of the resident interval: the windowed passes of problem.cu
// stream only the timeslots the window overlaps.  The iterate and the two-loop recursion stay on the
// host, as in bfgsfit_minibatch_visibilities.
struct RowWindow {
  dirac_b200_problem *pr;
  double nu;
  long long r0, nr;
  void set_window(long long row0, long long nrows) {
    r0 = row0;
    nr = nrows;
  }
  double cost(const double *p) {
    if (nr <= 0) return 0.0;
    return dirac_b200_cost_window(pr, p, r0, nr, nu);
  }
  void grad(const double *p, double *g) {
    if (nr <= 0) {
      memset(g, 0, sizeof(double) * pr->d.npar);
      return;
    }
    dirac_b200_grad_window(pr, p, g, r0, nr, nu);
  }
};

// lbfgs_fit_robust_wrapper_minibatch on the resident problem (lmfit.c:1027-1029); p: host, npar, in/out
void db_lbfgs_fit_minibatch(dirac_b200_problem *pr, double *p, int m, int itmax, int M, double nu) {
  RowWindow F;
  F.pr = pr;
  F.nu = nu;
  F.r0 = 0;
  F.nr = pr->d.R;
  minibatch::lbfgs_fit_robust_wrapper_minibatch(F, p, m, pr->d.R, itmax, M);
}

static int minibatch_fit(double *x, int N, int Nbase, int tilesz, baseline_t *barr,
                         clus_source_t *carr, double *coh, int M, int Mt, int Nf, double *p,
                         const double *y, const double *z, const double *rho, int max_lbfgs,
                         int lbfgs_m, double robust_nu, double *res_0, double *res_1,
                         persistent_data_t *indata) {
  const int m = N * Mt * 8;
  const long long R = (long long)Nbase * tilesz;
  const double n = (double)R * Nf * 8.0;
  MultiChan F;
  F.m = m; F.Mt = Mt; F.N = N; F.nu = robust_nu; F.y = y; F.z = z; F.rho = rho;
  F.gtmp.resize(m);
  // channel c: coh[c][row][M][4] (complex), x[c][row][8]  (robust_batchmode_lbfgs.c:1176-1183)
  for (int c = 0; c < Nf; c++)
    F.ch.push_back(dirac_b200_create(N, Nbase, tilesz, barr, carr, M, Mt,
                                     coh + (size_t)c * 8 * M * R, x + (size_t)c * 8 * R));
  *res_0 = F.cost(p);
  // lbfgs_fit (lbfgs.c:933-950): persistent data -> minibatch variant
  minibatch::lbfgs_fit_minibatch(F, p, m, max_lbfgs, lbfgs_m, indata);
  *res_1 = F.cost(p);
  *res_0 *= 1.0 / n;
  *res_1 *= 1.0 / n;
  for (auto *pr : F.ch) dirac_b200_destroy(pr);
  return 0;
}

extern "C" int bfgsfit_minibatch_visibilities(double *u, double *v, double *w, double *x, int N,
                                              int Nbase, int tilesz, baseline_t *barr,
                                              clus_source_t *carr, double *coh, int M, int Mt,
                                              double *freqs, int Nf, double fdelta, double *p, int Nt,
                                              int max_lbfgs, int lbfgs_m, int gpu_threads,
                                              int solver_mode, double robust_nu, double *res_0,
                                              double *res_1, persistent_data_t *indata,
                                              int nminibatch, int totalminibatch) {
  (void)u; (void)v; (void)w; (void)freqs; (void)fdelta; (void)Nt; (void)gpu_threads;
  (void)solver_mode; (void)nminibatch; (void)totalminibatch;
  return minibatch_fit(x, N, Nbase, tilesz, barr, carr, coh, M, Mt, Nf, p, nullptr, nullptr, nullptr,
                       max_lbfgs, lbfgs_m, robust_nu, res_0, res_1, indata);
}

extern "C" int bfgsfit_minibatch_consensus(double *u, double *v, double *w, double *x, int N,
                                           int Nbase, int tilesz, baseline_t *barr,
                                           clus_source_t *carr, double *coh, int M, int Mt,
                                           double *freqs, int Nf, double fdelta, double *p, double *y,
                                           double *z, double *rho, int Nt, int max_lbfgs, int lbfgs_m,
                                           int gpu_threads, int solver_mode, double robust_nu,
                                           double *res_0, double *res_1, persistent_data_t *indata,
                                           int nminibatch, int totalminibatch) {
  (void)u; (void)v; (void)w; (void)freqs; (void)fdelta; (void)Nt; (void)gpu_threads;
  (void)solver_mode; (void)nminibatch; (void)totalminibatch;
  return minibatch_fit(x, N, Nbase, tilesz, barr, carr, coh, M, Mt, Nf, p, y, z, rho, max_lbfgs,
                       lbfgs_m, robust_nu, res_0, res_1, indata);
}

// ---- the same two calls with the GPU build's argument list ---------------------------------------------
// Under HAVE_CUDA the reference declares bfgsfit_minibatch_visibilities / _consensus with
// `short *hbb, int *ptoclus` in place of `baseline_t *barr, clus_source_t *carr` (Dirac.h:315-319,
// 343-347; minibatch_mode.cpp:332-342,438): hbb[2 row] = (sta1, sta2) as shorts, (-1, -1) for a flagged
// row (rearrange_baselines, baseline_utils.c:123-137), ptoclus[2 k] = (nchunk, p[0]) of cluster k with the
// chunks of a cluster contiguous in the Jones vector.  One symbol cannot carry two signatures, so these
// are exported under their own names; INTEGRATION.md says how a GPU-build driver binds them.
//
// dirac_b200_barr_from_hbb rebuilds the baseline_t rows: stations by position in the canonical order
// (a flagged row has lost its pair), flag 1 where hbb marks the row.  Returns -1 if an unflagged row
// does not carry the canonical pair of its position.  Host arithmetic, no GPU needed.
extern "C" int dirac_b200_barr_from_hbb(int N, int Nbase, int tilesz, const short *hbb,
                                        baseline_t *barr) {
  generate_baselines(Nbase, tilesz, N, barr, 1);
  const long long R = (long long)Nbase * tilesz;
  for (long long r = 0; r < R; r++) {
    const int a = hbb[2 * r], b = hbb[2 * r + 1];
    if (a < 0 || b < 0) {
      barr[r].flag = 1;
    } else {
      barr[r].flag = 0;
      if (a != barr[r].sta1 || b != barr[r].sta2) return -1;
    }
  }
  return 0;
}

namespace {
struct HbbTables {
  std::vector<baseline_t> barr;
  std::vector<clus_source_t> carr;
  std::vector<int> poff;
  HbbTables(int N, int Nbase, int tilesz, const short *hbb, int M, int Mt, const int *ptoclus)
      : barr((size_t)Nbase * tilesz), carr(M), poff(Mt > 0 ? Mt : 1) {
    if (dirac_b200_barr_from_hbb(N, Nbase, tilesz, hbb, barr.data())) {
      fprintf(stderr, "dirac_b200: hbb is not in the row order of generate_baselines; unsupported "
                      "row order\n");
      exit(1);
    }
    memset(carr.data(), 0, sizeof(clus_source_t) * M);
    int mt = 0;
    for (int k = 0; k < M; k++) {
      carr[k].nchunk = ptoclus[2 * k];
      if (mt + carr[k].nchunk > Mt) {
        fprintf(stderr, "dirac_b200: ptoclus names more than Mt = %d chunks\n", Mt);
        exit(1);
      }
      carr[k].p = poff.data() + mt;
      for (int c = 0; c < carr[k].nchunk; c++) poff[mt + c] = ptoclus[2 * k + 1] + 8 * N * c;
      mt += carr[k].nchunk;
    }
  }
};
}  // namespace

extern "C" int bfgsfit_minibatch_visibilities_hbb(
    double *u, double *v, double *w, double *x, int N, int Nbase, int tilesz, short *hbb, int *ptoclus,
    double *coh, int M, int Mt, double *freqs, int Nf, double fdelta, double *p, int Nt, int max_lbfgs,
    int lbfgs_m, int gpu_threads, int solver_mode, double robust_nu, double *res_0, double *res_1,
    persistent_data_t *indata, int nminibatch, int totalminibatch) {
  HbbTables t(N, Nbase, tilesz, hbb, M, Mt, ptoclus);
  return bfgsfit_minibatch_visibilities(u, v, w, x, N, Nbase, tilesz, t.barr.data(), t.carr.data(),
                                        coh, M, Mt, freqs, Nf, fdelta, p, Nt, max_lbfgs, lbfgs_m,
                                        gpu_threads, solver_mode, robust_nu, res_0, res_1, indata,
                                        nminibatch, totalminibatch);
}

extern "C" int bfgsfit_minibatch_consensus_hbb(
    double *u, double *v, double *w, double *x, int N, int Nbase, int tilesz, short *hbb, int *ptoclus,
    double *coh, int M, int Mt, double *freqs, int Nf, double fdelta, double *p, double *y, double *z,
    double *rho, int Nt, int max_lbfgs, int lbfgs_m, int gpu_threads, int solver_mode,
    double robust_nu, double *res_0, double *res_1, persistent_data_t *indata, int nminibatch,
    int totalminibatch) {
  HbbTables t(N, Nbase, tilesz, hbb, M, Mt, ptoclus);
  return bfgsfit_minibatch_consensus(u, v, w, x, N, Nbase, tilesz, t.barr.data(), t.carr.data(), coh,
                                     M, Mt, freqs, Nf, fdelta, p, y, z, rho, Nt, max_lbfgs, lbfgs_m,
                                     gpu_threads, solver_mode, robust_nu, res_0, res_1, indata,
                                     nminibatch, totalminibatch);
}
