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
// for all channels of the minibatch.  The channels become one resident band ([chan][M][4][R]
// coherencies, [chan][4][R] data, planar): the Student's-t cost of every channel is one k_stream_band
// launch, its gradient one residual launch of the same kernel and one k_grad_tma_band launch, each
// with one host readback.  The iterate, the curvature pairs and the two-loop recursion (2 M dot
// products over 8 N Mt doubles) stay on the host like the reference's.  Control flow: restated decision for decision; the line search is the reference's
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

// ---- minibatch bands on the device (problem.h) ---------------------------------------------------------
BandDev *db_band_create(int N, int Nbase, int tilesz, const clus_source_t *carr, int M, int Mt,
                        int maxnc, cudaStream_t st) {
  require_gpu();
  if (Nbase != N * (N - 1) / 2) {
    fprintf(stderr, "dirac_b200: Nbase=%d is not N(N-1)/2 for N=%d; only the canonical baseline "
                    "set of generate_baselines is supported\n", Nbase, N);
    exit(1);
  }
  BandDev *bd = new BandDev();
  bd->N = N; bd->Nbase = Nbase; bd->tilesz = tilesz; bd->M = M; bd->Mt = Mt;
  bd->maxnc = maxnc > 0 ? maxnc : 1;
  bd->R = (long long)Nbase * tilesz;
  bd->npar = 8ll * N * Mt;
  bd->st = st;
  std::vector<ClusterDesc> clus(M);
  std::vector<int> poff;
  for (int k = 0; k < M; k++) {
    clus[k].nchunk = carr[k].nchunk;
    clus[k].chunk0 = (int)poff.size();
    for (int c = 0; c < carr[k].nchunk; c++) poff.push_back(carr[k].p[c]);
  }
  if ((int)poff.size() != Mt) {
    fprintf(stderr, "dirac_b200: sum of nchunk (%d) != Mt (%d)\n", (int)poff.size(), Mt);
    exit(1);
  }
  std::vector<TileDesc> tiles;
  db_build_tiles(N, tiles);
  bd->ntile = (int)tiles.size();
  std::vector<short2> pq;
  for (int p = 0; p < N - 1; p++)
    for (int q = p + 1; q < N; q++) pq.push_back(make_short2((short)p, (short)q));
  bd->clus = (ClusterDesc *)db_malloc(sizeof(ClusterDesc) * M);
  bd->chunk_poff = (int *)db_malloc(sizeof(int) * Mt);
  bd->tiles = (TileDesc *)db_malloc(sizeof(TileDesc) * tiles.size());
  bd->blpq = (short2 *)db_malloc(sizeof(short2) * Nbase);
  DB_CHECK(cudaMemcpyAsync(bd->clus, clus.data(), sizeof(ClusterDesc) * M, cudaMemcpyHostToDevice, st));
  DB_CHECK(cudaMemcpyAsync(bd->chunk_poff, poff.data(), sizeof(int) * Mt, cudaMemcpyHostToDevice, st));
  DB_CHECK(cudaMemcpyAsync(bd->tiles, tiles.data(), sizeof(TileDesc) * tiles.size(),
                           cudaMemcpyHostToDevice, st));
  DB_CHECK(cudaMemcpyAsync(bd->blpq, pq.data(), sizeof(short2) * Nbase, cudaMemcpyHostToDevice, st));
  bd->pp = (double *)db_malloc(sizeof(double) * bd->npar);
  bd->g = (double *)db_malloc(sizeof(double) * bd->npar);
  bd->partials = (double *)db_malloc(sizeof(double) * db_band_nblocks(Nbase, tilesz, bd->maxnc));
  bd->scal = (double *)db_malloc(sizeof(double));
  bd->counters = (unsigned int *)db_malloc(sizeof(unsigned int));
  DB_CHECK(cudaMemsetAsync(bd->counters, 0, sizeof(unsigned int), st));
  DB_CHECK(cudaMallocHost((void **)&bd->h_scal, sizeof(double)));
  bd->res = (double2 *)db_malloc(sizeof(double2) * 4 * (size_t)bd->R * bd->maxnc);
  db_stream_sync(st);  // the host tables go out of scope
  return bd;
}

void db_band_destroy(BandDev *bd) {
  if (!bd) return;
  cudaStreamSynchronize(bd->st);
  db_free(bd->clus); db_free(bd->chunk_poff); db_free(bd->tiles); db_free(bd->blpq);
  db_free(bd->pp); db_free(bd->g); db_free(bd->partials); db_free(bd->scal); db_free(bd->counters);
  db_free(bd->res);
  cudaFreeHost(bd->h_scal);
  delete bd;
}

// one k_stream_band launch over the band's channels at the Jones in bd->pp: the Student's-t cost
// (cost != 0, lands in bd->scal) or the residual e = x - V of every channel into bd->res
static void band_pass(BandDev *bd, const BandView &b, double nu, bool cost) {
  StreamAllArgs a;
  memset(&a, 0, sizeof(a));
  a.coh = b.coh; a.x = b.x; a.flag = b.flag; a.pp = bd->pp; a.clus = bd->clus;
  a.chunk_poff = bd->chunk_poff; a.blpq = bd->blpq; a.out = cost ? nullptr : bd->res;
  a.partials = bd->partials; a.cost = bd->scal; a.counter = bd->counters; a.R = bd->R; a.N = bd->N;
  a.Nbase = bd->Nbase; a.tilesz = bd->tilesz; a.M = bd->M;
  a.out_mode = cost ? 0 : 1;
  a.cost_mode = cost ? 2 : 0;
  a.inv_nu = (nu > 0.0) ? 1.0 / nu : 0.0;
  db_prof_begin(13, (double)bd->R * b.nc * (64.0 * bd->M + 65.0 + (cost ? 0.0 : 64.0)), bd->st);
  db_launch_band_tma(&a, b.nc, bd->st);
  db_prof_end(bd->st);
  db_count_launch(1);
}

// ---- multi-channel cost / gradient of one band ---------------------------------------------------------
struct BandFn {
  BandDev *bd;
  BandView b;
  double nu;
  const double *y, *z, *rho;  // consensus terms (null: none)

  // robust_cost_func_multifreq (robust_batchmode_lbfgs.c:1096-1139): one launch over all channels
  double cost(const double *p) {
    const int m = (int)bd->npar, N = bd->N;
    double f = 0.0;
    if (b.nc > 0) {
      DB_CHECK(cudaMemcpyAsync(bd->pp, p, sizeof(double) * m, cudaMemcpyHostToDevice, bd->st));
      band_pass(bd, b, nu, true);
      DB_CHECK(cudaMemcpyAsync(bd->h_scal, bd->scal, sizeof(double), cudaMemcpyDeviceToHost, bd->st));
      db_stream_sync(bd->st);
      f = *bd->h_scal;
    }
    if (y && z && rho) {
      for (int ci = 0; ci < bd->Mt; ci++) {
        double a = 0.0, c = 0.0;
        for (int i = 8 * N * ci; i < 8 * N * (ci + 1); i++) {
          const double xp = p[i] - z[i];
          a += xp * y[i];
          c += xp * xp;
        }
        f += a + rho[ci] * 0.5 * c;
      }
    }
    return f;
  }
  // robust_grad_func_multifreq (robust_batchmode_lbfgs.c:1300-1445): the single-channel Student's-t
  // gradient summed over the channels WITH THE REFERENCE'S SIGN: cpu_calc_deriv_multifreq
  // accumulates -2 sum xr dV / (nu + xr^2) with xr = model - data (:1291), the full-batch
  // cpu_calc_deriv_robust +2 (robust_lbfgs.c:299, the true gradient, which dirac_b200_grad returns).
  // The minibatch LBFGS therefore starts uphill (first step: 2^-15 of the gradient after 15 failed
  // halvings) and only turns once the curvature pairs have negative y^T s; reproduced as is
  // (DESIGN.md 7.8).  Here e = data - model, so the kernel's scale is +2.  The residual pass and the
  // gradient pass cover every channel in one launch each; the Jones go up and g comes down once.
  // The consensus terms enter as the reference writes them (:1420-1438).
  void grad(const double *p, double *g) {
    const int m = (int)bd->npar, N = bd->N;
    if (b.nc > 0) {
      DB_CHECK(cudaMemcpyAsync(bd->pp, p, sizeof(double) * m, cudaMemcpyHostToDevice, bd->st));
      band_pass(bd, b, 0.0, false);
      DB_CHECK(cudaMemsetAsync(bd->g, 0, sizeof(double) * m, bd->st));
      GradArgs a;
      memset(&a, 0, sizeof(a));
      a.coh = b.coh; a.res = bd->res; a.flag = b.flag; a.pp = bd->pp; a.clus = bd->clus;
      a.chunk_poff = bd->chunk_poff; a.tiles = bd->tiles; a.g = bd->g; a.R = bd->R; a.N = N;
      a.Nbase = bd->Nbase; a.tilesz = bd->tilesz; a.M = bd->M; a.robust = 1; a.nu = nu;
      a.scale = 2.0;
      db_prof_begin(14, (double)bd->R * b.nc * (64.0 * bd->M + 65.0) + 64.0 * N * bd->Mt, bd->st);
      db_launch_grad_band_tma(&a, bd->ntile, b.nc, bd->st);
      db_prof_end(bd->st);
      db_count_launch(1);
      DB_CHECK(cudaMemcpyAsync(g, bd->g, sizeof(double) * m, cudaMemcpyDeviceToHost, bd->st));
      db_stream_sync(bd->st);
      DB_CHECK(cudaGetLastError());
    } else {
      memset(g, 0, sizeof(double) * m);
    }
    if (y && z && rho)
      for (int ci = 0; ci < bd->Mt; ci++)
        for (int i = 8 * N * ci; i < 8 * N * (ci + 1); i++) g[i] += -y[i] - rho[ci] * (p[i] - z[i]);
  }
};

// bfgsfit_minibatch_visibilities / _consensus (robust_batchmode_lbfgs.c:1446-1577) on a resident band.
// A band without channels has n = 0 data: its costs are 0 x 1/0 = NaN and its zero gradient stops the
// LBFGS before the first step, as in the reference.
void db_band_fit(BandDev *bd, const BandView &b, double *p, const double *y, const double *z,
                 const double *rho, int max_lbfgs, int lbfgs_m, double robust_nu, double *res_0,
                 double *res_1, persistent_data_t *indata) {
  BandFn F = {bd, b, robust_nu, y, z, rho};
  const double n = (double)bd->R * b.nc * 8.0;
  *res_0 = F.cost(p);
  // lbfgs_fit (lbfgs.c:933-950): persistent data -> minibatch variant
  minibatch::lbfgs_fit_minibatch(F, p, (int)bd->npar, max_lbfgs, lbfgs_m, indata);
  *res_1 = F.cost(p);
  *res_0 *= 1.0 / n;
  *res_1 *= 1.0 / n;
}

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

// the reference's host arrays as one band: channel c's coherencies coh[c][row][M][4] (complex) and data
// x[c][row][8] (robust_batchmode_lbfgs.c:1176-1183) go up once, into the planar band layout, with the
// flags of barr's rows; the buffers live as long as ds
static BandView band_stage(DeviceScope &ds, const double *x, int N, int Nbase, int tilesz,
                           const baseline_t *barr, const double *coh, int M, int Nf) {
  const long long R = (long long)Nbase * tilesz;
  std::vector<unsigned char> hflag(R);
  db_canonical_flags(N, Nbase, tilesz, barr, hflag.data());
  const int nc = Nf > 0 ? Nf : 0;
  double2 *dcoh = ds.alloc<double2>((size_t)M * 4 * R * (nc ? nc : 1));
  double2 *dx = ds.alloc<double2>((size_t)4 * R * (nc ? nc : 1));
  unsigned char *dflag = ds.upload(hflag);
  long long rows_per = (128ll << 20) / ((long long)M * 64);
  if (rows_per < 1) rows_per = 1;
  if (rows_per > R) rows_per = R;
  // stages rows_per rows of one channel's coherencies, or one channel's data
  const size_t nstage = (size_t)rows_per * M * 4 > (size_t)4 * R ? (size_t)rows_per * M * 4 : 4 * R;
  double2 *stage = ds.alloc<double2>(nstage);
  for (int c = 0; c < nc; c++) {
    double2 *cc = dcoh + (size_t)c * M * 4 * R;
    for (long long r0 = 0; r0 < R; r0 += rows_per) {
      const int nr = (int)((R - r0 < rows_per) ? (R - r0) : rows_per);
      DB_CHECK(cudaMemcpyAsync(stage, coh + ((size_t)c * R + r0) * M * 8, (size_t)nr * M * 64,
                               cudaMemcpyHostToDevice, ds.st));
      db_launch_coh_to_planar(stage, cc, r0, nr, M, R, ds.st);
      db_count_launch(1);
    }
    db_count_coh_host_bytes((size_t)R * M * 64);
    DB_CHECK(cudaMemcpyAsync(stage, x + (size_t)c * 8 * R, (size_t)R * 64, cudaMemcpyHostToDevice,
                             ds.st));
    db_launch_vis_to_planar(stage, dx + (size_t)c * 4 * R, R, ds.st);
    db_count_launch(1);
  }
  BandView b = {dcoh, dx, dflag, nc};
  return b;
}

static int minibatch_fit(double *x, int N, int Nbase, int tilesz, baseline_t *barr,
                         clus_source_t *carr, double *coh, int M, int Mt, int Nf, double *p,
                         const double *y, const double *z, const double *rho, int max_lbfgs,
                         int lbfgs_m, double robust_nu, double *res_0, double *res_1,
                         persistent_data_t *indata) {
  {
    DeviceScope ds;
    BandDev *bd = db_band_create(N, Nbase, tilesz, carr, M, Mt, Nf, ds.st);
    const BandView b = band_stage(ds, x, N, Nbase, tilesz, barr, coh, M, Nf);
    db_band_fit(bd, b, p, y, z, rho, max_lbfgs, lbfgs_m, robust_nu, res_0, res_1, indata);
    db_band_destroy(bd);
    ds.sync();
  }
  return 0;
}

// Test hook (not in the public headers): the band passes the minibatch fits run, on one band staged
// as minibatch_fit stages it, in a BandDev of capacity maxnc >= Nf.  The npts Jones vectors p[i]
// (8 N Mt each) are evaluated in order with the fits' own cost and gradient: cost[i] the Student's-t
// cost summed over the channels (plus the consensus terms when y, z, rho are given), grad[i] its
// gradient with the reference's minibatch sign; res [Nf][R][8] (or null) the residual x - V of the
// last point's gradient pass.  Returns -1 for Nf < 0, Nf > maxnc or npts < 1, before any device work.
extern "C" int dirac_b200_band_eval(int N, int Nbase, int tilesz, baseline_t *barr, clus_source_t *carr,
                                    int M, int Mt, const double *coh, const double *x, int Nf,
                                    int maxnc, int npts, const double *p, const double *y,
                                    const double *z, const double *rho, double nu, double *cost,
                                    double *grad, double *res) {
  if (Nf < 0 || Nf > maxnc || npts < 1) return -1;
  {
    DeviceScope ds;
    BandDev *bd = db_band_create(N, Nbase, tilesz, carr, M, Mt, maxnc, ds.st);
    const BandView b = band_stage(ds, x, N, Nbase, tilesz, barr, coh, M, Nf);
    BandFn F = {bd, b, nu, y, z, rho};
    const size_t m = (size_t)bd->npar;
    for (int i = 0; i < npts; i++) {
      cost[i] = F.cost(p + i * m);
      F.grad(p + i * m, grad + i * m);
    }
    if (res && Nf > 0) {
      double2 *stage = ds.alloc<double2>((size_t)4 * bd->R);
      for (int c = 0; c < Nf; c++) {
        db_launch_vis_from_planar(bd->res + (size_t)c * 4 * bd->R, stage, bd->R, ds.st);
        db_count_launch(1);
        DB_CHECK(cudaMemcpyAsync(res + (size_t)c * 8 * bd->R, stage, (size_t)bd->R * 64,
                                 cudaMemcpyDeviceToHost, ds.st));
      }
    }
    db_band_destroy(bd);
    ds.sync();
  }
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
