// Drop-in entry points of the Dirac C API for the calibration hot path.
//
// sagefit_visibilities restates the SAGE/EM orchestration of lmfit.c:778-1053 on a device-resident
// problem: the residual of the full model stays in HBM for the whole call, each cluster visit is
//   [hidden data + first normal equations] -> LM iterations -> [residual with the new Jones]
// and the host only sees scalars and the 8N-vectors the LM decisions need.
#include <math.h>
#include <string.h>
#include <thread>
#include <vector>

#include "../../include/dirac_b200.h"
#include "problem.h"

void db_lm_chunk(dirac_b200_problem *pr, int k, int ck, double *pblk_dev, double2 *r, int itmax,
                 const double *opts, int linsolv, int os, int randomize, double *info,
                 bool hidden_ready);
void db_rlm_chunk(dirac_b200_problem *pr, int k, int ck, double *pblk_dev, double2 *r, int itmax,
                  int linsolv, int os, int randomize, double nulow, double nuhigh,
                  double *robust_nu, double *info, bool hidden_ready);
bool db_cluster_needs_rowmap(const dirac_b200_problem *pr, int k);
void db_cluster_hidden(dirac_b200_problem *pr, int k, double2 *r, int sign, double beta);
int db_lbfgs_fit(dirac_b200_problem *pr, double *p, int m, int itmax, int M, int robust,
                 double nu, bool res_held);
void db_lbfgs_fit_minibatch(dirac_b200_problem *pr, double *p, int m, int itmax, int M, double nu);
void db_rtr_chunk(dirac_b200_problem *pr, int k, int ck, double *pblk_dev, double2 *r, int kind,
                  int itmax_a, int itmax_b, double nulow, double nuhigh, double *robust_nu,
                  double *info, bool hidden_ready, const double *aug_y, const double *aug_bz,
                  double aug_rho);
// internal solver mode of dirac_b200_sagefit_admm_rtr: every visit by rtr_solve_nocuda_robust_admm
#define SM_RTR_ADMM_ 7

static bool is_robust_mode(int solver_mode) {
  return solver_mode == SM_OSLM_OSRLM_RLBFGS || solver_mode == SM_RLM_RLBFGS ||
         solver_mode == SM_RTR_OSRLM_RLBFGS || solver_mode == SM_NSD_RLBFGS ||
         solver_mode == SM_RTR_ADMM_;
}

// SAGE/EM on an already resident problem.  pp: host, in/out.  If x_out != NULL the final residual is
// written there (API layout).  Mirrors lmfit.c:778-1053.
extern "C" int dirac_b200_sagefit(dirac_b200_problem *pr, double *pp, double *x_out,
                                  int max_emiter, int max_iter, int max_lbfgs, int lbfgs_m,
                                  int linsolv, int solver_mode, double nulow, double nuhigh,
                                  int randomize, double *mean_nu, double *res_0, double *res_1) {
  if (solver_mode < 0 || solver_mode > 6 + (pr->aug_rho ? 1 : 0)) {
    fprintf(stderr, "%s: %d: undefined solver mode\n", __FILE__, __LINE__);  // lmfit.c:957-962
    exit(1);
  }
  DevProblem &d = pr->d;
  const int M = d.M;
  const int m = (int)pr->d.npar;
  const long long n = (long long)d.Nbase * d.tilesz * 8;
  const ClusterDesc *hc = d.h_clus;
  // every solve derives the Gram tensors of the coherencies afresh (nothing computed from the inputs
  // of a previous call is reused, even when the same coherencies are still resident)
  if (pr->lm.ready) memset(pr->lm.T_valid, 0, d.Mt);
  // CPU-path LM thresholds (lmfit.c:801)
  double opts[5] = {1e-3, 1e-15, 1e-15, 1e-20, -1e-6};
  double info[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  double robust_nu0 = nulow;
  double rtr_nu = nulow;  // lmdata.robust_nu of the RTR / NSD visits
  // cluster-sharded run (DESIGN.md §9): M local clusters, global cluster index k0 + cj; per-cluster
  // bookkeeping vectors are global and summed over the ranks after every sweep
  const bool sharded = pr->world > 1;
  const int MG = sharded ? pr->m_global : M;
  const int k0 = sharded ? pr->k_global0 : 0;
  std::vector<double> nerr(MG, 0.0), robust_nuM(MG, 0.0);
  const bool robust = is_robust_mode(solver_mode);
  // Sharded sweep exchange: ONE message per sweep, [residual delta | Jones delta | nerr], formed on
  // the device, summed over the ranks by one all-reduce on the library's stream
  const size_t xb_len = (size_t)8 * d.R + (size_t)m + (size_t)MG;
  if (sharded) {
    db_lm_init(pr);
    if (!pr->pm) pr->pm = (decltype(pr->pm))db_malloc(sizeof(double2) * 4 * d.R);
    if (!pr->xb) {
      pr->xb = (double *)db_malloc(sizeof(double) * (xb_len + 8));
      pr->pp_start = (double *)db_malloc(sizeof(double) * ((size_t)m + 8));
    }
  }
  // sum a small host vector over the ranks through the device scratch pr->g
  auto allreduce_host = [&](double *v, int cnt) {
    DB_CHECK(cudaMemcpyAsync(pr->g, v, sizeof(double) * cnt, cudaMemcpyHostToDevice, d.stream));
    db_allreduce(pr, pr->g, cnt);
    DB_CHECK(cudaMemcpyAsync(v, pr->g, sizeof(double) * cnt, cudaMemcpyDeviceToHost, d.stream));
    db_stream_sync(d.stream);
  };

  DB_CHECK(cudaMemcpyAsync(d.pp, pp, sizeof(double) * m, cudaMemcpyHostToDevice, d.stream));
  // residual of the current model: r = x - sum_k model_k, res_0 = ||r|| / n   (lmfit.c:866-869)
  // (r is pr->res, read afresh where it is used: an LM visit may hand back its residual in another
  // buffer, lm.cu db_lm_chunk)
  db_predict_dev(pr, d.pp, pr->res, 1, 1, 0.0, 0);
  *res_0 = sqrt(db_read_scalar(pr, 0)) / (double)n;

  int weighted_iter = 0;
  const int total_iter = MG * max_iter;
  const int iter_bar = (int)ceil((0.80 / (double)MG) * ((double)total_iter));
  for (int ci = 0; ci < max_emiter; ci++) {
    if (sharded) {
      // remember the state every rank starts the sweep from
      DB_CHECK(cudaMemcpyAsync(pr->pm, pr->res, sizeof(double2) * 4 * d.R, cudaMemcpyDeviceToDevice,
                               d.stream));
      DB_CHECK(cudaMemcpyAsync(pr->pp_start, d.pp, sizeof(double) * m, cudaMemcpyDeviceToDevice,
                               d.stream));
      for (int g = 0; g < MG; g++)
        if (g < k0 || g >= k0 + M) nerr[g] = 0.0;  // other ranks' entries come back by the sum
    }
    {
      // plain LM this sweep?  then assemble + factorise every cluster's first system as one batch
      const bool last_em = (ci == max_emiter - 1);
      const bool plain = (solver_mode == SM_LM_LBFGS) || (solver_mode == SM_OSLM_LBFGS && last_em);
      if (plain && linsolv == 0 && max_iter > 0 && !weighted_iter && !pr->aug_rho)
        db_prefactor_sweep(pr, opts[0]);
    }
    for (int cl = 0; cl < M; cl++) {
      const int cj = cl;          // local cluster index (device tables)
      const int cg = k0 + cl;     // global cluster index (bookkeeping)
      int this_itermax;
      if (weighted_iter) {
        this_itermax = (int)((0.20 * nerr[cg]) * ((double)total_iter)) + iter_bar;
      } else {
        this_itermax = max_iter;
      }
      if (this_itermax > 0) {
        double init_res = 0.0, final_res = 0.0;
        // hybrid chunks that do not tile the interval evenly: hidden data and residual of the whole
        // cluster with the reference's row-based chunk map, the LM fits in between
        const bool hr = db_cluster_needs_rowmap(pr, cj);
        if (hr) db_cluster_hidden(pr, cj, pr->res, +1, pr->world > 1 ? pr->beta : 1.0);
        for (int ck = 0; ck < hc[cj].nchunk; ck++) {
          const int poff = d.h_chunk_poff[hc[cj].chunk0 + ck];
          double *pblk = d.pp + poff;
          const bool last = (ci == max_emiter - 1);
          if (solver_mode == SM_RTR_ADMM_) {
            // ADMM J-update as the reference does it (admm_solve.c:331-352): robust RTR on the
            // consensus-augmented cost, whatever solver_mode the caller named
            if (!ci) rtr_nu = robust_nu0;
            db_rtr_chunk(pr, cj, ck, pblk, pr->res, 5, this_itermax + 5, this_itermax + 10, nulow,
                         nuhigh, &rtr_nu, info, hr, pr->aug_y_host + poff, pr->aug_bz_host + poff,
                         pr->aug_rho[cg]);
            if (last) robust_nuM[cg] += rtr_nu;
            init_res += info[0];
            final_res += info[1];
            continue;
          }
          if (pr->aug_rho)  // consensus terms of this block (dirac_b200_sagefit_admm)
            db_lm_set_aug(pr->aug_dev + poff, pr->aug_dev + d.npar + poff, pr->aug_y_host + poff,
                          pr->aug_bz_host + poff, pr->aug_rho[cg]);
          if (solver_mode == SM_OSLM_LBFGS) {
            db_lm_chunk(pr, cj, ck, pblk, pr->res, this_itermax, opts, linsolv, last ? 0 : 1,
                        randomize, info, hr);
          } else if (solver_mode == SM_LM_LBFGS) {
            db_lm_chunk(pr, cj, ck, pblk, pr->res, this_itermax, opts, linsolv, 0, randomize, info,
                        hr);
          } else if (solver_mode == SM_RLM_RLBFGS) {
            if (last) {
              double nu = robust_nu0;
              db_rlm_chunk(pr, cj, ck, pblk, pr->res, this_itermax, linsolv, 0, randomize, nulow,
                           nuhigh, &nu, info, hr);
              robust_nuM[cg] += nu;
            } else {
              db_lm_chunk(pr, cj, ck, pblk, pr->res, this_itermax, opts, linsolv, 1, randomize,
                          info, hr);
            }
          } else if (solver_mode == SM_RTR_OSLM_LBFGS) {
            // RSD + RTR (lmfit.c:934-937)
            db_rtr_chunk(pr, cj, ck, pblk, pr->res, 4, this_itermax + 5, this_itermax + 10, nulow,
                         nuhigh, &rtr_nu, info, hr, nullptr, nullptr, 0.0);
          } else if (solver_mode == SM_RTR_OSRLM_RLBFGS) {
            // robust RTR; nu persists from visit to visit after the first sweep (lmfit.c:938-947)
            if (!ci) rtr_nu = robust_nu0;
            db_rtr_chunk(pr, cj, ck, pblk, pr->res, 5, this_itermax + 5, this_itermax + 10, nulow,
                         nuhigh, &rtr_nu, info, hr, nullptr, nullptr, 0.0);
            if (last) robust_nuM[cg] += rtr_nu;
          } else if (solver_mode == SM_NSD_RLBFGS) {
            // Nesterov's accelerated descent (lmfit.c:948-957)
            if (!ci) rtr_nu = robust_nu0;
            db_rtr_chunk(pr, cj, ck, pblk, pr->res, 6, this_itermax + 15, 0, nulow, nuhigh, &rtr_nu,
                         info, hr, nullptr, nullptr, 0.0);
            if (last) robust_nuM[cg] += rtr_nu;
          } else {  // SM_OSLM_OSRLM_RLBFGS
            if (last) {
              double nu = robust_nu0;
              db_rlm_chunk(pr, cj, ck, pblk, pr->res, this_itermax, linsolv, 1, randomize, nulow,
                           nuhigh, &nu, info, hr);
              robust_nuM[cg] += nu;
            } else {
              db_lm_chunk(pr, cj, ck, pblk, pr->res, this_itermax, opts, linsolv, 1, randomize,
                          info, hr);
            }
          }
          init_res += info[0];
          final_res += info[1];
          if (pr->aug_rho) db_lm_set_aug(nullptr, nullptr, nullptr, nullptr, 0.0);
        }
        if (hr) db_cluster_hidden(pr, cj, pr->res, -1, pr->world > 1 ? pr->beta : 1.0);
        if (init_res > 0.0) {
          nerr[cg] = (init_res - final_res) / init_res;
          if (nerr[cg] < 0.0) nerr[cg] = 0.0;
        } else {
          nerr[cg] = 0.0;
        }
        if (robust && ci == max_emiter - 1) robust_nuM[cg] /= (double)hc[cj].nchunk;
      }
    }
    if (sharded) {
      // r <- r_start + sum_ranks (r_local - r_start), pp <- pp_start + sum_ranks (pp_local - pp_start)
      // (every rank changed only its own clusters' Jones blocks), nerr <- sum of the local entries
      double *xb = pr->xb;
      double2 *xr = reinterpret_cast<double2 *>(xb);
      double2 *xp = reinterpret_cast<double2 *>(xb + (size_t)8 * d.R);
      DB_CHECK(cudaMemcpyAsync(xr, pr->res, sizeof(double2) * 4 * d.R, cudaMemcpyDeviceToDevice,
                               d.stream));
      db_launch_axpby(pr->pm, xr, 4 * d.R, -1.0, 1.0, d.stream);
      DB_CHECK(cudaMemcpyAsync(xp, d.pp, sizeof(double) * m, cudaMemcpyDeviceToDevice, d.stream));
      db_launch_axpby(reinterpret_cast<double2 *>(pr->pp_start), xp, m / 2, -1.0, 1.0, d.stream);
      DB_CHECK(cudaMemcpyAsync(xb + (size_t)8 * d.R + m, nerr.data(), sizeof(double) * MG,
                               cudaMemcpyHostToDevice, d.stream));
      db_allreduce(pr, xb, (long long)xb_len);
      DB_CHECK(cudaMemcpyAsync(nerr.data(), xb + (size_t)8 * d.R + m, sizeof(double) * MG,
                               cudaMemcpyDeviceToHost, d.stream));
      DB_CHECK(cudaMemcpyAsync(pr->res, pr->pm, sizeof(double2) * 4 * d.R, cudaMemcpyDeviceToDevice,
                               d.stream));
      db_launch_axpby(xr, pr->res, 4 * d.R, 1.0, 1.0, d.stream);
      DB_CHECK(cudaMemcpyAsync(d.pp, pr->pp_start, sizeof(double) * m, cudaMemcpyDeviceToDevice,
                               d.stream));
      db_launch_axpby(xp, reinterpret_cast<double2 *>(d.pp), m / 2, 1.0, 1.0, d.stream);
      db_count_launch(4);
      db_stream_sync(d.stream);  // nerr steers the next sweep's iteration budgets
    }
    double total_err = 0.0;
    for (int cj = 0; cj < MG; cj++) total_err += fabs(nerr[cj]);
    if (total_err > 0.0)
      for (int cj = 0; cj < MG; cj++) nerr[cj] *= 1.0 / total_err;
    if (randomize) weighted_iter = !weighted_iter;
  }
  if (robust) {
    if (sharded) allreduce_host(robust_nuM.data(), MG);
    double s = 0.0;
    for (int cj = 0; cj < MG; cj++) s += fabs(robust_nuM[cj]);
    robust_nu0 = s / (double)MG;
    if (robust_nu0 < nulow) robust_nu0 = nulow;
    else if (robust_nu0 > nuhigh) robust_nu0 = nuhigh;
  }
  DB_CHECK(cudaMemcpyAsync(pp, d.pp, sizeof(double) * m, cudaMemcpyDeviceToHost, d.stream));
  db_stream_sync(d.stream);

  // Every visit of the sweeps leaves pr->res = x - sum_k model_k at the Jones it hands back (the
  // sharded merge adds the ranks' changes to it), so the full-batch LBFGS stage starts from that
  // residual, and each step it accepts leaves the residual at the new iterate in the same place.
  const bool minibatch = max_lbfgs > 0 && robust && lbfgs_m < 0;
  const bool lbfgs_stage = max_lbfgs > 0 && (!robust || lbfgs_m != 0);
  int steps = 0;  // accepted full-batch LBFGS steps
  if (max_lbfgs > 0) {
    if (robust) {
      if (lbfgs_m > 0) {
        steps = db_lbfgs_fit(pr, pp, m, max_lbfgs, lbfgs_m, 1, robust_nu0, true);
      } else if (lbfgs_m < 0) {
        // stochastic LBFGS over 5 row windows of the interval (lmfit.c:1027-1029)
        db_lbfgs_fit_minibatch(pr, pp, m, max_lbfgs, -lbfgs_m, robust_nu0);
      }
    } else {
      steps = db_lbfgs_fit(pr, pp, m, max_lbfgs, lbfgs_m, 0, 0.0, true);
    }
  }
  // final residual, in place in x   (lmfit.c:1039-1044)
  // (the LBFGS stages move the host Jones only)
  if (lbfgs_stage)
    DB_CHECK(cudaMemcpyAsync(d.pp, pp, sizeof(double) * m, cudaMemcpyHostToDevice, d.stream));
  // After an LBFGS step the residual in pr->res is the line model's at the answer, formed from a
  // fresh x - V0.  Without one it is the sweeps' (a visit adds and subtracts its cluster's model, and
  // on a problem solved to rounding level that rounding could show as res_1 > res_0), or, after the
  // minibatch stage, only some rows' residual: predicted afresh then, as the reference does.
  if (steps > 0 || (db_opt(DB_OPT_SWEEP_RESIDUAL) && !minibatch)) {
    db_launch_sumsq(pr->res, 4 * d.R, pr->partials, d.scal, d.counters, d.stream);
    db_count_launch(1);
  } else {
    db_predict_dev(pr, d.pp, pr->res, 1, 1, 0.0, 0);
  }
  *res_1 = sqrt(db_read_scalar(pr, 0)) / (double)n;
  if (x_out) db_download_vis(pr, pr->res, x_out);
  *mean_nu = robust_nu0;
  DB_CHECK(cudaGetLastError());
  return (*res_1 > *res_0) ? -1 : 0;
}

extern "C" int sagefit_visibilities(double *u, double *v, double *w, double *x, int N, int Nbase,
                                    int tilesz, baseline_t *barr, clus_source_t *carr,
                                    double *coh, int M, int Mt, double freq0, double fdelta,
                                    double *pp, double uvmin, int Nt, int max_emiter, int max_iter,
                                    int max_lbfgs, int lbfgs_m, int gpu_threads, int linsolv,
                                    int solver_mode, double nulow, double nuhigh, int randomize,
                                    double *mean_nu, double *res_0, double *res_1) {
  (void)u; (void)v; (void)w; (void)freq0; (void)fdelta; (void)uvmin; (void)Nt; (void)gpu_threads;
  dirac_b200_problem *pr = dirac_b200_create(N, Nbase, tilesz, barr, carr, M, Mt, coh, x);
  int rv = dirac_b200_sagefit(pr, pp, x, max_emiter, max_iter, max_lbfgs, lbfgs_m, linsolv,
                              solver_mode, nulow, nuhigh, randomize, mean_nu, res_0, res_1);
  dirac_b200_destroy(pr);
  return rv;
}

#define SAGEFIT_ALIAS(name)                                                                      \
  extern "C" int name(double *u, double *v, double *w, double *x, int N, int Nbase, int tilesz,  \
                      baseline_t *barr, clus_source_t *carr, double *coh, int M, int Mt,         \
                      double freq0, double fdelta, double *pp, double uvmin, int Nt,             \
                      int max_emiter, int max_iter, int max_lbfgs, int lbfgs_m, int gpu_threads, \
                      int linsolv, int solver_mode, double nulow, double nuhigh, int randomize,  \
                      double *mean_nu, double *res_0, double *res_1) {                           \
    return sagefit_visibilities(u, v, w, x, N, Nbase, tilesz, barr, carr, coh, M, Mt, freq0,     \
                                fdelta, pp, uvmin, Nt, max_emiter, max_iter, max_lbfgs, lbfgs_m, \
                                gpu_threads, linsolv, solver_mode, nulow, nuhigh, randomize,     \
                                mean_nu, res_0, res_1);                                          \
  }
SAGEFIT_ALIAS(sagefit_visibilities_dual_pt_flt)
SAGEFIT_ALIAS(sagefit_visibilities_dual_pt)
SAGEFIT_ALIAS(sagefit_visibilities_dual_pt_one_gpu)

// LBFGS over all clusters on a resident problem, as bfgsfit_visibilities runs it (lmfit.c:1056-1180):
// pp host, in/out; the cost before and after; the residual at the solution goes to pr->res only when
// keep_residual (a caller that forms its own residual spares the store)
int db_bfgsfit_dev(dirac_b200_problem *pr, double *pp, int max_lbfgs, int lbfgs_m, int solver_mode,
                   double mean_nu, double *res_0, double *res_1, bool keep_residual) {
  DevProblem &d = pr->d;
  const int m = d.N * d.Mt * 8;
  const long long n = (long long)d.Nbase * d.tilesz * 8;
  DB_CHECK(cudaMemcpyAsync(d.pp, pp, sizeof(double) * m, cudaMemcpyHostToDevice, d.stream));
  db_predict_dev(pr, d.pp, nullptr, 0, 1, 0.0, 0);
  *res_0 = sqrt(db_read_scalar(pr, 0)) / (double)n;
  if (max_lbfgs > 0) {
    int M_ = lbfgs_m > 0 ? lbfgs_m : -lbfgs_m;
    if (is_robust_mode(solver_mode)) {
      db_lbfgs_fit(pr, pp, m, max_lbfgs, M_, 1, mean_nu, false);
    } else {
      db_lbfgs_fit(pr, pp, m, max_lbfgs, M_, 0, 0.0, false);
    }
  }
  DB_CHECK(cudaMemcpyAsync(d.pp, pp, sizeof(double) * m, cudaMemcpyHostToDevice, d.stream));
  db_predict_dev(pr, d.pp, keep_residual ? pr->res : nullptr, keep_residual ? 1 : 0, 1, 0.0, 0);
  *res_1 = sqrt(db_read_scalar(pr, 0)) / (double)n;
  return (*res_1 > *res_0) ? -1 : 0;
}

extern "C" int bfgsfit_visibilities(double *u, double *v, double *w, double *x, int N, int Nbase,
                                    int tilesz, baseline_t *barr, clus_source_t *carr,
                                    double *coh, int M, int Mt, double freq0, double fdelta,
                                    double *pp, double uvmin, int Nt, int max_lbfgs, int lbfgs_m,
                                    int gpu_threads, int solver_mode, double mean_nu,
                                    double *res_0, double *res_1) {
  (void)u; (void)v; (void)w; (void)freq0; (void)fdelta; (void)uvmin; (void)Nt; (void)gpu_threads;
  dirac_b200_problem *pr = dirac_b200_create(N, Nbase, tilesz, barr, carr, M, Mt, coh, x);
  const int rv = db_bfgsfit_dev(pr, pp, max_lbfgs, lbfgs_m, solver_mode, mean_nu, res_0, res_1, true);
  db_download_vis(pr, pr->res, x);
  DB_CHECK(cudaGetLastError());
  dirac_b200_destroy(pr);
  return rv;
}

extern "C" int bfgsfit_visibilities_gpu(double *u, double *v, double *w, double *x, int N,
                                        int Nbase, int tilesz, baseline_t *barr,
                                        clus_source_t *carr, double *coh, int M, int Mt,
                                        double freq0, double fdelta, double *pp, double uvmin,
                                        int Nt, int max_lbfgs, int lbfgs_m, int gpu_threads,
                                        int solver_mode, double mean_nu, double *res_0,
                                        double *res_1) {
  return bfgsfit_visibilities(u, v, w, x, N, Nbase, tilesz, barr, carr, coh, M, Mt, freq0, fdelta,
                              pp, uvmin, Nt, max_lbfgs, lbfgs_m, gpu_threads, solver_mode, mean_nu,
                              res_0, res_1);
}

// ------------------------------------------------------------------------------------------------
// index / flag helpers the driver calls directly (host, bit-exact integer work)
// ------------------------------------------------------------------------------------------------
// canonical row order (0,1),(0,2)...(N-2,N-1) per timeslot; flags untouched
// (baselinegen_threadfn, baseline_utils.c:438-466)
extern "C" int generate_baselines(int Nbase, int tilesz, int N, baseline_t *barr, int Nt) {
  (void)Nt;
  for (int t = 0; t < tilesz; t++) {
    int sta1 = 0, sta2 = 1;
    baseline_t *b = barr + (size_t)t * Nbase;
    for (int cj = 0; cj < Nbase; cj++) {
      b[cj].sta1 = sta1;
      b[cj].sta2 = sta2;
      if (sta2 < N - 1) {
        sta2++;
      } else if (sta1 < N - 2) {
        sta1++;
        sta2 = sta1 + 1;
      } else {
        sta1 = 0;
        sta2 = 1;
      }
    }
  }
  return 0;
}

// flag[ci] > 0 -> barr.flag = 1 and the 8 data reals zeroed, else barr.flag = 0
// (preflag_threadfn, baseline_utils.c:206-227)
extern "C" int preset_flags_and_data(int Nbase, double *flag, baseline_t *barr, double *x, int Nt) {
  (void)Nt;
  for (int ci = 0; ci < Nbase; ci++) {
    if (flag[ci] > 0.0) {
      barr[ci].flag = 1;
      for (int c = 0; c < 8; c++) x[8 * (size_t)ci + c] = 0.0;
    } else {
      barr[ci].flag = 0;
    }
  }
  return 0;
}

// uv-distance taper of the data, the driver's -W option, applied between preset_flags_and_data and the
// coherency prediction (fullbatch_mode.cpp:329-332): every row is scaled by 1 / (1 + 1.8 exp(-0.05 d)),
// d = |(u,v)| freq0 in wavelengths (u, v arrive divided by c); rows beyond 400 wavelengths are left
// alone (threadfn_setblweight / ncp_weight, updatenu.c:339-372).  A 1 GB pass at 512 stations: split
// over Nt host threads like the reference's.
extern "C" void whiten_data(int Nbase, double *x, double *u, double *v, double freq0, int Nt) {
  auto taper = [=](long long r0, long long r1) {
    for (long long r = r0; r < r1; r++) {
      const double uu = u[r] * freq0, vv = v[r] * freq0;
      const double ud = sqrt(uu * uu + vv * vv);
      if (ud > 400.0) continue;  // weight exactly 1
      const double a = 1.0 / (1.0 + 1.8 * exp(-0.05 * ud));
      for (int c = 0; c < 8; c++) x[8 * r + c] *= a;
    }
  };
  if (Nt < 1) Nt = 1;
  const long long per = ((long long)Nbase + Nt - 1) / Nt;
  if (Nt == 1 || Nbase < (1 << 16)) {
    taper(0, Nbase);
    return;
  }
  std::vector<std::thread> th;
  for (long long r0 = per; r0 < Nbase; r0 += per)
    th.emplace_back(taper, r0, r0 + per < Nbase ? r0 + per : (long long)Nbase);
  taper(0, per < Nbase ? per : (long long)Nbase);
  for (auto &t : th) t.join();
}
