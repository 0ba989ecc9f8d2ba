// Riemannian trust-region (RTR), Riemannian steepest-descent (RSD) and Nesterov (NSD) solvers of one
// (cluster, chunk): solver_mode 4 (SM_RTR_OSLM_LBFGS), 5 (SM_RTR_OSRLM_RLBFGS, the reference
// driver's default -j 5, src/MS/data.cpp:69) and 6 (SM_NSD_RLBFGS).
//
// Control flow: rtr_algo.h (restatement of rtr_solve.c / rtr_solve_robust.c, decision for decision).
//
// Data flow: NOT the reference's.  One streaming pass condenses the chunk's rows into per-baseline
// tensors (k_rtr_stats); every cost / gradient / Hessian-vector product the solvers ask for is then
// an O(Nbase) kernel (k_rtr_eval) instead of a pass over all rows (kernels_rtr.cu).  The host keeps
// the 8N-vectors and takes the decisions, as in the LM family (lm.cu).
#include <math.h>
#include <string.h>
#include <algorithm>
#include <vector>

#include "../../include/dirac_b200.h"
#include "problem.h"
#include "rtr.h"
#include "rtr_algo.h"

int db_cluster_pass(dirac_b200_problem *pr, int k, const double *pblk_dev, const double2 *in,
                    double2 *out, int mode, int write_out, double *jte_dev, int cost_slot, int t0,
                    int t1, const double2 *wt, double beta, bool jte_zeroed,
                    const double *pblk_old, bool form_hidden = false);
void db_chunk_range(const DevProblem &d, int k, int ck, int *t0, int *t1);

struct RtrWork {
  int N, Nbase, nslice;
  double2 *TDpart, *TD;   // [nslice][Nbase][32], [Nbase][32]
  double *scpart, *sc;    // [nslice][3][Nbase], [3][Nbase]
  double *xdev, *edev;    // [8N] each
  double *outdev;         // [8N | N | N | 4]
  double *h;              // pinned: x [8N], eta [8N], out [8N + 2N + 4]
  // mailbox of k_rtr_eval: results and completion flag in host-mapped memory
  double *mbox, *mbox_dev;              // [8N | N | N | flag]
  unsigned int *arrive;                 // device
  unsigned long long epoch;
};

static RtrWork *rtr_init(dirac_b200_problem *pr) {
  if (pr->rtr) return pr->rtr;
  DevProblem &d = pr->d;
  RtrWork *w = new RtrWork();
  w->N = d.N;
  w->Nbase = d.Nbase;
  // (baseline block, time slice) CTAs: about one per SM.  More slices shorten the rows per thread but
  // every slice writes (and the reduction re-reads) 528 B of partial tensors per baseline, against
  // 128 B per row streamed: at 62 stations x 120 timeslots 10 slices already add 35 % of traffic
  const int nbb = (d.Nbase + 127) / 128;
  int ns = (db_sm_count() + nbb - 1) / nbb;
  if (ns > d.tilesz) ns = d.tilesz;
  if (ns < 1) ns = 1;
  w->nslice = ns;
  const size_t nb = (size_t)d.Nbase;
  w->TD = (double2 *)db_malloc(sizeof(double2) * 32 * nb);
  w->sc = (double *)db_malloc(sizeof(double) * 3 * nb);
  w->TDpart = ns > 1 ? (double2 *)db_malloc(sizeof(double2) * 32 * nb * ns) : nullptr;
  w->scpart = ns > 1 ? (double *)db_malloc(sizeof(double) * 3 * nb * ns) : nullptr;
  const size_t n8 = (size_t)8 * d.N;
  w->xdev = (double *)db_malloc(sizeof(double) * n8);
  w->edev = (double *)db_malloc(sizeof(double) * n8);
  w->outdev = (double *)db_malloc(sizeof(double) * (n8 + 2 * d.N + 8));
  DB_CHECK(cudaMallocHost((void **)&w->h, sizeof(double) * (3 * n8 + 2 * d.N + 16)));
  DB_CHECK(cudaHostAlloc((void **)&w->mbox, sizeof(double) * (n8 + 2 * d.N + 16),
                         cudaHostAllocMapped));
  DB_CHECK(cudaHostGetDevicePointer((void **)&w->mbox_dev, w->mbox, 0));
  memset(w->mbox, 0, sizeof(double) * (n8 + 2 * d.N + 16));
  w->arrive = (unsigned int *)db_malloc(256);
  DB_CHECK(cudaMemsetAsync(w->arrive, 0, 256, d.stream));
  w->epoch = 0;
  pr->rtr = w;
  return w;
}

void db_rtr_free(dirac_b200_problem *pr) {
  RtrWork *w = pr->rtr;
  if (!w) return;
  db_free(w->TD); db_free(w->sc);
  if (w->TDpart) { db_free(w->TDpart); db_free(w->scpart); }
  db_free(w->xdev); db_free(w->edev); db_free(w->outdev);
  cudaFreeHost(w->h);
  cudaFreeHost(w->mbox);
  db_free(w->arrive);
  delete w;
  pr->rtr = nullptr;
}

// ------------------------------------------------------------------------------------------------
// device evaluator (the concept rtr_algo.h asks for) on the condensed chunk
// ------------------------------------------------------------------------------------------------
struct RtrDevEval {
  dirac_b200_problem *pr;
  RtrWork *w;
  int k, t0, t1, N, n8;
  long long nrows;            // rows of the chunk, flagged ones included (the reference's M)
  std::vector<double> x_on_dev;  // the Jones w->xdev holds (empty: unknown)
  bool force_dev = false;     // Jones through device memory at any N (test hook only)
  int last_ns = 0, last_tslice = 0;  // time slicing of the last condensation
  bool last_inline = false;          // the last evaluation had its vectors in the parameter block

  // condense the rows of the chunk.  xw != null: Student's-t row weights at xw with nu; returns
  // sum(log w - w) then
  double condense(const double *xw_host, double nu, bool tensors) {
    DevProblem &d = pr->d;
    RtrStatsArgs a;
    a.coh_k = d.coh + (size_t)k * 4 * d.R;
    a.d = pr->lm.dbuf;
    a.flag = d.flag;
    a.blpq = d.blpq;
    a.xw = nullptr;
    if (xw_host) {
      upload_x(xw_host);
      a.xw = w->xdev;
    }
    a.nu = nu;
    a.R = d.R; a.N = d.N; a.Nbase = d.Nbase;
    a.t_begin = t0; a.t_end = t1;
    const int nt = t1 - t0;
    int ns = w->nslice < nt ? w->nslice : nt;
    a.tslice = (nt + ns - 1) / ns;
    ns = (nt + a.tslice - 1) / a.tslice;
    last_ns = ns;
    last_tslice = a.tslice;
    a.TD = ns > 1 ? w->TDpart : w->TD;
    a.sc = ns > 1 ? w->scpart : w->sc;
    a.tensors = tensors ? 1 : 0;
    db_prof_begin(9, (double)nt * d.Nbase * 129.0, d.stream);
    db_launch_rtr_stats(&a, ns, d.stream);
    db_prof_end(d.stream);
    db_count_launch(1);
    if (ns > 1) {
      if (tensors)
        db_launch_rtr_reduce((const double *)w->TDpart, (double *)w->TD, (size_t)64 * d.Nbase, ns,
                             d.stream);
      db_launch_rtr_reduce(w->scpart, w->sc, (size_t)3 * d.Nbase, ns, d.stream);
      db_count_launch(tensors ? 2 : 1);
    }
    if (!xw_host) return 0.0;
    db_launch_rtr_plane_sum(w->sc, d.Nbase, 1, w->outdev, d.stream);
    db_count_launch(1);
    DB_CHECK(cudaMemcpyAsync(w->h + 2 * n8, w->outdev, sizeof(double), cudaMemcpyDeviceToHost,
                             d.stream));
    db_stream_sync(d.stream);
    return w->h[2 * n8];
  }

  // the Jones go up only when they changed: every Hessian-vector product of one truncated-CG run
  // is taken at the same point (every call ends with a stream synchronisation, so the pinned staging
  // buffer is free again)
  void upload_x(const double *x) {
    if (x_on_dev.size() == (size_t)n8 && !memcmp(x_on_dev.data(), x, sizeof(double) * n8)) return;
    memcpy(w->h, x, sizeof(double) * n8);
    DB_CHECK(cudaMemcpyAsync(w->xdev, w->h, sizeof(double) * n8, cudaMemcpyHostToDevice,
                             pr->d.stream));
    x_on_dev.assign(x, x + n8);
  }

  // one launch of k_rtr_eval
  void launch(const double *x, const double *eta, double *fcost, double *vec, double *cnt) {
    DevProblem &d = pr->d;
    // results come back through the mailbox: no device-to-host copy, no stream synchronisation
    const bool inl = N <= RTR_INLINE_MAXN && !force_dev;
    last_inline = inl;
    RtrEvalInl P;
    RtrEvalArgs &a = P.a;
    a.TD = w->TD; a.sc = w->sc; a.x = w->xdev; a.eta = eta ? w->edev : nullptr;
    a.out = vec ? w->outdev : nullptr;
    a.cost = fcost ? w->outdev + n8 : nullptr;
    a.count = cnt ? w->outdev + n8 + N : nullptr;
    a.N = N; a.Nbase = d.Nbase;
    a.arrive = w->arrive;
    a.hmail = w->mbox_dev;
    a.flag = reinterpret_cast<unsigned long long *>(w->mbox_dev + n8 + 2 * N + 2);
    a.epoch = ++w->epoch;
    if (inl) {
      // Jones and tangent vector ride in the parameter block: the evaluation is one launch
      memcpy(P.xin, x, sizeof(double) * n8);
      if (eta) memcpy(P.ein, eta, sizeof(double) * n8);
    } else {
      double *he = w->h + n8;
      upload_x(x);
      if (eta) {
        memcpy(he, eta, sizeof(double) * n8);
        DB_CHECK(cudaMemcpyAsync(w->edev, he, sizeof(double) * n8, cudaMemcpyHostToDevice,
                                 d.stream));
      }
    }
    db_prof_begin(10, 2.0 * d.Nbase * (512.0 + 24.0), d.stream);
    if (inl) db_launch_rtr_eval_inl(&P, d.stream);
    else db_launch_rtr_eval(&a, d.stream);
    db_prof_end(d.stream);
    db_count_launch(1);
    db_flag_wait(reinterpret_cast<volatile unsigned long long *>(w->mbox + n8 + 2 * N + 2),
                 a.epoch, d.stream);
    const double *ho = w->mbox;
    if (vec) memcpy(vec, ho, sizeof(double) * n8);
    if (fcost) {
      double s = 0.0;
      for (int i = 0; i < N; i++) s += ho[n8 + i];
      *fcost = s;
    }
    if (cnt) memcpy(cnt, ho + n8 + N, sizeof(double) * N);
  }

  // ---- evaluator concept ----
  void raw(const double *x, const double *eta, double *fcost, double *vec) {
    launch(x, eta, fcost, vec, nullptr);
  }
  void counts(double *c) {
    std::vector<double> x0(n8, 0.0);
    launch(x0.data(), nullptr, nullptr, nullptr, c);
  }
  void unit_weights() { condense(nullptr, 0.0, true); }
  double weights_at(const double *x, double nu, bool keep) {
    return condense(x, nu, keep) / (double)nrows;
  }
};

// ------------------------------------------------------------------------------------------------
// one (cluster, chunk) visit.  kind: 4 RSD+RTR, 5 robust RTR, 6 robust NSD.  robust_nu: in/out
// (lmdata.robust_nu of the reference persists from visit to visit, lmfit.c:938-957).
// ------------------------------------------------------------------------------------------------
// aug_y / aug_bz != null (kind 5): the consensus-augmented cost of the ADMM J-update
// (rtr_solve_nocuda_robust_admm); host vectors of this block.
void db_rtr_chunk(dirac_b200_problem *pr, int k, int ck, double *pblk_dev, double2 *r, int kind,
                  int itmax_a, int itmax_b, double nulow, double nuhigh, double *robust_nu,
                  double *info, bool hidden_ready, const double *aug_y, const double *aug_bz,
                  double aug_rho) {
  DevProblem &d = pr->d;
  db_lm_init(pr);
  LMWork &lw = pr->lm;
  RtrWork *w = rtr_init(pr);
  int t0, t1;
  db_chunk_range(d, k, ck, &t0, &t1);
  const int n8 = 8 * d.N;
  if (t1 <= t0) {  // empty chunk: nothing to fit, zero cost
    if (kind != 6) info[0] = 0.0;
    info[1] = 0.0;
    return;
  }
  const double beta = pr->world > 1 ? pr->beta : 1.0;
  if (!hidden_ready) {
    if (beta != 1.0)
      DB_CHECK(cudaMemcpyAsync(lw.pold, pblk_dev, sizeof(double) * n8, cudaMemcpyDeviceToDevice,
                               d.stream));
    // hidden data d = beta r + f(p_old)   (lmfit.c:890-891)
    db_cluster_pass(pr, k, pblk_dev, r, lw.dbuf, 2, 1, nullptr, 1, t0, t1, nullptr, beta,
                    false, nullptr);
  }
  RtrDevEval E;
  E.pr = pr; E.w = w; E.k = k; E.t0 = t0; E.t1 = t1; E.N = d.N; E.n8 = n8;
  E.nrows = (long long)(t1 - t0) * d.Nbase;
  std::vector<double> x(n8);
  DB_CHECK(cudaMemcpyAsync(w->h, pblk_dev, sizeof(double) * n8, cudaMemcpyDeviceToHost, d.stream));
  db_stream_sync(d.stream);
  memcpy(x.data(), w->h, sizeof(double) * n8);
  rtr::Admm aug = {aug_y, aug_bz, aug_rho};
  rtr::solve_chunk(E, kind, x.data(), itmax_a, itmax_b, nulow, nuhigh, robust_nu, info,
                   !db_opt(DB_OPT_RTR_NU_UNJOINED), aug_y ? &aug : nullptr);
  memcpy(w->h, x.data(), sizeof(double) * n8);
  DB_CHECK(cudaMemcpyAsync(pblk_dev, w->h, sizeof(double) * n8, cudaMemcpyHostToDevice, d.stream));
  // residual of the chunk with the final Jones: r = d - f(p)  (lmfit.c:980-981)
  if (!hidden_ready)
    db_cluster_pass(pr, k, pblk_dev, lw.dbuf, r, 3, 1, nullptr, 1, t0, t1, nullptr, beta,
                    false, beta != 1.0 ? lw.pold : nullptr);
  db_stream_sync(d.stream);  // w->h is reused by the next visit
}

// test hook: the device evaluator of cluster k, chunk ck, exactly as a solver visit drives it (same
// condense, same launch, same mailbox).  The hidden data of the chunk are the problem's data vector
// (dirac_b200_set_data) as they stand, copied into the visit's hidden-data buffer.
//   xw        null: unit weights; else Student's-t row weights at xw with nu (weights_at), `keep`
//             selects whether they apply to the evaluations (the tensors are rebuilt) or only the
//             scalars (sum(log w - w), unflagged rows) are condensed
//   force_dev Jones and tangent vectors through device memory at any N
//   ops[i]    evaluation i (host vectors x + 8N i, eta + 8N i): RTR_HOOK_* bits.  COUNTS alone is the
//             evaluator's counts(); otherwise one launch with the requested outputs
//   out       cost[neval], vec[neval][8N], cnt[neval][N]
//   info      [sum(log w - w) / rows (0 for unit weights), nslice, tslice] of the condensation,
//             [3] 1 if the last evaluation had its vectors in the parameter block
enum { RTR_HOOK_COST = 1, RTR_HOOK_VEC = 2, RTR_HOOK_COUNTS = 4, RTR_HOOK_ETA = 8,
       RTR_HOOK_UNIT = 16 };
extern "C" void dirac_b200_rtr_eval(dirac_b200_problem *pr, int k, int ck, const double *xw,
                                    double nu, int keep, int force_dev, int neval, const int *ops,
                                    const double *x, const double *eta, double *cost, double *vec,
                                    double *cnt, double *info) {
  DevProblem &d = pr->d;
  db_lm_init(pr);
  RtrWork *w = rtr_init(pr);
  int t0, t1;
  db_chunk_range(d, k, ck, &t0, &t1);
  if (t1 <= t0) {
    fprintf(stderr, "dirac_b200_rtr_eval: chunk %d of cluster %d is empty\n", ck, k);
    exit(1);
  }
  const int n8 = 8 * d.N;
  DB_CHECK(cudaMemcpyAsync(pr->lm.dbuf, d.x, sizeof(double2) * 4 * d.R, cudaMemcpyDeviceToDevice,
                           d.stream));
  RtrDevEval E;
  E.pr = pr; E.w = w; E.k = k; E.t0 = t0; E.t1 = t1; E.N = d.N; E.n8 = n8;
  E.nrows = (long long)(t1 - t0) * d.Nbase;
  E.force_dev = force_dev != 0;
  info[0] = 0.0;
  if (xw) info[0] = E.weights_at(xw, nu, keep != 0);
  else E.unit_weights();
  info[1] = E.last_ns;
  info[2] = E.last_tslice;
  for (int i = 0; i < neval; i++) {
    const int op = ops[i];
    if (op & RTR_HOOK_UNIT) E.unit_weights();
    if ((op & ~RTR_HOOK_UNIT) == RTR_HOOK_COUNTS) {
      E.counts(cnt + (size_t)i * d.N);
      continue;
    }
    E.launch(x + (size_t)i * n8, (op & RTR_HOOK_ETA) ? eta + (size_t)i * n8 : nullptr,
             (op & RTR_HOOK_COST) ? cost + i : nullptr,
             (op & RTR_HOOK_VEC) ? vec + (size_t)i * n8 : nullptr,
             (op & RTR_HOOK_COUNTS) ? cnt + (size_t)i * d.N : nullptr);
  }
  info[3] = E.last_inline ? 1.0 : 0.0;
  db_stream_sync(d.stream);
  DB_CHECK(cudaGetLastError());
}
