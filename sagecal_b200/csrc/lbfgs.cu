// LBFGS (two-loop recursion + Fletcher line search) on top of the device cost / gradient passes.
//
// The iteration logic restates lbfgs_fit_fullbatch (lbfgs.c:479-640), mult_hessian (:33-111),
// linesearch (:298-430), linesearch_zoom (:211-290) and cubic_interp (:116-205): same constants,
// same order of cost evaluations, same acceptance tests, because every comparison steers the
// iterates and parity with the CPU reference is judged on the solved Jones.
//
// What differs is the cost of a cost evaluation.  Every evaluation of the reference's line search
// is at x_k + alpha p_k (the reference moves a scratch vector xp along p_k by axpy; we track the
// same alpha with the same sequence of additions).  One pass over the coherencies per LBFGS
// iteration (k_stream_all<1>) leaves the line model e(alpha) = E0 - alpha E1 - alpha^2 E2 in HBM/L2;
// each of the 10-30 cost evaluations of the iteration is then a 192 B/row reduction (k_line_eval)
// instead of a full predict over all clusters, and the residual at the accepted step feeds the
// gradient pass (k_grad_tma_split) directly.  Per iteration: 2 passes over the coherencies instead of
// ~30 (cost_func / robust_cost_func, robust_lbfgs.c:674-726; func_grad(_robust), :569-669,322-416).
//
// The iterate, the gradient, the search direction and the (s, y) history live on the device; the
// two-loop recursion is one cluster kernel (kernels_lbfgs.cu).  The host keeps what is scalar: the
// line search's decisions on costs that come back as a quartic's coefficients (Gaussian) or one
// number per evaluation (Student's t), and ||g|| for the stopping test.
#include <float.h>
#include <math.h>
#include <string.h>
#include <vector>

#include "problem.h"

extern "C" {
int db_lbfgs_direction_max_pairs(void);
void db_launch_lbfgs_direction(double *pk, const double *gk, const double *s, const double *y,
                               const double *rho, int m, int npairs, int next, cudaStream_t st);
void db_launch_lbfgs_nrm2(const double *g, int m, double *out, cudaStream_t st);
void db_launch_lbfgs_step(const double *xk, const double *pk, const double *gk, double *xk1,
                          double *sk, double *yk, int m, double alpha, cudaStream_t st);
void db_launch_lbfgs_update(const double *gk, const double *sk, double *yk, const double *xk1,
                            double *xk, int m, double *rho_slot, double *out, cudaStream_t st);
void db_launch_line_eval(const double2 *E0, const double2 *E1, const double2 *E2, long long n4,
                         double alpha, int mode, double inv_nu, double *partials, double *out,
                         unsigned int *counter, cudaStream_t st);
void db_launch_line_residual(const double2 *E0, const double2 *E1, const double2 *E2, double2 *res,
                             long long n4, double alpha, cudaStream_t st);
void db_launch_line_poly(const double2 *E0, const double2 *E1, const double2 *E2, long long n4,
                         double *partials, double *out, unsigned int *counter, cudaStream_t st);
}

struct LbfgsCtx {
  dirac_b200_problem *pr;
  int robust;
  double nu;
  int m;
  long long ncost, ngrad;
  double poly[5];  // Gaussian cost along the current line: sum_j poly[j] alpha^j
};

static void line_alloc(dirac_b200_problem *pr) {
  if (pr->E0) return;
  DevProblem &d = pr->d;
  const size_t n = (size_t)4 * d.R;
  const size_t nb = (size_t)db_stream_all_nblocks(d.Nbase, d.tilesz);
  // one allocation: the three parts of the line model travel in ONE all-reduce when sharded; the
  // per-CTA quartic sums of a single-GPU pass follow them
  pr->E0 = (decltype(pr->E0))db_malloc(sizeof(double2) * n * 3 + sizeof(double) * 5 * nb);
  pr->E1 = pr->E0 + n;
  pr->E2 = pr->E1 + n;
  pr->poly_part = reinterpret_cast<double *>(pr->E2 + n);
}

// line model along pk from xk (both device vectors)
static void line_setup(LbfgsCtx *c, const double *xk, const double *pk) {
  dirac_b200_problem *pr = c->pr;
  DevProblem &d = pr->d;
  line_alloc(pr);
  StreamAllArgs s;
  memset(&s, 0, sizeof(s));
  s.coh = d.coh; s.x = d.x; s.flag = d.flag; s.pp = xk; s.pk = pk; s.clus = d.clus;
  s.chunk_poff = d.chunk_poff; s.blpq = d.blpq; s.E0 = pr->E0; s.E1 = pr->E1; s.E2 = pr->E2;
  s.R = d.R; s.N = d.N; s.Nbase = d.Nbase; s.tilesz = d.tilesz; s.M = d.M;
  s.partial = (pr->world > 1) ? 1 : 0;  // 1: the raw sums V0,V1,V2 of the local clusters
  // the Gaussian cost along the line is a quartic in alpha: five sums, then every cost evaluation of
  // the line search is arithmetic on the host.  One GPU has E0 in the line-model pass and takes the
  // sums there; sharded runs form E0 after the all-reduce and sum with k_line_poly
  const bool want_poly = !c->robust && !db_opt(DB_OPT_LINE_DIRECT);
  const bool fold_poly = want_poly && pr->world <= 1;
  s.poly_part = fold_poly ? pr->poly_part : nullptr;
  if (db_overlap_available(pr) && d.tilesz >= 8) {
    // Sharded: the kernel runs in time chunks; each chunk's 12 slices (3 vectors x 4 polarisation
    // planes) are summed over the ranks on the communication stream while the next chunk is computed
    static cudaEvent_t ev_chunk[8], ev_done;
    static bool have_ev = false;
    if (!have_ev) {
      for (int i = 0; i < 8; i++) DB_CHECK(cudaEventCreateWithFlags(&ev_chunk[i], cudaEventDisableTiming));
      DB_CHECK(cudaEventCreateWithFlags(&ev_done, cudaEventDisableTiming));
      have_ev = true;
    }
    cudaStream_t cs = db_comm_stream();
    const int nch = 8;
    const int per = (d.tilesz + nch - 1) / nch;
    db_prof_begin(7, (double)d.R * (64.0 * d.M + 65.0 + 192.0), d.stream);
    int ci = 0;
    for (int t0 = 0; t0 < d.tilesz; t0 += per, ci++) {
      const int t1 = (t0 + per < d.tilesz) ? t0 + per : d.tilesz;
      const long long r0 = (long long)t0 * d.Nbase, nr = (long long)(t1 - t0) * d.Nbase;
      StreamAllArgs c2 = s;
      c2.coh = s.coh + r0; c2.x = s.x + r0; c2.flag = s.flag + r0;
      c2.E0 = s.E0 + r0; c2.E1 = s.E1 + r0; c2.E2 = s.E2 + r0;
      c2.tilesz = t1 - t0; c2.row0 = r0;
      db_launch_line_setup_tma(&c2, d.stream);
      db_count_launch(1);
      DB_CHECK(cudaEventRecord(ev_chunk[ci], d.stream));
      DB_CHECK(cudaStreamWaitEvent(cs, ev_chunk[ci], 0));
      double *seg[12];
      long long cnt[12];
      for (int v = 0; v < 3; v++)
        for (int c = 0; c < 4; c++) {
          double2 *base = (v == 0 ? pr->E0 : v == 1 ? pr->E1 : pr->E2) + (long long)c * d.R + r0;
          seg[v * 4 + c] = reinterpret_cast<double *>(base);
          cnt[v * 4 + c] = 2 * nr;
        }
      db_allreduce_segments(pr, seg, cnt, 12, cs);
    }
    db_prof_end(d.stream);
    DB_CHECK(cudaEventRecord(ev_done, cs));
    DB_CHECK(cudaStreamWaitEvent(d.stream, ev_done, 0));
    db_launch_axpby(d.x, pr->E0, 4 * d.R, 1.0, -1.0, d.stream);  // E0 = x - V0
    db_count_launch(1);
  } else {
    db_prof_begin(7, (double)d.R * (64.0 * d.M + 65.0 + 192.0), d.stream);
    const unsigned nparts = db_launch_line_setup_tma(&s, d.stream);
    db_prof_end(d.stream);
    db_count_launch(1);
    if (fold_poly) {
      db_launch_line_poly_finish(pr->poly_part, nparts, pr->partials, d.scal + 16, d.counters,
                                 d.stream);
      db_count_launch(1);
    }
    if (pr->world > 1) {
      // sum the model polynomials of all ranks, then E0 = x - V0
      db_allreduce(pr, pr->E0, 3 * 8 * d.R);  // E0 | E1 | E2 are contiguous
      db_launch_axpby(d.x, pr->E0, 4 * d.R, 1.0, -1.0, d.stream);
      db_count_launch(1);
    }
  }
  if (want_poly) {
    if (!fold_poly) {
      db_launch_line_poly(pr->E0, pr->E1, pr->E2, 4 * d.R, pr->partials, d.scal + 16, d.counters,
                          d.stream);
      db_count_launch(1);
    }
    DB_CHECK(cudaMemcpyAsync(d.h_scal + 16, d.scal + 16, 5 * sizeof(double), cudaMemcpyDeviceToHost,
                             d.stream));
    db_stream_sync(d.stream);
    for (int j = 0; j < 5; j++) c->poly[j] = d.h_scal[16 + j];
  }
}

// phi(alpha) = cost(xk + alpha pk)
static double line_cost(LbfgsCtx *c, double alpha) {
  dirac_b200_problem *pr = c->pr;
  DevProblem &d = pr->d;
  if (!c->robust && !db_opt(DB_OPT_LINE_DIRECT)) {
    c->ncost++;
    const double *q = c->poly;
    return q[0] + alpha * (q[1] + alpha * (q[2] + alpha * (q[3] + alpha * q[4])));
  }
  db_launch_line_eval(pr->E0, pr->E1, pr->E2, 4 * d.R, alpha, c->robust ? 2 : 1,
                      c->robust ? 1.0 / c->nu : 0.0, pr->partials, d.scal, d.counters, d.stream);
  db_count_launch(1);
  c->ncost++;
  return db_read_scalar(pr, 0);
}

// gradient at p (device) into g (device) from the residual at p in pr->res: taken from the line
// model at alpha (RES_LINE), formed by a fresh predict (RES_PREDICT), or already there (RES_HELD)
enum { RES_PREDICT, RES_LINE, RES_HELD };
static void grad_eval(LbfgsCtx *c, const double *p, double *g, int res_src, double alpha) {
  dirac_b200_problem *pr = c->pr;
  DevProblem &d = pr->d;
  if (res_src == RES_LINE) {
    db_launch_line_residual(pr->E0, pr->E1, pr->E2, pr->res, 4 * d.R, alpha, d.stream);
    db_count_launch(1);
  } else if (res_src == RES_PREDICT) {
    db_predict_dev(pr, p, pr->res, 1, 0, 0.0, 0);
  }
  db_grad_dev(pr, p, g, c->robust, c->nu);
  c->ngrad++;
}

// In the three functions below `xa` is the position of the reference's scratch vector xp along
// the line (xp = xk + xa*pk); every my_daxpy(m,pk,t,xp) of the reference is `xa += t` here.
static double cubic_interp(LbfgsCtx *c, double a, double b, double *xa, double step) {
  double f0, f1, f0d, f1d, p01, p02, z0, fz0, aa, cc;
  *xa = a;
  f0 = line_cost(c, *xa);
  *xa += step;
  p01 = line_cost(c, *xa);
  *xa += -2.0 * step;
  p02 = line_cost(c, *xa);
  f0d = (p01 - p02) / (2.0 * step);
  *xa += -a + step + b;
  f1 = line_cost(c, *xa);
  *xa += step;
  p01 = line_cost(c, *xa);
  *xa += -2.0 * step;
  p02 = line_cost(c, *xa);
  f1d = (p01 - p02) / (2.0 * step);

  aa = 3.0 * (f0 - f1) / (b - a) + (f1d - f0d);
  p01 = aa * aa - f0d * f1d;
  if (p01 > 0.0) {
    cc = sqrt(p01);
    z0 = b - (f1d + cc - aa) * (b - a) / (f1d - f0d + 2.0 * cc);
    aa = (a > b) ? a : b;
    cc = (a < b) ? a : b;
    if (z0 > aa || z0 < cc) {
      fz0 = f0 + f1;
    } else {
      *xa += -b + step + a + z0 * (b - a);
      fz0 = line_cost(c, *xa);
    }
    if (f0 < f1 && f0 < fz0) return a;
    if (f1 < fz0) return b;
    return z0;
  }
  return (f0 < f1) ? a : b;
}

static double linesearch_zoom(LbfgsCtx *c, double a, double b, double *xa, double phi_0,
                              double gphi_0, double sigma, double rho, double t1, double t2,
                              double t3, double step) {
  double alphaj = 0.0, phi_j, phi_aj, gphi_j, p01, p02, aj = a, bj = b, alphak = 1.0;
  int ci = 0, found_step = 0;
  (void)t1;
  while (ci < 10) {
    p01 = aj + t2 * (bj - aj);
    p02 = bj - t3 * (bj - aj);
    alphaj = cubic_interp(c, p01, p02, xa, step);
    *xa = alphaj;
    phi_j = line_cost(c, *xa);
    *xa += -alphaj + aj;
    phi_aj = line_cost(c, *xa);
    if ((phi_j > phi_0 + rho * alphaj * gphi_0) || phi_j >= phi_aj) {
      bj = alphaj;
    } else {
      *xa += -aj + alphaj + step;
      p01 = line_cost(c, *xa);
      *xa += -2.0 * step;
      p02 = line_cost(c, *xa);
      gphi_j = (p01 - p02) / (2.0 * step);
      if ((aj - alphaj) * gphi_j <= step) {
        alphak = alphaj;
        found_step = 1;
        break;
      }
      if (fabs(gphi_j) <= -sigma * gphi_0) {
        alphak = alphaj;
        found_step = 1;
        break;
      }
      if (gphi_j * (bj - aj) >= 0) bj = aj;
      aj = alphaj;
    }
    ci++;
  }
  if (!found_step) alphak = alphaj;
  return alphak;
}

static double linesearch(LbfgsCtx *c, double alpha1, double sigma, double rho, double t1,
                         double t2, double t3, double step) {
  double xa;
  double alphai, alphai1, phi_0, phi_alphai, phi_alphai1, p01, p02, gphi_0, gphi_i, alphak, mu, tol;
  alphak = 1.0;
  phi_0 = line_cost(c, 0.0);
  tol = (0.01 * phi_0 < 1e-6) ? 0.01 * phi_0 : 1e-6;
  xa = 0.0;
  xa += step;
  p01 = line_cost(c, xa);
  xa += -2.0 * step;
  p02 = line_cost(c, xa);
  gphi_0 = (p01 - p02) / (2.0 * step);
  mu = (tol - phi_0) / (rho * gphi_0);
  if (!isnormal(mu)) return mu;
  int ci = 1;
  alphai = alpha1;
  alphai1 = 0.0;
  phi_alphai1 = phi_0;
  while (ci < 10) {
    xa = alphai;
    phi_alphai = line_cost(c, xa);
    if (phi_alphai < tol) {
      alphak = alphai;
      break;
    }
    if ((phi_alphai > phi_0 + alphai * gphi_0) || (ci > 1 && phi_alphai >= phi_alphai1)) {
      alphak = linesearch_zoom(c, alphai1, alphai, &xa, phi_0, gphi_0, sigma, rho, t1, t2, t3, step);
      break;
    }
    xa += step;
    p01 = line_cost(c, xa);
    xa += -2.0 * step;
    p02 = line_cost(c, xa);
    gphi_i = (p01 - p02) / (2.0 * step);
    if (fabs(gphi_i) <= -sigma * gphi_0) {
      alphak = alphai;
      break;
    }
    if (gphi_i >= 0) {
      alphak = linesearch_zoom(c, alphai, alphai1, &xa, phi_0, gphi_0, sigma, rho, t1, t2, t3, step);
      break;
    }
    if (mu <= (2.0 * alphai - alphai1)) {
      alphai1 = alphai;
      alphai = mu;
    } else {
      p01 = 2.0 * alphai - alphai1;
      double hi = alphai + t1 * (alphai - alphai1);
      p02 = (mu < hi) ? mu : hi;
      alphai = cubic_interp(c, p01, p02, &xa, step);
    }
    phi_alphai1 = phi_alphai;
    ci++;
  }
  return alphak;
}

// What one run of the iteration did, for the tests (dirac_b200_lbfgs_trace); per iteration k:
// the accepted step, the cost evaluations of its line search, the history slot it wrote, ||g|| after
// the update and the iterate after it (m doubles).  Arrays of at least itmax entries.
struct LbfgsTrace {
  double *alphak;
  long long *ncost;
  int *slot;
  double *gnorm;
  double *iterates;
  int niter;
};

// p: m x 1 in/out (host).  robust != 0 -> Student's-t cost with nu.  res_held: pr->res already is
// the residual x - V(p), so the first gradient needs no predict.
// Iteration logic of lbfgs_fit_fullbatch (lbfgs.c:479-640); vectors on the device.
// Returns the number of accepted steps.  On return pr->res is the residual at the returned p: every
// accepted step leaves the line residual at the new iterate there, and a loop that ends without a
// step leaves the one it started from.
static int lbfgs_run(dirac_b200_problem *pr, double *p, int m, int itmax, int M, int robust,
                      double nu, bool res_held, LbfgsTrace *tr) {
  DevProblem &d = pr->d;
  LbfgsCtx ctx;
  ctx.pr = pr;
  ctx.robust = robust;
  ctx.nu = nu;
  ctx.m = m;
  ctx.ncost = ctx.ngrad = 0;
  if (tr) tr->niter = 0;
  if (M < 1) M = 1;
  if (M > db_lbfgs_direction_max_pairs()) {
    // the alpha_i of one recursion live in the shared memory of k_lbfgs_direction
    fprintf(stderr, "dirac_b200: LBFGS memory size %d exceeds the %d pairs the two-loop recursion "
                    "can hold; the LBFGS stage is skipped\n", M, db_lbfgs_direction_max_pairs());
    return 0;
  }
  // one allocation: xk | xk1 | gk | pk | s[M] | y[M] | rho[M]
  double *ws = (double *)db_malloc(sizeof(double) * ((size_t)m * (4 + 2 * (size_t)M) + M + 8));
  double *xk = ws, *xk1 = xk + m, *gk = xk1 + m, *pk = gk + m, *s = pk + m,
         *y = s + (size_t)m * M, *rho = y + (size_t)m * M;
  double *nrm_dev = d.scal + 24;
  double step, alphak;
  int ck, ci, cm;
  DB_CHECK(cudaMemcpyAsync(xk, p, sizeof(double) * m, cudaMemcpyHostToDevice, d.stream));
  grad_eval(&ctx, xk, gk, res_held ? RES_HELD : RES_PREDICT, 0.0);
  db_launch_lbfgs_nrm2(gk, m, nrm_dev, d.stream);
  db_count_launch(1);
  double gradnrm = sqrt(db_read_scalar(pr, 24));
  const double STOP = 1e-17;  // CLM_STOP_THRESH, Dirac_common.h:43
  if (gradnrm < STOP) {
    ck = itmax;
    step = 0.0;
  } else {
    ck = 0;
    double t = 1e-3 / gradnrm;
    if (t > 1e-6) t = 1e-6;
    step = (t > 1e-9) ? t : 1e-9;
  }
  cm = 0;
  ci = 0;
  while (ck < itmax && isnormal(gradnrm) && gradnrm > STOP) {
    const long long ncost0 = ctx.ncost;
    db_launch_lbfgs_direction(pk, gk, s, y, rho, m, ck < M ? ck : M, ci, d.stream);
    db_count_launch(1);
    line_setup(&ctx, xk, pk);
    alphak = linesearch(&ctx, 10.0, 0.1, 0.01, 9, 0.1, 0.5, step);
    if (!isnormal(alphak) || fabs(alphak) < 1e-12) break;  // CLM_EPSILON
    double *sk = s + (size_t)cm;
    double *yk = y + (size_t)cm;
    db_launch_lbfgs_step(xk, pk, gk, xk1, sk, yk, m, alphak, d.stream);
    grad_eval(&ctx, xk1, gk, RES_LINE, alphak);
    db_launch_lbfgs_update(gk, sk, yk, xk1, xk, m, rho + ci, nrm_dev, d.stream);
    db_count_launch(2);
    gradnrm = sqrt(db_read_scalar(pr, 24));
    if (tr) {
      tr->alphak[ck] = alphak;
      tr->ncost[ck] = ctx.ncost - ncost0;
      tr->slot[ck] = ci;
      tr->gnorm[ck] = gradnrm;
      DB_CHECK(cudaMemcpy(tr->iterates + (size_t)m * ck, xk, sizeof(double) * m,
                          cudaMemcpyDeviceToHost));
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
  DB_CHECK(cudaMemcpyAsync(p, xk, sizeof(double) * m, cudaMemcpyDeviceToHost, d.stream));
  db_stream_sync(d.stream);
  db_free(ws);
  return (int)ctx.ngrad - 1;  // one gradient at the start, one per accepted step
}

int db_lbfgs_fit(dirac_b200_problem *pr, double *p, int m, int itmax, int M, int robust,
                 double nu, bool res_held) {
  return lbfgs_run(pr, p, m, itmax, M, robust, nu, res_held, nullptr);
}

// test hook: the line model of the resident problem along pk from xk (host vectors of npar doubles),
// exactly as one LBFGS iteration of a single-GPU solve sets it up.  Out (host):
//   E       3 x 8R doubles, E0 | E1 | E2 in API layout (e(a) = E0 - a E1 - a^2 E2)
//   poly    the 5 coefficients of the Gaussian cost along the line (k_line_poly)
//   costs   [2 * nalpha]: k_line_eval at alphas[i], Gaussian (2i) and Student's-t with nu (2i + 1)
//   res     8R doubles: k_line_residual at alpha_res, API layout
//   shape   (TB, NST, WARPS) of the k_stream_all<1> launch that ran
extern "C" void dirac_b200_line_model(dirac_b200_problem *pr, const double *xk, const double *pk,
                                      int nalpha, const double *alphas, double nu,
                                      double alpha_res, double *E, double *poly, double *costs,
                                      double *res, int *shape) {
  DevProblem &d = pr->d;
  LbfgsCtx c;
  c.pr = pr; c.robust = 0; c.nu = nu; c.m = (int)d.npar; c.ncost = c.ngrad = 0;
  double *dx = (double *)db_malloc(sizeof(double) * 2 * d.npar);
  double *dp = dx + d.npar;
  DB_CHECK(cudaMemcpyAsync(dx, xk, sizeof(double) * d.npar, cudaMemcpyHostToDevice, d.stream));
  DB_CHECK(cudaMemcpyAsync(dp, pk, sizeof(double) * d.npar, cudaMemcpyHostToDevice, d.stream));
  db_line_setup_shape_reset();
  line_setup(&c, dx, dp);
  db_line_setup_shape(shape);
  for (int j = 0; j < 5; j++) poly[j] = c.poly[j];
  for (int i = 0; i < nalpha; i++)
    for (int mode = 1; mode <= 2; mode++) {
      db_launch_line_eval(pr->E0, pr->E1, pr->E2, 4 * d.R, alphas[i], mode,
                          mode == 2 ? 1.0 / nu : 0.0, pr->partials, d.scal, d.counters, d.stream);
      costs[2 * i + mode - 1] = db_read_scalar(pr, 0);
    }
  db_download_vis(pr, pr->E0, E);
  db_download_vis(pr, pr->E1, E + 8 * d.R);
  db_download_vis(pr, pr->E2, E + 16 * d.R);
  db_launch_line_residual(pr->E0, pr->E1, pr->E2, pr->res, 4 * d.R, alpha_res, d.stream);
  db_download_vis(pr, pr->res, res);
  DB_CHECK(cudaGetLastError());
  db_free(dx);
}

// test hook: the quartic of the line model left by the last dirac_b200_line_model, by the separate
// pass over E0, E1 and E2 (k_line_poly) that sharded runs take; poly: 5 doubles out (host)
extern "C" void dirac_b200_line_poly(dirac_b200_problem *pr, double *poly) {
  DevProblem &d = pr->d;
  db_launch_line_poly(pr->E0, pr->E1, pr->E2, 4 * d.R, pr->partials, d.scal + 16, d.counters,
                      d.stream);
  DB_CHECK(cudaMemcpyAsync(d.h_scal + 16, d.scal + 16, 5 * sizeof(double), cudaMemcpyDeviceToHost,
                           d.stream));
  db_stream_sync(d.stream);
  DB_CHECK(cudaGetLastError());
  for (int j = 0; j < 5; j++) poly[j] = d.h_scal[16 + j];
}

// test hook: the residual the resident problem holds (what the solvers left in pr->res), API layout
extern "C" void dirac_b200_residual(dirac_b200_problem *pr, double *out) {
  db_download_vis(pr, pr->res, out);
  DB_CHECK(cudaGetLastError());
}

// test hook: LBFGS on the resident problem's data from p (host, npar doubles, in/out) as bfgsfit runs
// it, with the trace of every iteration (LbfgsTrace; arrays of itmax entries, iterates itmax x npar).
// Returns the number of iterations, or -1 if the memory size M cannot be held.
extern "C" int dirac_b200_lbfgs_trace(dirac_b200_problem *pr, double *p, int itmax, int M, int robust,
                                      double nu, double *alphak, long long *ncost, int *slot,
                                      double *gnorm, double *iterates) {
  if ((M < 1 ? 1 : M) > db_lbfgs_direction_max_pairs()) return -1;
  LbfgsTrace tr;
  tr.alphak = alphak; tr.ncost = ncost; tr.slot = slot; tr.gnorm = gnorm; tr.iterates = iterates;
  lbfgs_run(pr, p, (int)pr->d.npar, itmax, M, robust, nu, false, &tr);
  return tr.niter;
}

// test hook: one two-loop recursion (k_lbfgs_direction) on host vectors exactly as db_lbfgs_fit
// launches it: g [m], s and y [Mmem][m], rho [Mmem]; pk [m] out.  Returns -1 without launching if
// npairs > Mmem, next >= Mmem or the kernel cannot hold npairs.
extern "C" int dirac_b200_lbfgs_direction(int m, int Mmem, int npairs, int next, const double *g,
                                          const double *s, const double *y, const double *rho,
                                          double *pk) {
  if (m < 1 || Mmem < 1 || npairs < 0 || npairs > Mmem || next < 0 || next >= Mmem ||
      npairs > db_lbfgs_direction_max_pairs())
    return -1;
  const size_t nv = (size_t)m * (2 + 2 * (size_t)Mmem) + Mmem;
  double *w = (double *)db_malloc(sizeof(double) * nv);
  double *dg = w, *dpk = dg + m, *ds = dpk + m, *dy = ds + (size_t)m * Mmem,
         *drho = dy + (size_t)m * Mmem;
  DB_CHECK(cudaMemcpy(dg, g, sizeof(double) * m, cudaMemcpyHostToDevice));
  DB_CHECK(cudaMemcpy(ds, s, sizeof(double) * m * Mmem, cudaMemcpyHostToDevice));
  DB_CHECK(cudaMemcpy(dy, y, sizeof(double) * m * Mmem, cudaMemcpyHostToDevice));
  DB_CHECK(cudaMemcpy(drho, rho, sizeof(double) * Mmem, cudaMemcpyHostToDevice));
  db_launch_lbfgs_direction(dpk, dg, ds, dy, drho, m, npairs, next, 0);
  DB_CHECK(cudaGetLastError());
  DB_CHECK(cudaMemcpy(pk, dpk, sizeof(double) * m, cudaMemcpyDeviceToHost));
  db_free(w);
  return 0;
}

// test hook: k_lbfgs_step then k_lbfgs_update as one iteration of db_lbfgs_fit runs them, with the
// pair written into slot ci of a rho[Mmem] array (rho_in host, copied).  Out (host): xk1, sk, yk [m],
// rho [Mmem], ||gk_new||^2 in gg[0], and xk after the update in xk_out [m].
extern "C" int dirac_b200_lbfgs_step_update(int m, double alpha, const double *xk, const double *pk,
                                            const double *gk_old, const double *gk_new, int Mmem,
                                            int ci, const double *rho_in, double *xk1, double *sk,
                                            double *yk, double *rho, double *gg, double *xk_out) {
  if (m < 1 || Mmem < 1 || ci < 0 || ci >= Mmem) return -1;
  const size_t nv = (size_t)m * 7 + Mmem + 1;
  double *w = (double *)db_malloc(sizeof(double) * nv);
  double *dx = w, *dp = dx + m, *dg0 = dp + m, *dg1 = dg0 + m, *dx1 = dg1 + m, *ds = dx1 + m,
         *dy = ds + m, *drho = dy + m, *dgg = drho + Mmem;
  DB_CHECK(cudaMemcpy(dx, xk, sizeof(double) * m, cudaMemcpyHostToDevice));
  DB_CHECK(cudaMemcpy(dp, pk, sizeof(double) * m, cudaMemcpyHostToDevice));
  DB_CHECK(cudaMemcpy(dg0, gk_old, sizeof(double) * m, cudaMemcpyHostToDevice));
  DB_CHECK(cudaMemcpy(dg1, gk_new, sizeof(double) * m, cudaMemcpyHostToDevice));
  DB_CHECK(cudaMemcpy(drho, rho_in, sizeof(double) * Mmem, cudaMemcpyHostToDevice));
  db_launch_lbfgs_step(dx, dp, dg0, dx1, ds, dy, m, alpha, 0);
  DB_CHECK(cudaGetLastError());
  DB_CHECK(cudaMemcpy(xk1, dx1, sizeof(double) * m, cudaMemcpyDeviceToHost));
  DB_CHECK(cudaMemcpy(sk, ds, sizeof(double) * m, cudaMemcpyDeviceToHost));
  db_launch_lbfgs_update(dg1, ds, dy, dx1, dx, m, drho + ci, dgg, 0);
  DB_CHECK(cudaGetLastError());
  DB_CHECK(cudaMemcpy(yk, dy, sizeof(double) * m, cudaMemcpyDeviceToHost));
  DB_CHECK(cudaMemcpy(rho, drho, sizeof(double) * Mmem, cudaMemcpyDeviceToHost));
  DB_CHECK(cudaMemcpy(gg, dgg, sizeof(double), cudaMemcpyDeviceToHost));
  DB_CHECK(cudaMemcpy(xk_out, dx, sizeof(double) * m, cudaMemcpyDeviceToHost));
  db_free(w);
  return 0;
}

// test hook: ||g||^2 of k_lbfgs_nrm2 for a host vector g [m]
extern "C" double dirac_b200_lbfgs_nrm2(int m, const double *g) {
  double *w = (double *)db_malloc(sizeof(double) * ((size_t)m + 1));
  double out;
  DB_CHECK(cudaMemcpy(w, g, sizeof(double) * m, cudaMemcpyHostToDevice));
  db_launch_lbfgs_nrm2(w, m, w + m, 0);
  DB_CHECK(cudaGetLastError());
  DB_CHECK(cudaMemcpy(&out, w + m, sizeof(double), cudaMemcpyDeviceToHost));
  db_free(w);
  return out;
}
