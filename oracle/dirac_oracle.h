/* TEST INFRASTRUCTURE ONLY — CPU restatement ("oracle") of the Dirac calibration hot path.
 *
 * Plain C99, single threaded, O(rows) (no dense Jacobian).  Each function cites the reference
 * file:line it follows (paths relative to /root/reference).  Pinned against the compiled reference
 * (oracle/_ref, built from the reference sources by oracle/Makefile) by tests/test_oracle_*.py and
 * against the committed golden vectors under tests/golden/ — the reference ships no known-answer
 * tests for this path (SURVEY.md 8c), so the compiled reference is the pin.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load this library.  The product (sagecal_b200/) never does.
 */
#ifndef DIRAC_ORACLE_H
#define DIRAC_ORACLE_H
#include <complex.h>

typedef struct {
  int N, Nbase, tilesz, M, Mt;
  const int *sta1, *sta2;        /* [Nbase*tilesz] */
  const unsigned char *flag;     /* [Nbase*tilesz] */
  const int *nchunk;             /* [M] */
  const int *chunk0;             /* [M] index of the first chunk of cluster k in chunk_off */
  const int *chunk_off;          /* [Mt] offset of each (cluster,chunk) 8N block in pp */
  const double complex *coh;     /* [row][M][4] */
} orc_problem;

void orc_generate_baselines(int Nbase, int tilesz, int N, int *sta1, int *sta2);
void orc_preset_flags_and_data(int n, const double *flag, unsigned char *bflag, double *x);

void orc_predict_full(const orc_problem *P, const double *pp, double *out);
void orc_predict_cluster(const orc_problem *P, int k, const double *pp, double *out);
void orc_predict_chunk(const orc_problem *P, int k, int t0, int ntiles, const double *pblk,
                       double *out);
double orc_cost(const orc_problem *P, const double *pp, const double *x, int robust, double nu);
void orc_grad(const orc_problem *P, const double *pp, const double *x, double *g, int robust,
              double nu);
double orc_normal_eq(const orc_problem *P, int k, int t0, int ntiles, const double *pblk,
                     const double *xd, const double *wt, double *JTJ, double *JTe);
void orc_normal_eq_os(const orc_problem *P, int k, int t0, int ntiles, const double *pblk,
                      const double *e_full, const double *wt, int l, double *JTJ, double *JTe);
int orc_lm_chunk(const orc_problem *P, int k, int t0, int ntiles, double *pblk, const double *xd,
                 int itmax, const double *opts, int linsolv, int os, double *info);
int orc_rlm_chunk(const orc_problem *P, int k, int t0, int ntiles, double *pblk, const double *xd,
                  int itmax, int linsolv, int os, double nulow, double nuhigh, double *robust_nu,
                  double *info);
double orc_update_w_and_nu(double nu0, double *w, const double *ed, int n, double nulow,
                           double nuhigh);
/* LM accept/reject decisions taken at rounding level since the last reset (see dirac_oracle.c) */
long orc_noise_decisions(int reset);
void orc_lbfgs(const orc_problem *P, double *pp, const double *x, int itmax, int M, int robust,
               double nu);
/* the two-loop recursion (lbfgs.c:33-111): pk = H g from M valid pairs, ii the slot written next */
void orc_mult_hessian(int m, double *pk, const double *gk, const double *s, const double *y,
                      const double *rho, int M, int ii);
/* what one LBFGS run did: per iteration k the accepted step, the cost evaluations of its line
 * search, the history slot written, ||g|| after the update and the iterate (m doubles); arrays of
 * itmax entries.  margin: the smallest margin of the line search's decisions over the run, in units
 * of the rounding noise of the costs behind them (see lb_decide) */
typedef struct {
  double *alphak;
  long long *ncost;
  int *slot;
  double *gnorm;
  double *iterates;
  int niter;
  double margin;
} orc_lbfgs_trace;
void orc_lbfgs_traced(const orc_problem *P, double *pp, const double *x, int itmax, int M,
                      int robust, double nu, orc_lbfgs_trace *tr);
/* margin (as in orc_lbfgs_trace) of the last LBFGS run, traced or not; HUGE_VAL before any */
double orc_lbfgs_last_margin(void);
/* RTR / RSD / NSD (solver_mode 4-6): per-row evaluators; the solver of one chunk is supplied by
 * oracle/rtr_harness.cpp (the control flow of rtr_algo.h on these evaluators) */
double orc_rtr_raw(const orc_problem *P, int k, int t0, int ntiles, const double *y,
                   const double *wt, const double *x, const double *eta, double *vec);
void orc_rtr_counts(const orc_problem *P, int t0, int ntiles, double *cnt);
double orc_rtr_weights(const orc_problem *P, int k, int t0, int ntiles, const double *y,
                       const double *x, double nu, double *wt);
typedef void (*orc_rtr_solver_fn)(const orc_problem *P, int k, int t0, int ntiles, const double *y,
                                  int kind, double *x, int itmax_a, int itmax_b, double nulow,
                                  double nuhigh, double *robust_nu, double *info);
void orc_set_rtr_solver(orc_rtr_solver_fn fn);
int orc_sagefit(const orc_problem *P, double *x, double *pp, int max_emiter, int max_iter,
                int max_lbfgs, int lbfgs_m, int linsolv, int solver_mode, double nulow,
                double nuhigh, double *mean_nu, double *res_0, double *res_1);
int orc_bfgsfit(const orc_problem *P, double *x, double *pp, int max_lbfgs, int lbfgs_m,
                int solver_mode, double mean_nu, double *res_0, double *res_1);

/* sky model in flat arrays: per cluster k sources [src0[k], src0[k+1]) */
typedef struct {
  int M;
  const int *src0;               /* [M+1] */
  const double *ll, *mm, *nn, *sI, *sQ, *sU, *sV;
  const unsigned char *stype;
  const double *gauss;           /* [nsrc][8]: eX,eY,eP,cxi,sxi,cphi,sphi,use_projection */
  const double *sI0, *sQ0, *sU0, *sV0, *f0, *spec_idx, *spec_idx1, *spec_idx2;
} orc_sky;

void orc_coherencies(const orc_sky *S, const double *u, const double *v, const double *w, int nrow,
                     double freq0, double fdelta, double uvmin, double uvmax, unsigned char *flag,
                     double complex *coh);
void orc_predict_multifreq(const orc_sky *S, const double *u, const double *v, const double *w,
                           int nrow, const double *freqs, int Nchan, double fdelta, int add_to_data,
                           double *x);
#endif
