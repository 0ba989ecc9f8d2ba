// The stochastic closing stage of sagefit (minibatch::lbfgs_fit_robust_wrapper_minibatch, the code
// the library runs on the host) with the cost and gradient of a row window supplied by the caller
// through function pointers, so that tests/test_oracle_minibatch_window.py can drive it on the CPU
// with the compiled reference's evaluators.  Built by that test into a temporary directory.
#include "../../sagecal_b200/csrc/minibatch_algo.h"

typedef double (*window_cost_fn)(const double *p, long long row0, long long nrows);
typedef void (*window_grad_fn)(const double *p, double *g, long long row0, long long nrows);

namespace {
struct CallbackWindow {
  window_cost_fn c;
  window_grad_fn g;
  int m;
  long long r0, nr;
  void set_window(long long row0, long long nrows) {
    r0 = row0;
    nr = nrows;
  }
  double cost(const double *p) { return nr > 0 ? c(p, r0, nr) : 0.0; }
  void grad(const double *p, double *out) {
    if (nr > 0) {
      g(p, out, r0, nr);
    } else {
      for (int i = 0; i < m; i++) out[i] = 0.0;
    }
  }
};
}  // namespace

extern "C" void window_fit(window_cost_fn c, window_grad_fn g, double *p, int m, long long nrows,
                           int itmax, int M) {
  CallbackWindow F;
  F.c = c;
  F.g = g;
  F.m = m;
  F.r0 = 0;
  F.nr = nrows;
  minibatch::lbfgs_fit_robust_wrapper_minibatch(F, p, m, nrows, itmax, M);
}

extern "C" void window_table(long long n, int nbatch, long long *off, long long *len) {
  for (int i = 0; i < nbatch; i++) minibatch::batch_window(n, nbatch, i, off + i, len + i);
}
