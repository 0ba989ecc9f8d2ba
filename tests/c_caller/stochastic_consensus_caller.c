/* A plain C host of the consensus stochastic-interval entry point: it compiles as C99 against
 * include/dirac_b200_stochastic.h alone, links against libdirac_b200, and calls the entry point with no
 * ADMM iterations and with no polynomial terms, which the library refuses (-1) before it touches the
 * device or any output.  It also takes the address of the host-only ADMM step. */
#include <stdio.h>
#include <string.h>

#include "dirac_b200_stochastic.h"

int main(void) {
  int (*fn)(double *, double *, double *, double *, int, int, int, int, baseline_t *, clus_source_t *,
            int, int, double *, int, double, double, double, int, int, int, int, double,
            persistent_data_t *, double *, int, double, int, int, int, double *, double *, double *,
            double *, int, double *, double *, double *, double *, int *) =
      dirac_b200_stochastic_consensus_interval;
  int (*step)(int, int, int, int, const double *, const double *, const double *, const double *,
              const double *, const double *, double *, double *, double *, double *, int *) =
      dirac_b200_consensus_bands_update;
  double u[3] = {0}, v[3] = {0}, w[3] = {0}, xo[24] = {0}, freqs[1] = {150e6}, pfreq[2] = {7, 7};
  double B[2] = {1, 1}, Bi[1] = {1}, rhok[1] = {5}, Z[2] = {3, 3};
  double r00[2] = {5, 5}, r01[2] = {5, 5}, r0 = 9, r1 = 9;
  int fband[1] = {4};
  baseline_t barr[3];
  clus_source_t carr[1];
  persistent_data_t pt[1];
  memset(barr, 0, sizeof(barr));
  memset(carr, 0, sizeof(carr));
  memset(pt, 0, sizeof(pt));
  const int cases[2][2] = {{0, 1}, {1, 0}};  /* (nadmm, Npoly) */
  for (int k = 0; k < 2; k++) {
    int rv = fn(u, v, w, xo, 3, 3, 1, 1, barr, carr, 1, 1, freqs, 1, 1e5, 0.0, 1e9, 1, 1, 4, 5, 2.0,
                pt, pfreq, -99999, 1e-9, 0, cases[k][0], cases[k][1], B, Bi, rhok, Z, 0, r00, r01, &r0,
                &r1, fband);
    if (rv != -1 || pfreq[0] != 7 || Z[0] != 3 || r00[0] != 5 || r01[1] != 5 || r0 != 9 || r1 != 9 ||
        fband[0] != 4) {
      printf("unexpected: case %d rv=%d\n", k, rv);
      return 1;
    }
  }
  if (step == 0) return 1;
  printf("STOCHASTIC_CONSENSUS_CALLER OK\n");
  return 0;
}
