/* A plain C host of the stochastic-interval header alone: it compiles as C99 against
 * include/dirac_b200_stochastic.h, links against libdirac_b200, and calls the entry point with more
 * bands than channels, which the library refuses (-1) before it touches the device or any output. */
#include <stdio.h>
#include <string.h>

#include "dirac_b200_stochastic.h"

int main(void) {
  int (*fn)(double *, double *, double *, double *, int, int, int, int, baseline_t *, clus_source_t *,
            int, int, double *, int, double, double, double, int, int, int, int, double,
            persistent_data_t *, double *, int, double, int, double *, double *) =
      dirac_b200_stochastic_interval;
  double u[3] = {0}, v[3] = {0}, w[3] = {0}, xo[24] = {0}, freqs[1] = {150e6}, pfreq[2] = {7, 7};
  double r0[2] = {5, 5}, r1[2] = {5, 5};
  baseline_t barr[3];
  clus_source_t carr[1];
  persistent_data_t pt[2];
  memset(barr, 0, sizeof(barr));
  memset(carr, 0, sizeof(carr));
  memset(pt, 0, sizeof(pt));
  int rv = fn(u, v, w, xo, 3, 3, 1, 1, barr, carr, 1, 1, freqs, 1, 1e5, 0.0, 1e9, 2, 1, 4, 5, 2.0, pt,
              pfreq, -99999, 1e-9, 0, r0, r1);
  if (rv != -1 || pfreq[0] != 7 || r0[0] != 5 || r1[1] != 5) {
    printf("unexpected: rv=%d\n", rv);
    return 1;
  }
  printf("STOCHASTIC_CALLER OK\n");
  return 0;
}
