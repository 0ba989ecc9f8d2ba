/* A plain C host of the federated header alone: it compiles as C99 against
 * include/dirac_b200_federated.h, links against libdirac_b200, and makes calls the library refuses
 * (-1) before it touches the device or any output: no solutions, a negative round count, a negative
 * ADMM iteration. */
#include <stdio.h>
#include <string.h>

#include "dirac_b200_federated.h"

int main(void) {
  int (*avg)(int, int, int, double *, int, int, int) = calculate_manifold_average_projectback;
  double Y[16];
  for (int i = 0; i < 16; i++) Y[i] = 7.0;
  int bad = 0;
  bad |= avg(1, 2, 0, Y, 10, 0, 1) != -1;
  bad |= avg(1, 2, 1, Y, -1, 0, 1) != -1;
  bad |= avg(0, 2, 1, Y, 10, 0, 1) != -1;
  bad |= dirac_b200_manifold_projectback_dev(1, 0, 1, Y, 10, NULL, NULL) != -1;
  for (int i = 0; i < 16; i++) bad |= Y[i] != 7.0;
  double r[2] = {1.0, 1.0}, J[8] = {0}, B[1] = {1.0}, Bi[1] = {1.0}, rho[1] = {1.0}, a[1] = {1.0};
  double Zavg[8] = {0}, X[8] = {0}, Yb[8] = {0}, Z[8], r0 = 5.0, r1 = 5.0;
  int fband[1] = {9};
  for (int i = 0; i < 8; i++) Z[i] = 3.0;
  bad |= dirac_b200_federated_bands_update(1, 1, 1, 1, -1, r, r, J, B, Bi, rho, a, Zavg, X, &r0, &r1,
                                           Yb, Z, fband) != -1;
  bad |= r0 != 5.0 || r1 != 5.0 || fband[0] != 9 || Z[0] != 3.0;
  /* no ADMM iterations: refused before the device is touched */
  double u[3] = {0}, v[3] = {0}, w[3] = {0}, xo[24] = {0}, freqs[1] = {150e6}, pfreq[8] = {7, 7};
  double q00[1] = {5}, q01[1] = {5};
  baseline_t barr[3];
  clus_source_t carr[1];
  persistent_data_t pt[1];
  memset(barr, 0, sizeof(barr));
  memset(carr, 0, sizeof(carr));
  memset(pt, 0, sizeof(pt));
  bad |= dirac_b200_stochastic_federated_interval(u, v, w, xo, 3, 3, 1, 1, barr, carr, 1, 1, freqs, 1,
                                                  1e5, 0.0, 1e9, 1, 1, 4, 5, 2.0, pt, pfreq, -99999,
                                                  1e-9, 0, 0, 1, B, Bi, rho, a, Z, 0, 0, 0, 1, NULL,
                                                  NULL, q00, q01, &r0, &r1, fband) != -1;
  bad |= pfreq[0] != 7 || q00[0] != 5 || r0 != 5.0 || fband[0] != 9;
  if (bad) {
    printf("unexpected\n");
    return 1;
  }
  printf("FEDERATED_CALLER OK\n");
  return 0;
}
