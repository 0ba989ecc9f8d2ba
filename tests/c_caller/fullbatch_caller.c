/* A plain C host of the full-batch tile header alone: it compiles as C99 against
 * include/dirac_b200_fullbatch.h, links against libdirac_b200, and calls both entry points with no
 * channels, which the library refuses (-1) before it touches the device or any output. */
#include <stdio.h>
#include <string.h>

#include "dirac_b200_fullbatch.h"

int main(void) {
  double u[3] = {0}, v[3] = {0}, w[3] = {0}, x[24] = {0}, xo[24] = {0}, freqs[1] = {150e6};
  double pp[24] = {7}, nu = 5, r0 = 5, r1 = 5, r00[1] = {5}, r01[1] = {5};
  double lon[3] = {0}, lat[3] = {0}, t[1] = {2456789.5};
  baseline_t barr[3];
  clus_source_t carr[1];
  memset(barr, 0, sizeof(barr));
  memset(carr, 0, sizeof(carr));
  int rv = dirac_b200_fullbatch_tile(u, v, w, x, xo, 3, 3, 1, barr, carr, 1, 1, 150e6, 1e5, freqs, 0,
                                     0.0, 1e9, pp, 3, 2, 10, 7, 0, 1, 2.0, 30.0, 0, 0, -99999, 1e-9, 0,
                                     0, 1, NULL, NULL, &nu, &r0, &r1, r00, r01);
  int rb = dirac_b200_fullbatch_tile_withbeam(
      u, v, w, x, xo, 3, 3, 1, barr, carr, 1, 1, 150e6, 1e5, freqs, 0, 0.0, 1e9, STAT_SINGLE, 0.0, 0.0,
      0.0, 0.0, 150e6, lon, lat, t, NULL, NULL, NULL, NULL, NULL, DOBEAM_NONE, pp, 3, 2, 10, 7, 0, 1,
      2.0, 30.0, 0, 0, -99999, 1e-9, 0, 0, 1, NULL, NULL, &nu, &r0, &r1, r00, r01);
  if (rv != -1 || rb != -1 || pp[0] != 7 || nu != 5 || r0 != 5 || r1 != 5 || r00[0] != 5) {
    printf("unexpected: rv=%d rb=%d\n", rv, rb);
    return 1;
  }
  printf("FULLBATCH_CALLER OK\n");
  return 0;
}
