/* A plain C host of the stochastic-interval entry points with station beams: it compiles as C99
 * against include/dirac_b200_stochastic.h alone, links against libdirac_b200, and calls both entry
 * points with doBeam = 7 (the lunar element beam), which the library refuses (-1) before it touches
 * the device or any output. */
#include <stdio.h>
#include <string.h>

#include "dirac_b200_stochastic.h"

int main(void) {
  double u[3] = {0}, v[3] = {0}, w[3] = {0}, xo[24] = {0}, freqs[1] = {150e6}, pfreq[2] = {7, 7};
  double lon[3] = {0.1, 0.1, 0.1}, lat[3] = {0.9, 0.9, 0.9}, t[1] = {2456789.3};
  double B[1] = {1}, Bi[1] = {1}, rhok[1] = {5}, Z[2] = {3, 3};
  double r00[1] = {5}, r01[1] = {5}, r0 = 9, r1 = 9;
  double ex[1] = {0}, *xx[3] = {ex, ex, ex};
  int Nelem[3] = {1, 1, 1}, fband[1] = {4};
  baseline_t barr[3];
  clus_source_t carr[1];
  persistent_data_t pt[1];
  memset(barr, 0, sizeof(barr));
  memset(carr, 0, sizeof(carr));
  memset(pt, 0, sizeof(pt));
  int rv = dirac_b200_stochastic_interval_withbeam(
      u, v, w, xo, 3, 3, 1, 1, barr, carr, 1, 1, freqs, 1, 1e5, 0.0, 1e9, STAT_SINGLE, 0.0, 1.0, 0.0,
      1.0, 150e6, lon, lat, t, Nelem, xx, xx, xx, NULL, 7, 1, 1, 4, 5, 2.0, pt, pfreq, -99999, 1e-9, 0,
      r00, r01);
  if (rv != -1 || pfreq[0] != 7 || r00[0] != 5 || r01[0] != 5) {
    printf("unexpected: interval rv=%d\n", rv);
    return 1;
  }
  rv = dirac_b200_stochastic_consensus_interval_withbeam(
      u, v, w, xo, 3, 3, 1, 1, barr, carr, 1, 1, freqs, 1, 1e5, 0.0, 1e9, STAT_SINGLE, 0.0, 1.0, 0.0,
      1.0, 150e6, lon, lat, t, Nelem, xx, xx, xx, NULL, 7, 1, 1, 4, 5, 2.0, pt, pfreq, -99999, 1e-9, 0,
      1, 1, B, Bi, rhok, Z, 0, r00, r01, &r0, &r1, fband);
  if (rv != -1 || pfreq[0] != 7 || Z[0] != 3 || r00[0] != 5 || r01[0] != 5 || r0 != 9 || r1 != 9 ||
      fband[0] != 4) {
    printf("unexpected: consensus interval rv=%d\n", rv);
    return 1;
  }
  printf("STOCHASTIC_BEAM_CALLER OK\n");
  return 0;
}
