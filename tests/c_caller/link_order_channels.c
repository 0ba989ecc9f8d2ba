/* TEST ONLY.  The linking recipe of INTEGRATION.md section 2 for the per-channel branch of the driver
 * (-b 1, fullbatch_mode.cpp:453-499), checked without a GPU: a host linked `-ldirac_b200` BEFORE the
 * reference's own library resolves the three calls of the channel loop to libdirac_b200.so.
 * Prints "<symbol> <library file>" per line; no compute call is made. */
#define _GNU_SOURCE
#include <dlfcn.h>
#include <stdio.h>
#include <string.h>

#include "dirac_b200.h"

/* a reference-only name, to show that the stand-in library is linked at all (Dirac_radio.h:110) */
extern int read_solutions(FILE *sfp, double *p, clus_source_t *carr, int N, int M);

static int where(const char *name, void *fn) {
  Dl_info info;
  if (!dladdr(fn, &info) || !info.dli_fname) {
    printf("%s ?\n", name);
    return 1;
  }
  const char *base = strrchr(info.dli_fname, '/');
  printf("%s %s\n", name, base ? base + 1 : info.dli_fname);
  return 0;
}

#define W(f) bad |= where(#f, (void *)f)
int main(void) {
  int bad = 0;
  W(precalculate_coherencies);
  W(bfgsfit_visibilities);
  W(bfgsfit_visibilities_gpu);
  W(calculate_residuals);
  W(dirac_b200_bfgsfit_channels);
  W(read_solutions);
  return bad;
}
