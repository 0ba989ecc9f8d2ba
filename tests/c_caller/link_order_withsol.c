/* TEST ONLY.  The linking recipe of INTEGRATION.md section 2 for the simulation-with-solutions branch
 * of the driver (fullbatch_mode.cpp:562-588), checked without a GPU: a host linked `-ldirac_b200`
 * BEFORE the reference's own library resolves the three simulation entry points to libdirac_b200.so
 * and the solution / ignore-list file readers to the reference library.
 * Prints "<symbol> <library file>" per line; no compute call is made. */
#define _GNU_SOURCE
#include <dlfcn.h>
#include <stdio.h>
#include <string.h>

#include "dirac_b200.h"

/* reference-only file readers (src/lib/Radio/Dirac_radio.h:110,116) */
extern int read_solutions(FILE *sfp, double *p, clus_source_t *carr, int N, int M);
extern int update_ignorelist(const char *ignfile, int *ignlist, int M, clus_source_t *carr);

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
  W(predict_visibilities_multifreq_withsol);
  W(predict_visibilities_multifreq_withsol_withbeam);
  W(predict_visibilities_withsol_withbeam_gpu);
  W(read_solutions);
  W(update_ignorelist);
  return bad;
}
