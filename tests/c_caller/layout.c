/* TEST ONLY.  Prints size, field offsets and enumerated constants of every struct / macro the C ABI
 * shares with the reference; compiled against include/dirac_b200.h by
 * tests/test_c_caller.py::test_struct_layouts_equal_the_reference_headers, and against the reference
 * headers (-DUSE_REF) by tests/golden/make_golden_headers.py, whose output the test compares with. */
#include <stddef.h>
#include <stdio.h>
#ifdef USE_REF
#include <Dirac.h>
#include <Dirac_radio.h>
#else
#include "dirac_b200.h"
#endif
#define S(t) printf("sizeof " #t " %zu\n", sizeof(t))
#define O(t, f) printf("offsetof " #t "." #f " %zu\n", offsetof(t, f))
int main(void) {
  S(baseline_t); O(baseline_t, sta1); O(baseline_t, sta2); O(baseline_t, flag);
  S(clus_source_t); O(clus_source_t, N); O(clus_source_t, id); O(clus_source_t, ll); O(clus_source_t, mm);
  O(clus_source_t, nn); O(clus_source_t, sI); O(clus_source_t, sQ); O(clus_source_t, sU); O(clus_source_t, sV);
  O(clus_source_t, ra); O(clus_source_t, dec); O(clus_source_t, stype); O(clus_source_t, ex);
  O(clus_source_t, nchunk); O(clus_source_t, p); O(clus_source_t, sI0); O(clus_source_t, sQ0);
  O(clus_source_t, sU0); O(clus_source_t, sV0); O(clus_source_t, f0); O(clus_source_t, spec_idx);
  O(clus_source_t, spec_idx1); O(clus_source_t, spec_idx2);
  S(exinfo_gaussian); O(exinfo_gaussian, eX); O(exinfo_gaussian, eY); O(exinfo_gaussian, eP);
  O(exinfo_gaussian, cxi); O(exinfo_gaussian, sxi); O(exinfo_gaussian, cphi); O(exinfo_gaussian, sphi);
  O(exinfo_gaussian, use_projection);
  S(exinfo_disk); O(exinfo_disk, eX); O(exinfo_disk, cxi); O(exinfo_disk, sphi); O(exinfo_disk, use_projection);
  S(exinfo_shapelet); O(exinfo_shapelet, n0); O(exinfo_shapelet, beta); O(exinfo_shapelet, modes);
  O(exinfo_shapelet, eX); O(exinfo_shapelet, eY); O(exinfo_shapelet, eP); O(exinfo_shapelet, cxi);
  O(exinfo_shapelet, sxi); O(exinfo_shapelet, cphi); O(exinfo_shapelet, sphi); O(exinfo_shapelet, use_projection);
  S(elementcoeff); O(elementcoeff, M); O(elementcoeff, Nmodes); O(elementcoeff, Nf); O(elementcoeff, beta);
  O(elementcoeff, pattern_phi); O(elementcoeff, pattern_theta); O(elementcoeff, preamble);
  O(persistent_data_t, y); O(persistent_data_t, s); O(persistent_data_t, rho); O(persistent_data_t, nfilled);
  O(persistent_data_t, vacant); O(persistent_data_t, lbfgs_m); O(persistent_data_t, m); O(persistent_data_t, Nt);
  printf("const STYPE %d %d %d %d %d\n", STYPE_POINT, STYPE_GAUSSIAN, STYPE_DISK, STYPE_RING, STYPE_SHAPELET);
  printf("const DOBEAM %d %d %d %d %d %d %d\n", DOBEAM_NONE, DOBEAM_ARRAY, DOBEAM_FULL, DOBEAM_ELEMENT, DOBEAM_ARRAY_WB, DOBEAM_FULL_WB, DOBEAM_ELEMENT_WB);
  printf("const STAT %d %d %d\n", STAT_NONE, STAT_SINGLE, STAT_TILE);
  printf("const SM %d %d %d %d %d %d %d\n", SM_LM_LBFGS, SM_OSLM_LBFGS, SM_OSLM_OSRLM_RLBFGS, SM_RLM_RLBFGS, SM_RTR_OSLM_LBFGS, SM_RTR_OSRLM_RLBFGS, SM_NSD_RLBFGS);
  return 0;
}
