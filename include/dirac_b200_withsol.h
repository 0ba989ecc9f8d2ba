/*
 * dirac_b200 — simulation with solutions (the driver's `-a 1|2|3 -p solutions.txt [-z ignore_file]`,
 * src/MS/fullbatch_mode.cpp:562-588): the three reference entry points of that branch, same names,
 * argument lists and meaning.  include/dirac_b200.h includes this header; it may also be included on
 * its own.  read_solutions and update_ignorelist read files on the host and stay with the
 * reference's library.
 */
#ifndef DIRAC_B200_WITHSOL_H
#define DIRAC_B200_WITHSOL_H

#include "dirac_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* replaces predict_visibilities_multifreq_withsol, src/lib/Radio/Dirac_radio.h:666
 * (residual.c:1342-1740).  Every cluster at a position k with ignorelist[k] == 0, whatever its id,
 * contributes J_p C_k(chan) J_q^H with the Jones of the row's hybrid chunk; flagged rows are
 * predicted like the others.  add_to_data: SIMUL_ONLY 1 writes the model alone, SIMUL_ADD 2 adds it
 * to x, SIMUL_SUB 3 subtracts it; any other value leaves x unchanged by the model, as the
 * reference's CPU builds do (its _gpu variant subtracts).  Then, as in calculate_residuals_multifreq,
 * every row of every channel is corrected once by the inverse Jones of the cluster whose id is ccid,
 * ignored or not. */
int predict_visibilities_multifreq_withsol(double *u, double *v, double *w, double *p, double *x,
                                           int *ignorelist, int N, int Nbase, int tilesz,
                                           baseline_t *barr, clus_source_t *carr, int M,
                                           double *freqs, int Nchan, double fdelta, double tdelta,
                                           double dec0, int Nt, int add_to_data, int ccid, double rho,
                                           int phase_only);

/* replace predict_visibilities_multifreq_withsol_withbeam, src/lib/Radio/Dirac_radio.h:490
 * (predict_withbeam.c:1452-1680), and predict_visibilities_withsol_withbeam_gpu, Dirac_radio.h:529
 * (predict_withbeam_cuda.c:2905-3130): predict_visibilities_multifreq_withsol with the station beams.
 * The correction by cluster ccid is applied once, after all clusters, as the reference's _gpu
 * variant does; its CPU variant corrects once per cluster not ignored (DESIGN.md section 7).  The
 * two entry points are the same call. */
int predict_visibilities_multifreq_withsol_withbeam(
    double *u, double *v, double *w, double *p, double *x, int *ignorelist, int N, int Nbase,
    int tilesz, baseline_t *barr, clus_source_t *carr, int M, double *freqs, int Nchan, double fdelta,
    double tdelta, double dec0, int bf_type, double b_ra0, double b_dec0, double ph_ra0,
    double ph_dec0, double ph_freq0, double *longitude, double *latitude, double *time_utc,
    int *Nelem, double **xx, double **yy, double **zz, elementcoeff *ecoeff, int doBeam, int Nt,
    int add_to_data, int ccid, double rho, int phase_only);
int predict_visibilities_withsol_withbeam_gpu(
    double *u, double *v, double *w, double *p, double *x, int *ignorelist, int N, int Nbase,
    int tilesz, baseline_t *barr, clus_source_t *carr, int M, double *freqs, int Nchan, double fdelta,
    double tdelta, double dec0, int bf_type, double b_ra0, double b_dec0, double ph_ra0,
    double ph_dec0, double ph_freq0, double *longitude, double *latitude, double *time_utc,
    int *Nelem, double **xx, double **yy, double **zz, elementcoeff *ecoeff, int doBeam, int Nt,
    int add_to_data, int ccid, double rho, int phase_only);

#ifdef __cplusplus
}
#endif
#endif
