/*
 * dirac_b200 — the per-channel refinement of a solve interval (driver option `-b 1`, Data::doChan,
 * src/MS/fullbatch_mode.cpp:453-499): the reference's single-channel residual with its name, argument
 * list and meaning, and the whole channel loop of an interval on one resident problem.
 * include/dirac_b200.h includes this header; it may also be included on its own.
 */
#ifndef DIRAC_B200_CHANNELS_H
#define DIRAC_B200_CHANNELS_H

#include "dirac_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* replaces calculate_residuals, src/lib/Radio/Dirac_radio.h:639 (residual.c:314-674), called at
 * fullbatch_mode.cpp:494.  x[row][8] -= sum over the clusters with id >= 0 of J_p C_k J_q^H, C_k
 * re-predicted from the sources at freq0 (smearing width fdelta, spectral-index fluxes), every row
 * whatever its flag, the Jones of a row from its hybrid chunk; then, if a cluster has id == ccid (the
 * last such one), every row is corrected by that cluster's (J + rho I)^-1.  tdelta, dec0 and Nt are
 * accepted and unused.  It is calculate_residuals_multifreq with one channel and phase_only == 0. */
int calculate_residuals(double *u, double *v, double *w, double *p, double *x, int N, int Nbase,
                        int tilesz, baseline_t *barr, clus_source_t *carr, int M, double freq0,
                        double fdelta, double tdelta, double dec0, int Nt, int ccid, double rho);

/* replaces the loop of fullbatch_mode.cpp:464-497 (precalculate_coherencies, bfgsfit_visibilities,
 * calculate_residuals per channel) for one interval.  The sky model, u, v, w, the station pairs and the
 * flags go to the device once; per channel only xo[ci] goes up and its residual comes down, and the
 * coherencies of a channel never leave the device.
 *   xo      [Nchan][Nbase*tilesz][8], data in, residual out (as calculate_residuals leaves it)
 *   barr    in/out: rows unflagged on entry whose uv distance in wavelengths at a channel's frequency
 *           lies outside [uvmin, uvmax] get flag 2 from that channel on, as precalculate_coherencies
 *           (predict.c:489-495) leaves them when it is handed the same barr channel after channel
 *   p       [8 N Mt] in: the Jones every channel starts from; out: the last channel's solution (:497)
 *   res_00, res_01   [Nchan] cost before and after the fit of each channel
 *   pfreq   [Nchan][8 N Mt] every channel's solution, or NULL
 * max_lbfgs, lbfgs_m, solver_mode, mean_nu as bfgsfit_visibilities takes them.  Returns 0. */
int dirac_b200_bfgsfit_channels(double *u, double *v, double *w, double *xo, int N, int Nbase,
                                int tilesz, baseline_t *barr, clus_source_t *carr, int M, int Mt,
                                double *freqs, int Nchan, double deltafch, double uvmin, double uvmax,
                                double *p, int max_lbfgs, int lbfgs_m, int solver_mode, double mean_nu,
                                int ccid, double rho, double *res_00, double *res_01, double *pfreq);

/* sky models uploaded and bytes of coherencies copied between host and device since the last reset */
void dirac_b200_transfer_stats(unsigned long long *sky_uploads, unsigned long long *coh_host_bytes,
                               int reset);

#ifdef __cplusplus
}
#endif
#endif
