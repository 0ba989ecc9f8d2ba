/*
 * dirac_b200 — stochastic calibration of a whole solution interval (`sagecal -N <epochs>
 * -M <minibatches> -w <bands>`, src/MS/minibatch_mode.cpp:364-509, without beams): the driver's loop
 * over epochs, minibatches and bands of channels in one call, with every coherency predicted straight
 * into device memory and kept there for the whole interval.
 * include/dirac_b200.h includes this header; it may also be included on its own.
 */
#ifndef DIRAC_B200_STOCHASTIC_H
#define DIRAC_B200_STOCHASTIC_H

#include "dirac_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* replaces minibatch_mode.cpp:368-506 for one interval when no beam is used (doBeam == 0):
 * precalculate_coherencies_multifreq per minibatch in the first epoch, bfgsfit_minibatch_visibilities
 * per (epoch, minibatch, band), then calculate_residuals_multifreq per (minibatch, band).  The sky
 * model, u, v, w, the station pairs, the chunk tables, the flags and the data go to the device once;
 * the coherencies of every (minibatch, channel) are predicted into device memory and never cross
 * PCIe, and the residuals come back once at the end.
 *   u, v, w      [minibatches][Nbase*tmb], in seconds (already scaled by 1/c, as the driver does)
 *   xo           [minibatches][Nchan][Nbase*tmb][8]: data in (as preset_flags_and_data left them),
 *                residual out (as calculate_residuals_multifreq leaves it)
 *   N, Nbase, tmb     stations, baselines N(N-1)/2, timeslots of one minibatch
 *   minibatches  minibatches of the interval
 *   barr         [minibatches][Nbase*tmb], rows in the canonical order of generate_baselines, flags as
 *                preset_flags_and_data left them; input only
 *   carr, M, Mt  the sky model: M clusters, Mt = sum of their hybrid chunks
 *   freqs        [Nchan] channel frequencies
 *   deltaf       the bandwidth of all Nchan channels: the smearing width of a channel is deltaf / Nchan
 *   uvmin, uvmax the uv cut in wavelengths, applied in the first epoch only: uvmin at freqs[0], uvmax at
 *                freqs[Nchan-1] (precalculate_coherencies_multifreq's rule)
 *   nsolbw       bands of channels, 1 <= nsolbw <= Nchan: band b holds ceil(Nchan/nsolbw) channels from
 *                channel b ceil(Nchan/nsolbw) on, the last band the rest, which may be none
 *                (minibatch_mode.cpp:92-116)
 *   nepochs      passes over the minibatches
 *   max_lbfgs, lbfgs_m, robust_nu   as bfgsfit_minibatch_visibilities takes them
 *   pt           [nsolbw] in/out: each band's persistent LBFGS state, as lbfgs_persist_init made them;
 *                an array of the persistent_data_t this library declares (dirac_b200.h)
 *   pfreq        [nsolbw][8 N Mt] in: each band's start Jones; out: its solution
 *   ccid, rho, phase_only   the correction of the residual, as calculate_residuals_multifreq takes it
 *   res_00, res_01          [nepochs][minibatches][nsolbw] out: every fit's cost before and after, over
 *                the band's 8 Nbase tmb nc data (a band of no channels: 0 x 1/0, NaN, as the reference)
 * Device memory: the interval's coherencies take minibatches x Nchan x M x Nbase x tmb x 64 bytes
 * (62 stations, 64 clusters, 4 minibatches of 30 timeslots, 8 channels: 7.4 GB), the data twice
 * minibatches x Nchan x Nbase x tmb x 64 bytes.  A failed allocation prints a message and exits.
 * What the driver does between intervals (its running averages of the costs, the band and global
 * resets, minibatch_mode.cpp:533-558) stays with the caller.
 * Returns 0, or -1 with a message on stderr and no output touched when nsolbw is outside [1, Nchan]. */
int dirac_b200_stochastic_interval(double *u, double *v, double *w, double *xo, int N, int Nbase,
                                   int tmb, int minibatches, baseline_t *barr, clus_source_t *carr,
                                   int M, int Mt, double *freqs, int Nchan, double deltaf,
                                   double uvmin, double uvmax, int nsolbw, int nepochs, int max_lbfgs,
                                   int lbfgs_m, double robust_nu, persistent_data_t *pt, double *pfreq,
                                   int ccid, double rho, int phase_only, double *res_00,
                                   double *res_01);

#ifdef __cplusplus
}
#endif
#endif
