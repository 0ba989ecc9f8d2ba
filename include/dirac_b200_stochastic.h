/*
 * dirac_b200 — stochastic calibration of a whole solution interval (`sagecal -N <epochs>
 * -M <minibatches> -w <bands>`, src/MS/minibatch_mode.cpp:364-509): the driver's loop over epochs,
 * minibatches and bands of channels in one call, with every coherency predicted straight into device
 * memory and kept there for the whole interval; and the same loop with spectral consensus over the
 * bands (`-A <nadmm>`, src/MS/minibatch_consensus_mode.cpp:450-672).  Each comes without station
 * beams and, as a _withbeam variant, with them (`-B <doBeam>`).
 * include/dirac_b200.h includes this header; it may also be included on its own.
 */
#ifndef DIRAC_B200_STOCHASTIC_H
#define DIRAC_B200_STOCHASTIC_H

#include "dirac_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* replaces minibatch_mode.cpp:368-506 for one interval when no beam is used (doBeam == 0; with beams
 * see dirac_b200_stochastic_interval_withbeam):
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

/* replaces minibatch_consensus_mode.cpp:453-672 for one interval when no beam is used (with beams:
 * dirac_b200_stochastic_consensus_interval_withbeam) (`sagecal -N
 * <epochs> -M <minibatches> -w <bands> -A <nadmm>`, which main.cpp runs when nadmm > 1 and nsolbw > 1):
 * the loop of dirac_b200_stochastic_interval inside nadmm ADMM iterations that tie the bands' Jones to
 * a polynomial in frequency.  Per minibatch, every band b is fitted as bfgsfit_minibatch_consensus
 * fits it, with y = Y_b, z = B_b Z and rho = rhok_b, and then dirac_b200_consensus_bands_update takes
 * the ADMM step.  Y is the call's own and starts from zero.  The coherencies are predicted once, in
 * (admm 0, epoch 0), and only that pass uses the uv cut.  robust_nu is fixed for the whole interval.
 * The arguments up to phase_only are those of dirac_b200_stochastic_interval; then:
 *   nadmm        ADMM iterations, >= 1
 *   Npoly        polynomial terms, >= 1
 *   B            [nsolbw][Npoly] the basis at the bands' mean frequencies (dirac_b200_consensus_basis)
 *   Bi           [Mt][Npoly][Npoly] (dirac_b200_consensus_prod_inverse of B and rhok)
 *   rhok         [nsolbw][Mt] the ADMM weight of every band and chunk
 *   Z            [Mt][Npoly][8N] in/out: the global polynomial solution; the driver keeps it from one
 *                interval to the next
 *   use_global   != 0: every band's solution becomes B_b Z after the loop, and the residuals use it
 *   res_00, res_01   [nadmm][nepochs][minibatches][nsolbw] out: every fit's cost before and after
 *   res_0, res_1 out: the driver's running averages after the loop (see dirac_b200_consensus_bands_update)
 *   fband        [nsolbw] out: the bad-band flags of the last minibatch
 * What the driver does between intervals (resetting flagged bands and all bands,
 * minibatch_consensus_mode.cpp:696-721) stays with the caller, which needs res_1 and fband for it.
 * Returns 0, or -1 with a message on stderr and no output touched when nsolbw is outside [1, Nchan],
 * nadmm < 1 or Npoly < 1. */
int dirac_b200_stochastic_consensus_interval(
    double *u, double *v, double *w, double *xo, int N, int Nbase, int tmb, int minibatches,
    baseline_t *barr, clus_source_t *carr, int M, int Mt, double *freqs, int Nchan, double deltaf,
    double uvmin, double uvmax, int nsolbw, int nepochs, int max_lbfgs, int lbfgs_m, double robust_nu,
    persistent_data_t *pt, double *pfreq, int ccid, double rho, int phase_only, int nadmm, int Npoly,
    double *B, double *Bi, double *rhok, double *Z, int use_global, double *res_00, double *res_01,
    double *res_0, double *res_1, int *fband);

/* the ADMM step of one minibatch of the consensus loop (minibatch_consensus_mode.cpp:540-601), host
 * arithmetic, no device needed; for a host that keeps its own loop of bfgsfit_minibatch_consensus
 * calls.  Decision for decision as the driver:
 *   res_0 = (res_0 + sum_b res_00[b]) / nsolbw, res_1 likewise: a running mixture, not a mean;
 *   fband[b] = 1 when resband[b] > 1.5 res_1, resband[b] = res_01[b] if res_00[b] > 0 and
 *   res_01[b] > 0, else 1e12 (a NaN res_1 flags no band);
 *   good bands: Y_b += rhok_b J_b;  z[p] = sum_b B_b[p] Y_b over band 0 whatever fband[0] says and the
 *   good bands from 1 on;  Z = update_global_z_multi(z, Bi);  good bands: Y_b -= rhok_b B_b Z.
 *   res_00, res_01   [nsolbw] the costs of this minibatch's fits
 *   pfreq        [nsolbw][8 N Mt] the bands' Jones J_b
 *   B, Bi, rhok  as dirac_b200_stochastic_consensus_interval takes them
 *   res_0, res_1 in/out;  Y [nsolbw][8 N Mt] in/out;  Z [Mt][Npoly][8N] in/out;  fband [nsolbw] out
 * Returns 0, or -1 with a message on stderr and nothing touched when N, Mt, nsolbw or Npoly is < 1. */
int dirac_b200_consensus_bands_update(int N, int Mt, int nsolbw, int Npoly, const double *res_00,
                                      const double *res_01, const double *pfreq, const double *B,
                                      const double *Bi, const double *rhok, double *res_0,
                                      double *res_1, double *Y, double *Z, int *fband);

/* dirac_b200_stochastic_interval with station beams (`sagecal -N -M -w -B <doBeam>`): replaces
 * minibatch_mode.cpp:368-506 for one interval with the driver's beam branches
 * precalculate_coherencies_multifreq_withbeam (:403-427) and calculate_residuals_multifreq_withbeam
 * (:485-500).  The arguments are those of dirac_b200_stochastic_interval with the beam arguments of
 * precalculate_coherencies_multifreq_withbeam inserted after uvmax:
 *   bf_type      STAT_SINGLE or STAT_TILE (array modes)
 *   b_ra0, b_dec0, ph_ra0, ph_dec0   tile beam centre and phase centre (rad), already precessed
 *   ph_freq0     the beam-former's reference frequency; the uv cut is taken at it
 *   longitude, latitude   [N] station positions (rad)
 *   time_utc     [minibatches][tmb] the timeslots' JD, as loadDataMinibatch fills them per minibatch
 *   Nelem, xx, yy, zz     per station the elements (STAT_TILE: the 16 dipoles of a tile, then the
 *                tiles), as readAuxData leaves them
 *   ecoeff       element modes: set_elementcoeffs for the narrow-band modes, set_elementcoeffs_wb over
 *                all Nchan channels for the wide-band ones
 *   doBeam       DOBEAM_NONE (0): exactly dirac_b200_stochastic_interval; 1..6 the array, full and
 *                element beams, narrow- and wide-band
 * The sky (carr ra / dec, the phase and beam centres) comes in precessed: Data::precess_source_locations
 * (minibatch_mode.cpp:394-397) stays with the caller.  Channel c of the first pass is predicted with
 * its own beam tables and, for wide-band element beams, coefficient set c; a row is cut in the first
 * pass when its uv distance at ph_freq0 lies outside [uvmin, uvmax].  The residual of band b is
 * corrected as calculate_residuals_multifreq_withbeam corrects it for &freqs[first channel of b]: its
 * tables use coefficient sets 0 .. nc-1, the band's own channel numbers.
 * Device memory: besides that of dirac_b200_stochastic_interval, one set of beam tables, rebuilt for
 * every (minibatch, channel) and (minibatch, band): tmb x ceil(Nchan/nsolbw) x S x N x 72 bytes at most
 * (S sources over all clusters; 8 bytes of array factor and 64 of E-Jones per entry, the array modes
 * only the first, the element modes only the second), and the element positions and coefficients.
 * Returns 0, or -1 with a message on stderr and no output touched, before any device work, when
 * nsolbw is outside [1, Nchan], doBeam is outside 0..6 (the lunar element beam needs CSPICE), an
 * array mode has a bf_type other than STAT_SINGLE / STAT_TILE or no Nelem / xx / yy / zz, an element
 * mode has no coefficient tables or a wide-band one fewer than Nchan sets, or a beam has no
 * longitude, latitude or time_utc. */
int dirac_b200_stochastic_interval_withbeam(
    double *u, double *v, double *w, double *xo, int N, int Nbase, int tmb, int minibatches,
    baseline_t *barr, clus_source_t *carr, int M, int Mt, double *freqs, int Nchan, double deltaf,
    double uvmin, double uvmax, int bf_type, double b_ra0, double b_dec0, double ph_ra0,
    double ph_dec0, double ph_freq0, double *longitude, double *latitude, double *time_utc,
    int *Nelem, double **xx, double **yy, double **zz, elementcoeff *ecoeff, int doBeam, int nsolbw,
    int nepochs, int max_lbfgs, int lbfgs_m, double robust_nu, persistent_data_t *pt, double *pfreq,
    int ccid, double rho, int phase_only, double *res_00, double *res_01);

/* dirac_b200_stochastic_consensus_interval with station beams (`-A <nadmm> -B <doBeam>`,
 * minibatch_consensus_mode.cpp:493-506,648-663): the beam arguments inserted after uvmax as in
 * dirac_b200_stochastic_interval_withbeam, with the same meaning, memory and refusals (and those of
 * the consensus call).  The beam's uv cut holds in (admm 0, epoch 0) only. */
int dirac_b200_stochastic_consensus_interval_withbeam(
    double *u, double *v, double *w, double *xo, int N, int Nbase, int tmb, int minibatches,
    baseline_t *barr, clus_source_t *carr, int M, int Mt, double *freqs, int Nchan, double deltaf,
    double uvmin, double uvmax, int bf_type, double b_ra0, double b_dec0, double ph_ra0,
    double ph_dec0, double ph_freq0, double *longitude, double *latitude, double *time_utc,
    int *Nelem, double **xx, double **yy, double **zz, elementcoeff *ecoeff, int doBeam, int nsolbw,
    int nepochs, int max_lbfgs, int lbfgs_m, double robust_nu, persistent_data_t *pt, double *pfreq,
    int ccid, double rho, int phase_only, int nadmm, int Npoly, double *B, double *Bi, double *rhok,
    double *Z, int use_global, double *res_00, double *res_01, double *res_0, double *res_1,
    int *fband);

#ifdef __cplusplus
}
#endif
#endif
