/*
 * dirac_b200 — full-batch calibration of one tile (`sagecal`'s default mode, with or without
 * `-B <doBeam>`, src/MS/fullbatch_mode.cpp:371-530, the !DoSim branch) in one call: the coherencies
 * at the tile's frequency, the SAGE fit and the full-resolution residual, with the sky, the data and
 * the coherencies staged on the device once; on one GPU, or sharded by cluster over one process per
 * GPU.  include/dirac_b200.h includes this header; it may also be included on its own.
 */
#ifndef DIRAC_B200_FULLBATCH_H
#define DIRAC_B200_FULLBATCH_H

#include "dirac_b200.h"
#include "dirac_b200_federated.h"

#ifdef __cplusplus
extern "C" {
#endif

/* replaces, for one tile without station beams (with beams: dirac_b200_fullbatch_tile_withbeam), the
 * driver's precalculate_coherencies -> sagefit_visibilities -> calculate_residuals_multifreq (or, with
 * -b 1, the per-channel loop of precalculate_coherencies, bfgsfit_visibilities and
 * calculate_residuals, fullbatch_mode.cpp:464-497).  The sky, u, v, w, the flags and the
 * channel-averaged data go to the device once; the coherencies are predicted into device memory and
 * never cross PCIe; x and xo come back once.
 *   u, v, w      [Nbase*tilesz] in seconds (already scaled by 1/c, as the driver does)      iodata.u/v/w
 *   x            [Nbase*tilesz][8] in: the channel-averaged data; out: the fit's residual, as
 *                sagefit_visibilities leaves it                                               iodata.x
 *   xo           [Nchan][Nbase*tilesz][8] in: the data of every channel; out: the residual, as
 *                calculate_residuals_multifreq leaves it (do_chan: as the -b 1 loop leaves it) iodata.xo
 *   N, Nbase, tilesz  stations, baselines N(N-1)/2, timeslots of the tile
 *   barr         [Nbase*tilesz] rows in the canonical order of generate_baselines, flags as
 *                preset_flags_and_data left them; out: the uv cut's flags (2) added, as
 *                precalculate_coherencies adds them (with do_chan, those of every channel too)
 *   carr, M, Mt  the sky model: M clusters, Mt = sum of their hybrid chunks; input only
 *   freq0        the tile's frequency: the coherencies of the fit are predicted at it     iodata.freq0
 *   deltaf       the bandwidth of all Nchan channels: the smearing width of the fit's coherencies;
 *                deltaf / Nchan that of one channel in the residual                     iodata.deltaf
 *   freqs        [Nchan] channel frequencies                                                iodata.freqs
 *   uvmin, uvmax the uv cut in wavelengths at freq0 (with do_chan, also at every channel)
 *                                                                    Data::min_uvcut, Data::max_uvcut
 *   pp           [8 N Mt] in: start Jones; out: the fit's solution (do_chan: the last channel's) p
 *   max_emiter, max_iter, max_lbfgs, lbfgs_m, linsolv, solver_mode, nulow, nuhigh, randomize
 *                as sagefit_visibilities takes them; the driver's first-tile substitutions (4x / 6x
 *                max_emiter, the LMCUT solver modes) stay with the caller, who passes what the driver
 *                would.  With do_chan the fit runs with max_lbfgs = 0, as the driver passes it.
 *   do_chan      0: the residual of all Nchan channels with the solution; != 0 (driver option -b 1):
 *                per channel the coherencies at freqs[c] (smearing deltaf / Nchan, the uv cut
 *                accumulating in barr), LBFGS from the fit's Jones with max_lbfgs, lbfgs_m,
 *                solver_mode and mean_nu, and the residual of that channel, without phase_only (the
 *                driver's calculate_residuals takes none)                               Data::doChan
 *   ccid, rho, phase_only   the correction of the residual by the cluster whose id is ccid, as
 *                calculate_residuals_multifreq takes it           Data::ccid, Data::rho, Data::phaseOnly
 *   rank, world  this process and the number of processes, one GPU each; world 1: one GPU
 *   allreduce, user   the sum over the ranks (the callback contract of dirac_b200_set_comm); NULL:
 *                the communicator of dirac_b200_nccl_init, which must then have `world` ranks
 *   mean_nu, res_0, res_1   out: as sagefit_visibilities writes them
 *   res_00, res_01   [Nchan] out with do_chan: every channel's cost before and after its LBFGS; not
 *                read otherwise (may be NULL)
 * Sharded (world > 1): every rank passes the same arguments (the whole carr and pp).  Rank r predicts
 * and fits only the contiguous block of ceil(M/world) clusters from r ceil(M/world) on, through
 * dirac_b200_create_shard with the hidden-data weight 1/world.  Each rank subtracts its own clusters'
 * corrected model (rank 0 from xo, the others from zero) and one all-reduce of Nchan x 8 x
 * Nbase x tilesz doubles sums them.  The correction cluster is looked up in the whole carr.  Every
 * rank returns the same pp, x, xo, barr, mean_nu, res_0 and res_1.
 * Device memory: the rank's coherencies, M_rank x Nbase x tilesz x 64 bytes (62 stations, 64
 * clusters, 120 timeslots: 929 MB), eight data-sized work buffers and xo, Nchan x Nbase x tilesz x 64
 * bytes.  A failed allocation after the check below prints a message and exits.
 * Returns 0 (whether or not res_1 < res_0), or -1 with a message on stderr and no output touched,
 * before any device work, when Nchan < 1, rank is outside [0, world), world > M, a rank's block of
 * clusters would be empty, world > 1 comes with neither a callback nor a communicator of that size,
 * do_chan is set with world > 1, or the memory above is more than the device has free. */
int dirac_b200_fullbatch_tile(
    double *u, double *v, double *w, double *x, double *xo, int N, int Nbase, int tilesz,
    baseline_t *barr, clus_source_t *carr, int M, int Mt, double freq0, double deltaf, double *freqs,
    int Nchan, double uvmin, double uvmax, double *pp, int max_emiter, int max_iter, int max_lbfgs,
    int lbfgs_m, int linsolv, int solver_mode, double nulow, double nuhigh, int randomize,
    int do_chan, int ccid, double rho, int phase_only, int rank, int world,
    dirac_b200_allreduce_fn allreduce, void *user, double *mean_nu, double *res_0, double *res_1,
    double *res_00, double *res_01);

/* dirac_b200_fullbatch_tile with station beams (`sagecal -B <doBeam>`): the driver's
 * precalculate_coherencies_withbeam(_gpu) and calculate_residuals_multifreq_withbeam(_gpu) branches.
 * The arguments are those of dirac_b200_fullbatch_tile with the beam arguments inserted after uvmax,
 * in the order of dirac_b200_stochastic_interval_withbeam:
 *   bf_type      STAT_SINGLE or STAT_TILE (array modes)                                  beam.bfType
 *   b_ra0, b_dec0, ph_ra0, ph_dec0   tile beam centre and phase centre (rad), already precessed
 *                                                               beam.b_ra0, b_dec0, p_ra0, p_dec0
 *   ph_freq0     the beam-former's reference frequency (the driver passes freq0)          iodata.freq0
 *   longitude, latitude   [N] station positions (rad)                                  beam.sx, beam.sy
 *   time_utc     [tilesz] the timeslots' JD                                             beam.time_utc
 *   Nelem, xx, yy, zz     per station the elements (STAT_TILE: the 16 dipoles of a tile, then the
 *                tiles), as readAuxData leaves them                      beam.Nelem, xx, yy, zz
 *   ecoeff       element modes: set_elementcoeffs for the narrow-band modes, set_elementcoeffs_wb over
 *                all Nchan channels for the wide-band ones                                   &ecoeff
 *   doBeam       DOBEAM_NONE (0): exactly dirac_b200_fullbatch_tile; 1..6 the array, full and element
 *                beams, narrow- and wide-band                                                  doBeam
 * The coherencies of the fit carry the beam at freq0 with the uv cut of
 * precalculate_coherencies_withbeam; the residual carries every channel's beam and, for wide-band
 * element beams, coefficient set c in channel c.  With do_chan the per-channel loop predicts and
 * subtracts without beams, as the driver's -b 1 loop does (DESIGN.md §7).
 * Device memory: besides that of dirac_b200_fullbatch_tile, the beam tables of the rank's S sources,
 * tilesz x Nchan x S x N x 72 bytes at most.
 * Returns 0, or -1 with a message and no output touched as dirac_b200_fullbatch_tile, and when doBeam
 * is outside 0..6 (the lunar element beam needs CSPICE), an array mode has a bf_type other than
 * STAT_SINGLE / STAT_TILE or no Nelem / xx / yy / zz, an element mode has no coefficient tables or a
 * wide-band one fewer than Nchan sets, or a beam has no longitude, latitude or time_utc. */
int dirac_b200_fullbatch_tile_withbeam(
    double *u, double *v, double *w, double *x, double *xo, int N, int Nbase, int tilesz,
    baseline_t *barr, clus_source_t *carr, int M, int Mt, double freq0, double deltaf, double *freqs,
    int Nchan, double uvmin, double uvmax, int bf_type, double b_ra0, double b_dec0, double ph_ra0,
    double ph_dec0, double ph_freq0, double *longitude, double *latitude, double *time_utc,
    int *Nelem, double **xx, double **yy, double **zz, elementcoeff *ecoeff, int doBeam, double *pp,
    int max_emiter, int max_iter, int max_lbfgs, int lbfgs_m, int linsolv, int solver_mode,
    double nulow, double nuhigh, int randomize, int do_chan, int ccid, double rho, int phase_only,
    int rank, int world, dirac_b200_allreduce_fn allreduce, void *user, double *mean_nu,
    double *res_0, double *res_1, double *res_00, double *res_01);

#ifdef __cplusplus
}
#endif

#endif
