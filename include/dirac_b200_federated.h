/*
 * dirac_b200 — the pieces of federated stochastic calibration (`sagecal-mpi -N <epochs> -M
 * <minibatches> -w <bands> -A <nadmm>`, src/MPI/sagecal_stochastic_slave.cpp and
 * sagecal_stochastic_master.cpp) with one rank per measurement set: a whole interval of the slave's
 * loop in one call per rank, with the master's projectback manifold average computed on every rank's
 * device after one all-reduce; and the pieces it is made of, for a host that keeps its own loop.
 * include/dirac_b200.h includes this header; it may also be included on its own.
 */
#ifndef DIRAC_B200_FEDERATED_H
#define DIRAC_B200_FEDERATED_H

#include "dirac_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* sum `count` doubles at device address `dev` over all ranks, in place, enqueued on the cudaStream_t
 * `stream` (the same contract as the callback of dirac_b200_set_comm) */
typedef void (*dirac_b200_allreduce_fn)(void *dev, long long count, void *stream, void *user);

/* replaces the stochastic slave's interval (sagecal_stochastic_slave.cpp:650-881) and, for it, the
 * master's exchange (sagecal_stochastic_master.cpp:334-354), for one measurement set on this rank, no
 * station beam.  nadmm x nepochs x minibatches x bands of bfgsfit_minibatch_consensus fits with the
 * consensus terms (y = Y_b, z = B_b Z, rho = rhok_b) on coherencies predicted once into device memory,
 * dirac_b200_federated_bands_update after every minibatch, and after the epochs of every ADMM
 * iteration the exchange:
 *   1. this rank writes Z into slot `rank` of a zeroed device buffer [world][8 N Npoly Mt];
 *   2. rank 0 appends its Mt draws cr_k (rand() % world when randomize, else 0);
 *   3. one all-reduce of the whole buffer, which only adds zeros and so gathers it exactly;
 *   4. every rank runs the projectback average (Niter 10 at ADMM 0, 2 after it, as the master does)
 *      and keeps slot `rank` as Zavg; the average is the same bit for bit on every rank;
 *   5. X_k += alphak[k] (Z_k - Zavg_k).
 * X, Y and Zavg belong to the call and start from zero.  Unlike the in-process consensus interval,
 * the uv cut holds in every pass (the slave predicts with the reloaded flags every time, DESIGN.md 7
 * item 24) and the fits see the cut (the slave's CPU build; item 25).
 * The arguments up to Npoly are those of dirac_b200_stochastic_consensus_interval; then:
 *   B        [nsolbw][Npoly] this rank's rows of dirac_b200_consensus_basis, taken over the bands'
 *            mean frequencies of ALL ranks plus the global minimum and maximum frequency, at the
 *            global reference frequency (the slave's setup_polynomials over the master's frequency
 *            list, :500-553): row f*nsolbw + b of that basis is band b of rank f
 *   Bi       [Mt][Npoly][Npoly] dirac_b200_consensus_prod_inverse_fed of B, rhok and alphak
 *   rhok     [nsolbw][Mt];  alphak [Mt] the federated weights (-u alpha, setweights)
 *   Z        [Mt][Npoly][8N] in/out: this rank's polynomial solution, kept by the caller
 *   use_global   != 0: every band's solution becomes B_b Z after the loop
 *   randomize    the master's first-projection draws (rank 0's rand() decides)
 *   rank, world  this rank and the number of ranks
 *   allreduce, user   the exchange's sum over the ranks; NULL: the communicator of
 *            dirac_b200_nccl_init, which must then have `world` ranks (world 1 needs neither)
 *   res_00, res_01   [nadmm][nepochs][minibatches][nsolbw] out: every fit's cost before and after
 *   res_0, res_1, fband   out: as dirac_b200_federated_bands_update left them after the last minibatch
 * What the slave does between intervals (its resets from res_1 and fband, :972-1006) stays with the
 * caller.  Returns 0, or -1 with a message and no output touched when nsolbw is outside [1, Nchan],
 * nadmm < 1, Npoly < 1, rank is outside [0, world), world > 64, or world > 1 with neither a callback nor
 * a communicator of that size. */
int dirac_b200_stochastic_federated_interval(
    double *u, double *v, double *w, double *xo, int N, int Nbase, int tmb, int minibatches,
    baseline_t *barr, clus_source_t *carr, int M, int Mt, double *freqs, int Nchan, double deltaf,
    double uvmin, double uvmax, int nsolbw, int nepochs, int max_lbfgs, int lbfgs_m, double robust_nu,
    persistent_data_t *pt, double *pfreq, int ccid, double rho, int phase_only, int nadmm, int Npoly,
    double *B, double *Bi, double *rhok, double *alphak, double *Z, int use_global, int randomize,
    int rank, int world, dirac_b200_allreduce_fn allreduce, void *user, double *res_00,
    double *res_01, double *res_0, double *res_1, int *fband);

/* replaces calculate_manifold_average_projectback (manifold_average.c:809), with its signature, so the
 * stochastic master links unchanged.  Y [Nf][M][8N] (host, in place): Nf solutions of M chunks, N
 * stations (N Npoly for polynomial solutions).  Per chunk every solution is aligned to the others up to
 * the unitary ambiguity of the chunk (Niter rounds of 2x2 Procrustes rotations towards the mean), and
 * the mean, rotated back onto each solution, replaces it.  The average runs on the device in one
 * kernel, with a fixed summation order: the same input gives the same output bit for bit.
 *   randomize  != 0: chunk k first projects onto solution rand() % Nf, drawn here for k = 0..M-1 in
 *              order; 0: onto solution 0.  This is the reference with Nt = 1; with more threads the
 *              reference's draws interleave between its threads in no fixed order.
 *   Nt         not used.
 * Returns 0, or -1 with a message on stderr and Y untouched when N, M or Nf is below 1, Niter is below
 * 0, or Nf is above 64 (the pairwise Grams of one chunk are kept in shared memory). */
int calculate_manifold_average_projectback(int N, int M, int Nf, double *Y, int Niter, int randomize,
                                           int Nt);

/* the same average on device memory: Y [Nf][M][8N] a device pointer; cr [M] host, the solution each
 * chunk first projects onto (NULL: solution 0 for all); stream a cudaStream_t (NULL: the legacy
 * stream).  Returns once the work is enqueued on the stream (cr is copied before the call returns);
 * -1 as above, or when a cr[k] is outside [0, Nf). */
int dirac_b200_manifold_projectback_dev(int N, int M, int Nf, double *Y, int Niter, const int *cr,
                                        void *stream);

/* replaces find_prod_inverse_full_fed (consensus_poly.c:546): Bi[k] = (sum_f rho[k + f*M] B_f B_f^T +
 * alpha[k] I)^-1, Npoly x Npoly per cluster, where every singular value s of the sum above 1e-12
 * becomes 1/(s + alpha[k]) and every other 1/alpha[k], as the reference forms it.  The sibling of
 * dirac_b200_consensus_prod_inverse.  Host arithmetic, no GPU needed. */
int dirac_b200_consensus_prod_inverse_fed(const double *B, double *Bi, int Npoly, int Nf, int M,
                                          const double *rho, const double *alpha);

/* The federated slave's ADMM step after the bands of one minibatch are fitted
 * (sagecal_stochastic_slave.cpp:731-852), with one measurement set per rank.  Host arithmetic, no GPU
 * needed.  Arguments as dirac_b200_consensus_bands_update, and:
 *   admm         the ADMM iteration, >= 0; from 1 on the federated term is added
 *   alphak       [Mt] the federated-averaging weight of every chunk
 *   Zavg, X      [Mt][Npoly][8N] the last manifold average of the ranks' Z and the running sum of
 *                alpha_k (Z_k - Zavg_k); read only when admm >= 1
 * It differs from dirac_b200_consensus_bands_update as the slave differs from the single-process
 * driver (DESIGN.md 7, items 20-22):
 *   res_0, res_1 out: the plain mean of res_00 / res_01 over the bands of this minibatch;
 *   fband[b]     out: resband[b] > 1.5 res_1, resband[b] = res_01[b] when both costs are > 0, else 1e12;
 *   z            sum over the GOOD bands of B_b (x) (Y_b + rho_b J_b): band 0 only when it is good;
 *   from admm 1 on, z[p][k] += alphak[k] Zavg[k][p] - X[k][p];
 *   Z = Bi z, and the good bands get Y_b -= rho_b B_b Z.
 * Returns 0, or -1 with a message and nothing touched when a size is below 1 or admm is negative. */
int dirac_b200_federated_bands_update(int N, int Mt, int nsolbw, int Npoly, int admm,
                                      const double *res_00, const double *res_01,
                                      const double *pfreq, const double *B, const double *Bi,
                                      const double *rhok, const double *alphak, const double *Zavg,
                                      const double *X, double *res_0, double *res_1, double *Y,
                                      double *Z, int *fband);

#ifdef __cplusplus
}
#endif

#endif
