/*
 * dirac_b200 — influence-function diagnostics (the driver's `-i 1`, src/MS/fullbatch_mode.cpp:526-530,
 * and the full-batch MPI slave in place of its residual, src/MPI/sagecal_slave.cpp:965-970): the
 * reference entry point with its name, argument list and meaning.  include/dirac_b200.h includes
 * this header; it may also be included on its own.
 */
#ifndef DIRAC_B200_DIAGNOSTICS_H
#define DIRAC_B200_DIAGNOSTICS_H

#include "dirac_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* replaces calculate_diagnostics_gpu, src/lib/Radio/Dirac_radio.h:676 (diagnostics.c:1020-1182,
 * influence_function.cu).  x is [Nchan][Nbase*tilesz][8], in and out.
 *  1. x -= J_p C_k J_q^H of every cluster k, whatever its id, every row and channel, with the Jones
 *     of the row's hybrid chunk (row / ceil(Nbase*tilesz / nchunk)) and the station beams when
 *     dobeam is set; the smearing width of a channel is fdelta / Nchan.
 *  2. Per cluster, on channel 0: the 4N x 4N Hessian of the unflagged rows, the 4N x Nbase
 *     right-hand side AdV (split station layout, rows 2p+{0,1} and 2N+2p+{0,1}) and, after the
 *     diagonal conditioning of the reference (every real diagonal entry with |h| < 1 becomes 1, the
 *     C integer abs of diagnostics.c:712; plus 0.5 rho[k] Fd1 when rho, Bpoly and Bi are all given,
 *     Bi at cluster k's Npoly x Npoly block), X = H^-1 AdV by an LU with pivoting.
 *  3. dR: of every row, flagged or not, kron(conj(J_q) C^T, I2) times the split-layout rows of
 *     station p of X, summed over clusters and timeslots into four Nbase x Nbase matrices.
 *  4. The eigenvalues of each of the four: x[8b+2c] = E_c[b], x[8b+2c+1] = E_c[Nbase+b] with E_c the
 *     interleaved (re, im) eigenvalues of correlation c in the solver's order, for channel 0 of
 *     timeslot 0, copied to every timeslot; channels >= 1 keep the step-1 residual.
 * Deviations from the reference (DESIGN.md section 7): fp64 throughout where it computes in fp32
 * with atomics (so results agree to fp32 rounding and are bit-identical run to run); LU in place of
 * cgels (the same solution for a nonsingular H); one GPU.  Every row of one baseline index must
 * join the same two stations in every timeslot, and no two baselines the same pair.
 * Nt, Nf and Mt are accepted and unused; tdelta and dec0 as in calculate_residuals_multifreq.
 * Size bound: the four dR matrices take 64*Nbase^2 bytes (229 MB at 62 stations, 4.2 GB at 128),
 * X another 64*N*Nbase*M.  When these, the Hessians and the eigenvalue workspace do not fit in free
 * device memory the call prints a message and returns -1 before any device work; the 512-station
 * shape (about 1.1 TB) is far outside it, as it is for the reference.  Malformed beam arguments,
 * chunk counts or station pairs also return -1 with a message.  Otherwise returns 0. */
int calculate_diagnostics_gpu(double *u, double *v, double *w, double *p, double *x, int N, int Nbase,
                              int tilesz, baseline_t *barr, clus_source_t *carr, int M, double *freqs,
                              int Nchan, double fdelta, double tdelta, double dec0, int bf_type,
                              double b_ra0, double b_dec0, double ph_ra0, double ph_dec0,
                              double ph_freq0, double *longitude, double *latitude, double *time_utc,
                              int *Nelem, double **xx, double **yy, double **zz, elementcoeff *ecoeff,
                              int dobeam, double *rho, double *Bpoly, double *Bi, int Mt, int Npoly,
                              int Nf, int Nt);

#ifdef __cplusplus
}
#endif
#endif
