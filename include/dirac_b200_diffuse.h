/*
 * dirac_b200 — coherencies of the diffuse cluster under spatial regularisation (sagecal-mpi
 * `-X lambda,mu,n0,fista_maxiter,cadence -D id`, src/MPI/sagecal_slave.cpp:669-695): the reference entry
 * point with its name, argument list and meaning, and its form on a resident problem.
 * include/dirac_b200.h includes this header; it may also be included on its own.
 */
#ifndef DIRAC_B200_DIFFUSE_H
#define DIRAC_B200_DIFFUSE_H

#include "dirac_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* replaces recalculate_diffuse_coherencies, src/lib/Radio/Dirac_radio.h:228 (diffuse_predict.c:295-586).
 * Rewrites cluster cid's four coherencies x[row][cid][0..3] of every row, flagged rows included, from
 * the shapelet sources of cluster cid and the spatial model Z (2N x 2G complex, column major,
 * G = sh_n0^2): the first source replaces the value and later sources add to it; a cluster without
 * sources is left untouched.  Nbase counts rows (baselines x timeslots).  tdelta, dec0, uvmin, uvmax,
 * Nt and use_cuda are accepted and unused: the computation always runs on the GPU, in fp64.  A cid
 * outside [0, M) or a source that is not a shapelet prints a message and exits (1), as the reference
 * does; so do shapelet orders outside 1..32 and orders whose product tensor leaves the double range. */
int recalculate_diffuse_coherencies(double *u, double *v, double *w, double *x, int N, int Nbase,
                                    baseline_t *barr, clus_source_t *carr, int M, double freq0,
                                    double fdelta, double tdelta, double dec0, double uvmin,
                                    double uvmax, int diffuse_cluster, int sh_n0, double sh_beta,
                                    double *Z, int Nt, int use_cuda);

/* the same into local cluster cid of a resident problem (u, v, w: Nbase*tilesz rows in the problem's
 * order); the coherencies never leave the device.  Call it before dirac_b200_sagefit_admm* when the
 * spatial model changes (INTEGRATION.md section 5b).  Returns 0. */
int dirac_b200_diffuse_coherencies(dirac_b200_problem *pr, const double *u, const double *v,
                                   const double *w, const clus_source_t *carr, double freq0,
                                   double fdelta, int cid, int sh_n0, double sh_beta,
                                   const double *Z);

#ifdef __cplusplus
}
#endif
#endif
