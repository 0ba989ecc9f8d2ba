// Internal: the influence-function kernels of calculate_diagnostics_gpu (kernels_influence.cu).
#pragma once
#include "../../include/dirac_b200.h"
#include "internal.cuh"

// the beam arguments of the *_withbeam entry points (coh_host.cu)
struct BeamSpec {
  int bf_type;
  double b_ra0, b_dec0, ph_ra0, ph_dec0, ph_freq0;
  const double *longitude, *latitude, *time_utc;
  int tilesz;
  const int *Nelem;
  double **xx, **yy, **zz;
  const elementcoeff *ecoeff;
  int doBeam;
};
// the beam arguments checked before any device work: true (with a message naming fn) if refused
bool beam_refused(const char *fn, const BeamSpec &b, int N, int Nchan);

// what the model stage of calculate_diagnostics_gpu leaves on the device (db_diagnostics_model)
struct DiagModel {
  double2 *x;                    // [Nchan][R][4] residual of every channel
  double2 *coh;                  // [M][R][4] coherencies of channel 0
  const double *p;               // Jones
  const int *clus_nchunk, *clus_chunk0, *chunk_poff;
};
class DeviceScope;
int db_diagnostics_model(DeviceScope &ds, const double *u, const double *v, const double *w,
                         const double *p, const double *x, int N, int Nbase, int tilesz,
                         const baseline_t *barr, const clus_source_t *carr, int M,
                         const double *freqs, int Nchan, double fdelta, const BeamSpec *beam,
                         DiagModel *out);

// Rows are r = t*Nbase + b; every row of baseline b joins stations sta1[b], sta2[b] (checked on the
// host), so per-baseline time sums are exact.  Complex matrices are column major.
struct InflArgs {
  int N, Nbase, T, M;
  long long R;                  // Nbase * T
  const double2 *coh;           // [M][R][4] coherencies of channel 0
  const double2 *res;           // [R][4] residual of channel 0
  const double *p;              // Jones, the API layout
  const int *clus_nchunk;       // [M]
  const int *clus_chunk0;       // [M] first entry of cluster k in chunk_poff
  const int *chunk_poff;        // offsets of the (cluster, chunk) blocks in p
  const int *sta1, *sta2;       // [Nbase]
  const unsigned char *flag;    // [R]
  const int *st_off;            // [N+1] CSR over stations of the entries in st_bl
  const int *st_bl;             // 2*b + side: baseline b with the station as sta1 (0) or sta2 (1)
  double2 *H;                   // [M][4N][4N] Hessians
  double2 *AdV;                 // [M][Nbase][4N] right-hand sides
  double2 *S;                   // [M][Nbase][4] sum over timeslots of conj(J_q) C^T (every row)
  const double2 *X;             // [M][Nbase][4N] solutions read by the dR pass
  double2 *dR;                  // [4][Nbase][Nbase] one matrix per correlation
};

extern "C" {
// H and AdV of all M clusters (zeroed first), and S
void db_launch_infl_assemble(const InflArgs *a, cudaStream_t st);
// the reference's diagonal conditioning: Re H_ii in (-1, 1) becomes 1, then + hadd[k] (hadd may be
// null)
void db_launch_infl_condition(const InflArgs *a, const double *hadd, cudaStream_t st);
// dR from S and X, written once
void db_launch_infl_dr(const InflArgs *a, cudaStream_t st);
// eigenvalues W [4][Nbase] (complex) into channel 0 of x ([R][4]), every timeslot
void db_launch_infl_eigs(const double2 *W, double2 *x, int Nbase, int T, cudaStream_t st);
}
