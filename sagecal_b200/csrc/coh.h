// Internal: packed sky model for the device-side coherency prediction.
#pragma once
#include "internal.cuh"

#define STYPE_POINT_ 0
#define STYPE_GAUSSIAN_ 1
#define STYPE_DISK_ 2
#define STYPE_RING_ 3
#define STYPE_SHAPELET_ 4

// one source, 240 bytes (multiple of 16: TMA bulk-copy granularity)
struct DevSource {
  double ll, mm, nn, sI, sQ, sU, sV, stype;
  double eX, eY, eP, cxi, sxi, cphi, sphi, use_projection;
  double sI0, sQ0, sU0, sV0, f0, spec_idx, spec_idx1, spec_idx2;
  double sh_n0, sh_beta, sh_off, pad_;  // shapelets: order, scale, first coefficient in CohArgs::modes
  double ra, dec;                       // direction of the source (beam tables)
};

#define COH_SEG_MAX 96  // sources staged per bulk copy (2 x 96 x 240 B = 45 KB of smem)
#define COH_SHAPELET_MAX_N0 32  // largest shapelet order the device kernel takes

// a run of <= COH_SEG_MAX sources of one cluster
struct CohSegment {
  int first;    // index into the packed source array
  int count;
  int cluster;
  int last;     // 1 if this run closes its cluster
};

struct CohArgs {
  const double *u, *v, *w;   // [R] seconds
  const DevSource *src;
  const double *modes;       // shapelet coefficients of all sources, back to back (may be null)
  const CohSegment *segs;
  int nseg;
  const double *freqs;       // device, [Nchan]
  int Nchan;
  double fdelta2;            // half channel width used for the |sinc| smearing
  double uvmin, uvmax;
  long long R;
  double2 *coh;              // MODE 0 out: planar [M][4][R]
  unsigned char *flag;       // MODE 0: uv-cut flags (may be null)
  double2 *xout;             // MODE 1, 2 in/out: [Nchan][R][4]
  // MODE 2 (full-resolution residual / simulation with solutions, residual.c:681-938,1342-1618)
  const int *sta1, *sta2;        // [R] stations of every row
  const double *p;               // Jones solutions (layout of pp)
  const int *clus_nchunk;        // [M]
  const int *clus_chunk0;        // [M] first entry of cluster k in chunk_poff
  const int *chunk_poff;         // [Mt]
  const signed char *clus_coef;  // [M] sign of J C J^H in x: -1 subtract, +1 add, 0 skip the cluster
  const double *pinv;            // inverse Jones of the correction cluster [nchunk][N][8], or null
  int pinv_nchunk, N;
  // station beams (predict_withbeam.c:300-420): tables per (timeslot, channel, source, station) made
  // by k_beam_tables; sta1 / sta2 and Nbase (rows per timeslot) are needed then in every mode
  const double *beam_af;         // array factor [T][Nchan][S][N], or null
  const double2 *beam_E;         // element beam E-Jones [T][Nchan][S][N][4], or null
  int beam_S;                    // sources over all clusters
  int Nbase;                     // rows per timeslot
};

// tables of the station beam towards every source (stationbeam.c:49-430, elementbeam.c:384-460)
struct BeamArgs {
  const DevSource *src;
  int S;
  const double *freqs;           // [Nf] channel frequencies
  int Nf;
  double f0;                     // beam-former reference frequency (ph_freq0)
  const double *time_jd;         // [T]
  int T;
  const double *lon, *lat;       // [N]
  int N;
  const int *elem_off;           // [N] first element of station n in ex / ey / ez
  const int *Nelem;              // [N] elements (STAT_SINGLE) / tiles (STAT_TILE) of station n
  const double *ex, *ey, *ez;
  int bf_type;                   // STAT_SINGLE 1, STAT_TILE 2
  double b_ra0, b_dec0, ra0, dec0;
  int wideband;                  // beam-former frequency = channel frequency, per-channel element coefficients
  // element beam coefficients (elementcoeff, Dirac_common.h:153-162)
  int ecM, ecNmodes;
  double ecbeta;
  const double2 *pat_phi, *pat_theta;  // [Nf_coeff][Nmodes]
  const double *preamble;        // [Nmodes]
  double *af;                    // out, or null
  double2 *E;                    // out, or null
};

// diffuse cluster (recalculate_diffuse_coherencies, diffuse_predict.c:295-586; kernels_diffuse.cu)
struct DiffuseSource {
  double ll, mm, nn, beta;   // direction; shapelet scale in the Fourier plane (exinfo_shapelet.beta)
  int n0, pad_;
  long long scoh;            // first entry in DiffuseArgs::scoh ([n0*n0][4] Stokes-weighted modes)
  long long cf1, cf2;        // first entries of its two product tensors in DiffuseArgs::cf
  long long cjq;             // first entry of its station products in DiffuseArgs::cjq ([N][n0*n0][4])
};
struct DiffuseArgs {
  const DiffuseSource *src;
  int ns;                    // sources, in the reference's order
  int N, sh;                 // stations; order of the spatial model (G = sh*sh modes)
  const double2 *Zt;         // [N][G][4] per-station spatial modes, 2x2 blocks transposed (:374-383)
  const double2 *scoh;
  const double *cf;
  double2 *cjq;              // scratch: C_Jq of every source and station
  const short2 *pairs;       // [npairs] stations (p, q) of each baseline
  int npairs;
  const long long *row_off;  // [npairs + 1] rows of baseline b: rows[row_off[b] .. row_off[b+1])
  const long long *rows;     //   or, when null, rows b + t*Nbase, t < ntime
  int ntime, Nbase;
  const double *u, *v, *w;   // [R] seconds
  double freq0, fdelta2;
  long long R;
  double2 *coh;              // planar [4][R] of the cluster, rewritten
};

extern "C" {
// station products, then the prediction of every row (profile kind 12); max_n0: largest source order
void db_launch_diffuse(const DiffuseArgs *a, int max_n0, cudaStream_t st);
void db_launch_coherencies(const CohArgs *a, cudaStream_t st);
void db_launch_predict_multifreq(const CohArgs *a, cudaStream_t st);
void db_launch_residual_multifreq(const CohArgs *a, cudaStream_t st);
void db_launch_beam_tables(const BeamArgs *a, cudaStream_t st);
}
