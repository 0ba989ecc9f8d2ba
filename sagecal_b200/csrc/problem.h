// Internal: the opaque dirac_b200_problem and the device-pointer primitives shared by the solvers.
#pragma once
#include <cusolverDn.h>
#include <cublas_v2.h>

#include <vector>

#include "../../include/dirac_b200.h"
#include "internal.cuh"

// blocked Cholesky of the sweep's batch of large systems (bigchol.cu)
struct BigChol;
// panels of nbk columns; inv_panel: the panel solve by the inverse of the diagonal block and a DGEMM;
// lookahead: panel j+1 on a second stream while the rest of panel j's trailing update runs
BigChol *db_bigchol_create(int n, int nbk, bool inv_panel, bool lookahead);
// what the LM runs (measured at n = 4096, 32 systems: DESIGN.md §5.2)
enum { BC_BLOCK = 256 };
static const bool BC_INV_PANEL = true, BC_LOOKAHEAD = true;
void db_bigchol_destroy(BigChol *bc);
// the batch: system b at A0 + b * stride, b < maxb (uploads the panels' pointer arrays)
void db_bigchol_bind_batch(BigChol *bc, double *A0, long long stride, int maxb);
void db_bigchol_factor_batch(BigChol *bc, int nb, int *info, int info_step, cudaStream_t st);

struct LMWork {
  bool ready;
  int n8;                 // 8N
  double *T;              // [Mt][Nbase][16] Gram tensors per (cluster, chunk), built on first use
  unsigned char *T_valid; // host, [Mt]
  double *Tsub;           // [Nbase][16] scratch (OS subsets, tests)
  double *JTJ0, *JTJ;     // [8N][8N]
  double *JTe, *JTe_new;  // [8N]
  double *Hst;            // [N][4]
  double *Dp;             // [8N]
  double *pnew;           // [8N]
  double *h_vec;          // pinned host scratch, 4*8N + 4N + 16
  int *devinfo;
  double *cswork;
  int lwork;
  bool own_chol;  // damped solves by the cluster Cholesky kernel (else cuSOLVER)
  double *bt_ws;  // large systems: workspace of the blocked triangular solves (kernels_bigtri.cu)
  BigChol *bc;    // large systems: blocked factorisation of the sweep's batch (bigchol.cu)
  double *jte_part;       // per-CTA station sums of the linear-mapped gradient pass
  bool step_armed, step_fused;  // trial point formed by the solver kernel's epilogue
  double *jtj_spec;       // J^T J assembled speculatively at the trial point (nullptr: none)
  cudaEvent_t ev_mail;    // marks the trial results' copy; the host waits on it, not on the stream
  double *tau;            // QR
  double *svdS, *svdU, *svdVT;
  cusolverDnHandle_t cs;
  cublasHandle_t cb;
  double2 *dbuf;          // [4][R] hidden data of the cluster being solved
  // robust LM (allocated on first use)
  double2 *wbuf;          // [4][R] sqrt-weights
  double2 *ebuf;          // [4][R] unweighted residual for the weight update
  double2 *os_eps, *os_w; // [4][R] misaligned ordered subsets: shifted residual / sqrt-weights + cut
  double *HP, *HQ;        // [N][2][10] station sums of the weighted normal matrix
  double *plast;          // [8N] device copy of the last evaluated trial point
  double *pold;           // [8N] Jones at the start of the visit (sharded closing pass)
  // normal matrices of ALL clusters of a sweep, assembled and factorised in one batch before the
  // sweep (each cluster's first LM solve then only needs the triangular solves)
  double *JB, *LB;        // [M][8N][8N] J^T J (cluster solvers only, else null) and the damped
                          // Cholesky factor
  size_t lb_stride;       // doubles between two factors in LB
  int lb_ld, binfo_step;  // leading dimension of a factor; ints per matrix in the status array
  double *HB;             // [M][N][4]
  double *mu_dev;         // [M] mu0 of each cluster
  double *h_mu;           // pinned
  int *binfo_dev, *h_binfo;
  double **LBptr_dev;     // [M] pointers into LB
  int *blist_dev, *btix_dev, *bpoff_dev;
  int *pref_slot;         // host [M]: slot of cluster k in the current batch, -1 if not prefactored
  const double *jtj0_cur; // matrix the damping loop of the current iteration starts from
  // in-place Cholesky of an unweighted system (8N beyond the cluster solver): the Gram tensors, Jones
  // and station sums the damped solves assemble J^T J + mu I from (sys_T null: the system is in JTJ0
  // or jtj0_cur and is copied with the damping)
  const double *sys_T, *sys_p, *sys_H;
};

struct dirac_b200_problem {
  DevProblem d;
  double *partials;
  int npartials;
  double2 *res;           // [4][R] residual of the full model
  double2 *vis_stage;     // [R][4] API-layout staging
  double *g;              // [8*N*Mt]
  LMWork lm;
  int own_stream;
  // cluster sharding over ranks: sum of a device buffer of doubles over all ranks (NCCL all-reduce,
  // supplied by the host); world == 1: never called
  int rank, world;
  void (*allreduce)(void *dev, long long count, void *stream, void *user);
  void *comm_user;
  int m_global;           // clusters over all ranks
  int k_global0;          // global index of local cluster 0
  double beta;            // hidden-data weight of the sharded SAGE sweep (1/world by default)
  // consensus (ADMM) terms of the running solve (dirac_b200_sagefit_admm), null otherwise
  const double *aug_y_host, *aug_bz_host, *aug_rho;  // host: [npar], [npar], [M]
  double *aug_dev;        // device: Y | BZ
  double2 *pm;            // [4][R] partial model / residual at the start of a sharded sweep
  double *xb;             // [8R + npar + m_global] sweep exchange message (sharded)
  double *pp_start;       // [npar] Jones at the start of a sharded sweep
  // LBFGS line model (allocated on first use)
  double2 *E0, *E1, *E2;  // [4][R] each
  double *poly_part;      // [5][db_stream_all_nblocks] per-CTA sums of the line quartic (one GPU)
  struct RtrWork *rtr;    // RTR / NSD solvers (rtr.cu), allocated on first use
};

// host waits on the device, timed (dirac_b200_host_stats): where the host-driven solver idles
void db_stream_sync(cudaStream_t st);
void db_event_sync(cudaEvent_t ev);
void db_flag_wait(const volatile unsigned long long *flag, unsigned long long epoch,
                  cudaStream_t st);
void *db_malloc(size_t bytes);
void db_free(void *p);
// device memory freed blocks hold in the allocator's cache (a failed cudaMalloc gives it back)
size_t db_cached_bytes();
// exits with a message if there is no CUDA device: this library has no CPU fallback
void require_gpu();

// Device state of one call: a non-blocking stream, created here (after require_gpu) or borrowed from a
// resident problem, and the cudaMalloc buffers allocated through alloc / upload.  The destructor waits
// for the stream (uncounted: on the normal path the call has already synced), frees the buffers and
// destroys the stream if it created it.
class DeviceScope {
 public:
  DeviceScope();
  explicit DeviceScope(cudaStream_t borrowed);
  ~DeviceScope();
  DeviceScope(const DeviceScope &) = delete;
  DeviceScope &operator=(const DeviceScope &) = delete;
  template <class T> T *alloc(size_t n) {
    void *p = nullptr;
    DB_CHECK(cudaMalloc(&p, sizeof(T) * n));
    bufs_.push_back(p);
    return (T *)p;
  }
  // at least one element is allocated, so that an empty table is still a valid pointer; the host
  // array must stay alive until the next wait on st
  template <class T> T *upload(const T *h, size_t n) {
    T *d = alloc<T>(n ? n : 1);
    if (n) DB_CHECK(cudaMemcpyAsync(d, h, sizeof(T) * n, cudaMemcpyHostToDevice, st));
    return d;
  }
  template <class T> T *upload(const std::vector<T> &h) { return upload(h.data(), h.size()); }
  // the counted host wait (dirac_b200_host_stats), then the check for a failed launch
  void sync();
  const cudaStream_t st;

 private:
  const bool own_;
  std::vector<void *> bufs_;
};

// planar [M][4][R] device coherencies -> host x[row][M][8] (the API layout) through a db_malloc stage
// of at most 128 MB; waits for the copies once and counts the bytes (dirac_b200_transfer_stats)
void db_download_coh(const double2 *coh, double *x, int M, long long R, cudaStream_t st);
void db_count_launch(int n);
void db_prof_begin(int kind, double bytes, cudaStream_t st);
void db_prof_end(cudaStream_t st);
// a timed span enclosing other timed launches (db_prof_close ends its own record)
int db_prof_open(int kind, double bytes, cudaStream_t st);
void db_prof_close(int rec, cudaStream_t st);
cudaStream_t db_new_stream(int *owned);
void db_upload_vis(dirac_b200_problem *pr, const double *h, double2 *dst);
void db_download_vis(dirac_b200_problem *pr, const double2 *src, double *h);
void db_predict_dev(dirac_b200_problem *pr, const double *pp_dev, double2 *out, int out_mode,
                    int cost_mode, double nu, int slot);
double db_read_scalar(dirac_b200_problem *pr, int slot);
void db_grad_dev(dirac_b200_problem *pr, const double *pp_dev, double *g_dev, int robust,
                 double nu);
// Student's-t cost and minibatch-sign gradient of the row window [r_lo, r_hi) (problem.cu)
double db_cost_window_dev(dirac_b200_problem *pr, const double *pp_dev, double2 *out, double nu,
                          long long r_lo, long long r_hi);
void db_grad_window_dev(dirac_b200_problem *pr, const double *pp_dev, double *g_dev, double nu,
                        long long r_lo, long long r_hi);
// bfgsfit_visibilities on a resident problem (sage.cu)
int db_bfgsfit_dev(dirac_b200_problem *pr, double *pp, int max_lbfgs, int lbfgs_m, int solver_mode,
                   double mean_nu, double *res_0, double *res_1, bool keep_residual);
// sky models uploaded / bytes of coherencies copied between host and device (dirac_b200_transfer_stats)
void db_count_sky_upload();
void db_count_coh_host_bytes(size_t bytes);
void db_lm_init(dirac_b200_problem *pr);
void db_prefactor_sweep(dirac_b200_problem *pr, double tau);
void db_allreduce(dirac_b200_problem *pr, void *dev, long long count);
// sum over the ranks of the process-wide communicator regardless of cluster sharding (consensus over
// subbands: every rank holds its own, unsharded problem); no-op without a communicator
void db_allreduce_world(dirac_b200_problem *pr, void *dev, long long count);
int db_nccl_world();
void db_allreduce_stream(dirac_b200_allreduce_fn fn, void *user, void *dev, long long count,
                         cudaStream_t st);
// the projectback manifold average on device memory (kernels_manifold.cu)
int db_manifold_projectback(double *Y, int n, int Mt, int Nf, int Niter, const int *cr,
                            cudaStream_t st);void db_lm_set_aug(const double *y_dev, const double *bz_dev, const double *y_host,
                   const double *bz_host, double rho);
int db_overlap_available(const dirac_b200_problem *pr);
cudaStream_t db_comm_stream();
void db_allreduce_segments(dirac_b200_problem *pr, double **ptr, const long long *count, int nseg,
                           cudaStream_t st);
extern "C" {
void db_launch_residual_cost(const double2 *x, const double2 *pm, double2 *out, long long n4,
                             int out_mode, int cost_mode, double inv_nu, double *partials,
                             double *cost, unsigned int *counter, cudaStream_t st);
void db_launch_sumsq(const double2 *v, long long n4, double *partials, double *out,
                     unsigned int *counter, cudaStream_t st);
void db_launch_axpby(const double2 *x, double2 *y, long long n4, double a, double b,
                     cudaStream_t st);
void db_launch_cluster_rowmap(const double2 *coh_k, const double2 *in, const double2 *in2,
                              double2 *out, const unsigned char *flag, const double *pp,
                              const int *chunk_poff, int nchunk, const short2 *blpq, long long R,
                              int Nbase, int sign, double beta, cudaStream_t st);
}

// ---- minibatch bands (minibatch.cu) ---------------------------------------------------------------
// A band: channels [c0, c0 + nc) of one minibatch, coherencies [nc][M][4][R] and data [nc][4][R] in the
// planar layout, the flags of the minibatch's R rows.  BandDev is the device state the bands of one
// shape share: chunk tables, tiles, station pairs, the Jones, the gradient, the residual of up to maxnc
// channels and the scratch of the one-launch cost reduction.
struct BandView {
  const double2 *coh, *x;
  const unsigned char *flag;
  int nc;
};
struct BandDev {
  int N, Nbase, tilesz, M, Mt, maxnc, ntile;
  long long R, npar;
  ClusterDesc *clus;
  int *chunk_poff;
  TileDesc *tiles;
  short2 *blpq;
  double *pp, *g, *partials, *scal, *h_scal;
  unsigned int *counters;
  double2 *res;
  cudaStream_t st;
};
void db_build_tiles(int N, std::vector<TileDesc> &tiles);
// the flags of barr's R rows, after checking that they are in the canonical order of generate_baselines
// (message and exit(1) otherwise, as dirac_b200_create)
void db_canonical_flags(int N, int Nbase, int tilesz, const baseline_t *barr, unsigned char *flag);
BandDev *db_band_create(int N, int Nbase, int tilesz, const clus_source_t *carr, int M, int Mt,
                        int maxnc, cudaStream_t st);
void db_band_destroy(BandDev *bd);
// bfgsfit_minibatch_visibilities / _consensus on a resident band: res_0, res_1 the costs before and
// after the fit over 8 R nc; p (host, 8 N Mt) in/out; y, z, rho: consensus terms or null
void db_band_fit(BandDev *bd, const BandView &b, double *p, const double *y, const double *z,
                 const double *rho, int max_lbfgs, int lbfgs_m, double robust_nu, double *res_0,
                 double *res_1, persistent_data_t *indata);

// z = B_b Z of every chunk (consensus.cu): Z [Mt][Npoly][8N], Bb the band's Npoly basis values, z [Mt][8N]
void db_consensus_bz(const double *Z, const double *Bb, int N, int Mt, int Npoly, double *z);

void db_lm_free(dirac_b200_problem *pr);
void db_rtr_free(dirac_b200_problem *pr);
