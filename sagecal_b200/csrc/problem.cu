// Device-resident problem ("one solve interval") and the thin dirac_b200_* layer over the kernels.
// Replaces the per-call H2D copies / cudaMalloc churn of the reference GPU path
// (clmfit_fl.c:193-225, lbfgs_cuda.c:93-131, mderiv.cu:1402-1460) with one resident copy.
#include <string.h>
#include <thread>
#include <vector>

#include "../../include/dirac_b200.h"
#include "internal.cuh"
#include "problem.h"

static unsigned long long g_launches = 0;
// host <-> device traffic of the two large operands a resident call keeps on the device
static unsigned long long g_sky_uploads = 0, g_coh_host_bytes = 0;
void db_count_sky_upload() { g_sky_uploads++; }
void db_count_coh_host_bytes(size_t bytes) { g_coh_host_bytes += bytes; }
extern "C" void dirac_b200_transfer_stats(unsigned long long *sky_uploads,
                                          unsigned long long *coh_host_bytes, int reset) {
  if (sky_uploads) *sky_uploads = g_sky_uploads;
  if (coh_host_bytes) *coh_host_bytes = g_coh_host_bytes;
  if (reset) g_sky_uploads = g_coh_host_bytes = 0;
}
void db_count_launch(int n) { g_launches += (unsigned long long)n; }
extern "C" unsigned long long dirac_b200_launch_count(void) { return g_launches; }

// ---- optional per-launch CUDA-event timing (bench.py's roofline leg) -----------------------------
struct ProfRec { cudaEvent_t a, b; int kind; double bytes; };
static std::vector<ProfRec> g_prof;
static std::vector<cudaEvent_t> g_evpool;
static int g_prof_on = 0;
static cudaEvent_t prof_event() {
  if (!g_evpool.empty()) { cudaEvent_t e = g_evpool.back(); g_evpool.pop_back(); return e; }
  cudaEvent_t e;
  DB_CHECK(cudaEventCreate(&e));
  return e;
}
// kinds: 13 k_stream_band (band cost or residual), 14 k_grad_tma_band (band gradient), 15
// k_beam_tables (station beam tables), 16 the stochastic interval's coherency predictions, 17
// k_manifold_projectback; calculate_diagnostics_gpu: 18 the model stage, 19 Hessians and right-hand
// sides, 20 the LU solves, 21 k_infl_dr, 22 the four eigenvalue problems, 23 the whole call;
// dirac_b200_fullbatch_tile: 24 the coherencies at freq0 (beam tables included), 25 the SAGE fit
#define DB_PROF_KINDS 26
static unsigned long long g_kind_count[DB_PROF_KINDS] = {0};
extern "C" unsigned long long dirac_b200_kernel_count(int kind) {
  return (kind >= 0 && kind < DB_PROF_KINDS) ? g_kind_count[kind] : 0ull;
}
void db_prof_begin(int kind, double bytes, cudaStream_t st) {
  if (kind >= 0 && kind < DB_PROF_KINDS) g_kind_count[kind]++;
  if (!g_prof_on) return;
  ProfRec r; r.a = prof_event(); r.b = prof_event(); r.kind = kind; r.bytes = bytes;
  DB_CHECK(cudaEventRecord(r.a, st));
  g_prof.push_back(r);
}
void db_prof_end(cudaStream_t st) {
  if (!g_prof_on) return;
  DB_CHECK(cudaEventRecord(g_prof.back().b, st));
}
// a timed span that may enclose other timed launches: db_prof_open returns its record (-1 when
// profiling is off), db_prof_close ends that record rather than the last one
int db_prof_open(int kind, double bytes, cudaStream_t st) {
  if (!g_prof_on) {
    if (kind >= 0 && kind < DB_PROF_KINDS) g_kind_count[kind]++;
    return -1;
  }
  db_prof_begin(kind, bytes, st);
  return (int)g_prof.size() - 1;
}
void db_prof_close(int rec, cudaStream_t st) {
  if (rec >= 0 && g_prof_on && rec < (int)g_prof.size()) DB_CHECK(cudaEventRecord(g_prof[rec].b, st));
}
extern "C" void dirac_b200_profile_enable(int on) {
  for (auto &r : g_prof) { g_evpool.push_back(r.a); g_evpool.push_back(r.b); }
  g_prof.clear();
  g_prof_on = on;
}
extern "C" int dirac_b200_profile_read(int kind, double *ms, double *bytes) {
  DB_CHECK(cudaDeviceSynchronize());
  int cnt = 0; double t = 0.0, by = 0.0;
  for (auto &r : g_prof) if (r.kind == kind) {
    float f = 0.f; DB_CHECK(cudaEventElapsedTime(&f, r.a, r.b)); t += f; by += r.bytes; cnt++;
  }
  if (ms) *ms = t;
  if (bytes) *bytes = by;
  return cnt;
}

// ---- stream the library works on: its own, unless the host supplies one ---------------------------
static cudaStream_t g_user_stream = nullptr;
static int g_have_user_stream = 0;
extern "C" void dirac_b200_set_stream(void *stream) {
  g_user_stream = (cudaStream_t)stream;
  g_have_user_stream = (stream != nullptr);
}
cudaStream_t db_new_stream(int *owned) {
  if (g_have_user_stream) { *owned = 0; return g_user_stream; }
  cudaStream_t st;
  DB_CHECK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  *owned = 1;
  return st;
}

// ---- test / tuning options ------------------------------------------------------------------------
static int g_opt[DB_OPT_COUNT] = {0, 0, 0, 0, 0, 0, 0, 0};
int db_opt(int id) { return (id >= 0 && id < DB_OPT_COUNT) ? g_opt[id] : 0; }
extern "C" int dirac_b200_set_option(const char *name, int value) {
  if (!strcmp(name, "cp_rows")) { g_opt[DB_OPT_CP_ROWS] = value; return 0; }
  if (!strcmp(name, "line_direct")) { g_opt[DB_OPT_LINE_DIRECT] = value; return 0; }
  if (!strcmp(name, "os_consistent")) { g_opt[DB_OPT_OS_CONSISTENT] = value; return 0; }
  // robust RTR / NSD: nu update as if the reference's unjoined thread sums were all still zero
  // (rtr_algo.h: update_weights)
  if (!strcmp(name, "rtr_nu_unjoined")) { g_opt[DB_OPT_RTR_NU_UNJOINED] = value; return 0; }
  // sagefit_visibilities_admm: LM on the augmented cost instead of the reference's robust RTR
  if (!strcmp(name, "admm_lm")) { g_opt[DB_OPT_ADMM_LM] = value; return 0; }
  // sagefit: hand back the residual the sweeps kept even when no LBFGS step replaced it (the one
  // the LBFGS stage starts from), instead of predicting it afresh
  if (!strcmp(name, "sweep_residual")) { g_opt[DB_OPT_SWEEP_RESIDUAL] = value; return 0; }
  return -1;
}
// SMs of the current device (grids of the one-wave kernels are sized from it)
int db_sm_count() {
  static int n[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (!n[dev]) {
    int v = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
    n[dev] = v;
  }
  return n[dev];
}

void require_gpu() {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    fprintf(stderr,
            "dirac_b200: no CUDA device available (%s). This library has no CPU fallback.\n",
            cudaGetErrorString(e));
    exit(1);
  }
}

// ---- caching device allocator ---------------------------------------------------------------------
// The drop-in entry points build and tear down a resident problem per call, like the reference
// (lmfit.c:831-1046 allocates and frees every scratch vector per call).  cudaMalloc/cudaFree of GBs
// cost milliseconds to hundreds of milliseconds (32 GB of coherencies at 512 stations: 50-350 ms
// measured) and serialise the device, so freed blocks are kept and handed out again when a request
// of exactly the same size comes back (the driver calls with the same shapes tile after tile).
// Bounded: the cache holds at most 75 % of the device's memory, so that a 512-station shard with its
// solver workspaces (55 GB) stays cached on an 80 GB H100 ($DIRAC_B200_CACHE_GB overrides, 0
// disables); a failed cudaMalloc gives the whole cache back and retries once;
// dirac_b200_release_cache() empties it on request.
#include <map>
#include <unordered_map>
static std::multimap<size_t, void *> g_free_blocks;
static std::unordered_map<void *, size_t> g_live_blocks;
static size_t g_cached_bytes = 0;
static size_t cache_cap() {
  static size_t cap = (size_t)-1;
  if (cap == (size_t)-1) {
    const char *e = getenv("DIRAC_B200_CACHE_GB");
    if (e) {
      cap = (size_t)(atof(e) * 1073741824.0);
    } else {
      size_t fr = 0, tot = 0;
      cap = (cudaMemGetInfo(&fr, &tot) == cudaSuccess) ? tot / 4 * 3 : ((size_t)6 << 30);
    }
  }
  return cap;
}
static void cache_release_all() {
  for (auto &kv : g_free_blocks) cudaFree(kv.second);
  g_free_blocks.clear();
  g_cached_bytes = 0;
}
extern "C" void dirac_b200_release_cache(void) { cache_release_all(); }
size_t db_cached_bytes() { return g_cached_bytes; }
void *db_malloc(size_t bytes) {
  bytes = (bytes + 255) & ~(size_t)255;
  auto it = g_free_blocks.find(bytes);
  void *p = nullptr;
  if (it != g_free_blocks.end()) {
    p = it->second;
    g_free_blocks.erase(it);
    g_cached_bytes -= bytes;
  } else {
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e != cudaSuccess) {  // give the cache back and retry once
      cudaGetLastError();
      cache_release_all();
      DB_CHECK(cudaMalloc(&p, bytes));
    }
  }
  g_live_blocks[p] = bytes;
  return p;
}
void db_free(void *p) {
  if (!p) return;
  auto it = g_live_blocks.find(p);
  if (it == g_live_blocks.end()) {
    cudaFree(p);
    return;
  }
  const size_t bytes = it->second;
  g_live_blocks.erase(it);
  if (g_cached_bytes + bytes > cache_cap()) {
    cudaFree(p);
  } else {
    g_free_blocks.insert({bytes, p});
    g_cached_bytes += bytes;
  }
}

static cudaStream_t new_call_stream() {
  require_gpu();
  cudaStream_t st;
  DB_CHECK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  return st;
}
DeviceScope::DeviceScope() : st(new_call_stream()), own_(true) {}
DeviceScope::DeviceScope(cudaStream_t borrowed) : st(borrowed), own_(false) {}
DeviceScope::~DeviceScope() {
  cudaStreamSynchronize(st);
  for (void *p : bufs_) cudaFree(p);
  if (own_) cudaStreamDestroy(st);
}
void DeviceScope::sync() {
  db_stream_sync(st);
  DB_CHECK(cudaGetLastError());
}

template <typename T>
static T *dev_alloc(size_t n) {
  return (T *)db_malloc(n * sizeof(T) + 16);
}

void db_build_tiles(int N, std::vector<TileDesc> &tiles) {
  int npb = (N - 1 + TILE_P - 1) / TILE_P;  // p in [0, N-2]
  int nqb = (N + TILE_Q - 1) / TILE_Q;
  for (int pb = 0; pb < npb; pb++)
    for (int qb = 0; qb < nqb; qb++) {
      int pmin = pb * TILE_P;
      int qmax = qb * TILE_Q + TILE_Q - 1;
      if (qmax > N - 1) qmax = N - 1;
      if (qmax > pmin) {
        TileDesc t;
        t.pb = (short)pb;
        t.qb = (short)qb;
        tiles.push_back(t);
      }
    }
}

static dirac_b200_problem *create_impl(int N, int Nbase, int tilesz, const baseline_t *barr,
                                       const clus_source_t *carr, int M, int Mt, const double *coh,
                                       const double *x, long long npar);

extern "C" dirac_b200_problem *dirac_b200_create(int N, int Nbase, int tilesz,
                                                 const baseline_t *barr, const clus_source_t *carr,
                                                 int M, int Mt, const double *coh,
                                                 const double *x) {
  return create_impl(N, Nbase, tilesz, barr, carr, M, Mt, coh, x, (long long)8 * N * Mt);
}

// One rank's shard of a cluster-sharded solve: carr/coh hold only the local clusters, whose
// carr[k].p[] are offsets into the GLOBAL Jones vector of npar doubles.
extern "C" dirac_b200_problem *dirac_b200_create_shard(int N, int Nbase, int tilesz,
                                                       const baseline_t *barr,
                                                       const clus_source_t *carr_local,
                                                       int M_local, int Mt_local,
                                                       long long npar_global, const double *coh,
                                                       const double *x) {
  return create_impl(N, Nbase, tilesz, barr, carr_local, M_local, Mt_local, coh, x, npar_global);
}

extern "C" void dirac_b200_set_comm(dirac_b200_problem *pr, int rank, int world,
                                    void (*allreduce)(void *, long long, void *, void *),
                                    void *user, int m_global, int k_global0, double beta) {
  pr->rank = rank;
  pr->world = world;
  pr->allreduce = allreduce;
  pr->comm_user = user;
  pr->m_global = m_global;
  pr->k_global0 = k_global0;
  pr->beta = (beta > 0.0) ? beta : 1.0 / (double)(world > 0 ? world : 1);
}


// the row order must be the canonical one (baseline_utils.c:445-461): checked, bit-exact
// (15.7 M rows at 512 stations x 120 timeslots: shared out over a few host threads by timeslot)
void db_canonical_flags(int N, int Nbase, int tilesz, const baseline_t *barr, unsigned char *hflag) {
  const long long R = (long long)Nbase * tilesz;
  const long long Nb = (long long)N * (N - 1) / 2;
  int nthr = (R > (1 << 20)) ? 8 : 1;
  if (nthr > tilesz) nthr = tilesz;
  std::vector<long long> bad(nthr, -1);
  auto work = [&](int th) {
    for (int t = th; t < tilesz; t += nthr) {
      long long r = (long long)t * Nb;
      for (int p = 0; p < N - 1; p++)
        for (int q = p + 1; q < N; q++, r++) {
          if (barr[r].sta1 != p || barr[r].sta2 != q) {
            if (bad[th] < 0) bad[th] = r;
            return;
          }
          hflag[r] = barr[r].flag;
        }
    }
  };
  if (nthr == 1) {
    work(0);
  } else {
    std::vector<std::thread> pool;
    for (int th = 0; th < nthr; th++) pool.emplace_back(work, th);
    for (auto &th : pool) th.join();
  }
  for (int th = 0; th < nthr; th++)
    if (bad[th] >= 0) {
      const long long r = bad[th];
      fprintf(stderr, "dirac_b200: barr[%lld]=(%d,%d) is not in the canonical order of "
                      "generate_baselines; unsupported row order\n", r, barr[r].sta1, barr[r].sta2);
      exit(1);
    }
}

static dirac_b200_problem *create_impl(int N, int Nbase, int tilesz, const baseline_t *barr,
                                       const clus_source_t *carr, int M, int Mt, const double *coh,
                                       const double *x, long long npar) {
  require_gpu();
  if (Nbase != N * (N - 1) / 2) {
    fprintf(stderr, "dirac_b200: Nbase=%d is not N(N-1)/2 for N=%d; only the canonical baseline "
                    "set of generate_baselines is supported\n", Nbase, N);
    exit(1);
  }
  if (N > 32767) {
    fprintf(stderr, "dirac_b200: N=%d stations exceed the supported 32767\n", N);
    exit(1);
  }
  dirac_b200_problem *pr = new dirac_b200_problem();
  memset(&pr->d, 0, sizeof(DevProblem));
  DevProblem &d = pr->d;
  d.N = N; d.Nbase = Nbase; d.tilesz = tilesz; d.M = M; d.Mt = Mt;
  d.R = (long long)Nbase * tilesz;
  d.npar = npar;
  pr->rank = 0; pr->world = 1; pr->allreduce = nullptr; pr->comm_user = nullptr;
  pr->m_global = M; pr->k_global0 = 0; pr->beta = 1.0;
  DB_CHECK(cudaGetDevice(&d.device));
  d.stream = db_new_stream(&pr->own_stream);
  const long long R = d.R;

  // --- data first: its upload (1 GB at 512 stations) runs while the host checks the row order ---
  d.x = dev_alloc<double2>((size_t)4 * R);
  pr->vis_stage = dev_alloc<double2>((size_t)4 * R);
  if (x) db_upload_vis(pr, x, d.x);

  // --- row order must be the canonical one ---
  std::vector<unsigned char> hflag(R);
  db_canonical_flags(N, Nbase, tilesz, barr, hflag.data());
  d.flag = dev_alloc<unsigned char>(R);
  DB_CHECK(cudaMemcpyAsync(d.flag, hflag.data(), R, cudaMemcpyHostToDevice, d.stream));
  db_stream_sync(d.stream);  // data and flags are up (hflag goes out of scope)

  // --- cluster / chunk tables ---
  d.h_clus = (ClusterDesc *)malloc(sizeof(ClusterDesc) * M);
  int mt = 0;
  for (int k = 0; k < M; k++) {
    d.h_clus[k].nchunk = carr[k].nchunk;
    d.h_clus[k].chunk0 = mt;
    mt += carr[k].nchunk;
  }
  if (mt != Mt) {
    fprintf(stderr, "dirac_b200: sum of nchunk (%d) != Mt (%d)\n", mt, Mt);
    exit(1);
  }
  d.h_chunk_poff = (int *)malloc(sizeof(int) * Mt);
  for (int k = 0; k < M; k++)
    for (int c = 0; c < carr[k].nchunk; c++) d.h_chunk_poff[d.h_clus[k].chunk0 + c] = carr[k].p[c];
  d.clus = dev_alloc<ClusterDesc>(M);
  d.chunk_poff = dev_alloc<int>(Mt);
  DB_CHECK(cudaMemcpy(d.clus, d.h_clus, sizeof(ClusterDesc) * M, cudaMemcpyHostToDevice));
  DB_CHECK(cudaMemcpy(d.chunk_poff, d.h_chunk_poff, sizeof(int) * Mt, cudaMemcpyHostToDevice));

  // --- tiles ---
  std::vector<TileDesc> tiles;
  db_build_tiles(N, tiles);
  d.ntile = (int)tiles.size();
  d.tiles = dev_alloc<TileDesc>(tiles.size());
  DB_CHECK(cudaMemcpy(d.tiles, tiles.data(), sizeof(TileDesc) * tiles.size(),
                      cudaMemcpyHostToDevice));

  {
    std::vector<short2> pq(Nbase);
    int b = 0;
    for (int p = 0; p < N - 1; p++)
      for (int q = p + 1; q < N; q++, b++) pq[b] = make_short2((short)p, (short)q);
    d.blpq = dev_alloc<short2>(Nbase);
    DB_CHECK(cudaMemcpy(d.blpq, pq.data(), sizeof(short2) * Nbase, cudaMemcpyHostToDevice));
  }

  // --- Jones, data, coherencies ---
  d.pp = dev_alloc<double>((size_t)d.npar);
  d.coh = dev_alloc<double2>((size_t)M * 4 * R);
  if (coh) {
    // chunked upload through a device staging buffer, transposed to planar on the device
    long long rows_per = (128ll << 20) / ((long long)M * 64);
    if (rows_per < 1) rows_per = 1;
    if (rows_per > R) rows_per = R;
    double2 *stage = dev_alloc<double2>((size_t)rows_per * M * 4);
    for (long long r0 = 0; r0 < R; r0 += rows_per) {
      int nr = (int)((R - r0 < rows_per) ? (R - r0) : rows_per);
      DB_CHECK(cudaMemcpyAsync(stage, coh + (size_t)r0 * M * 8, (size_t)nr * M * 64,
                               cudaMemcpyHostToDevice, d.stream));
      db_launch_coh_to_planar(stage, d.coh, r0, nr, M, R, d.stream);
      db_count_launch(1);
    }
    db_count_coh_host_bytes((size_t)R * M * 64);
    db_stream_sync(d.stream);
    db_free(stage);
  }

  // --- scratch ---
  const int nb2 = db_cluster_pass_nblocks(d.ntile, tilesz, 1);
  const int nb3 = db_stream_all_nblocks(Nbase, tilesz);
  pr->npartials = (nb2 > nb3 ? nb2 : nb3) + 1024;  // also covers the fixed-grid reductions
  pr->partials = dev_alloc<double>(pr->npartials);
  // scalars [0,64) followed by the LM mailbox (step, J^T e at two points, solver status): everything
  // the host needs after a trial comes back in ONE device-to-host copy
  d.scal = dev_alloc<double>(64 + 3 * 8 * (size_t)N + 8);
  DB_CHECK(cudaMemset(d.scal, 0, sizeof(double) * (64 + 3 * 8 * (size_t)N + 8)));
  DB_CHECK(cudaMallocHost((void **)&d.h_scal, (64 + 3 * 8 * (size_t)N + 8) * sizeof(double)));
  d.counters = dev_alloc<unsigned int>(16 + 1024);  // [0,16): grid reductions; then baseline groups
  DB_CHECK(cudaMemset(d.counters, 0, (16 + 1024) * sizeof(unsigned int)));
  pr->res = dev_alloc<double2>((size_t)4 * R);
  pr->g = dev_alloc<double>((size_t)d.npar);
  DB_CHECK(cudaGetLastError());
  return pr;
}

extern "C" void dirac_b200_destroy(dirac_b200_problem *pr) {
  if (!pr) return;
  DevProblem &d = pr->d;
  cudaStreamSynchronize(d.stream);
  db_lm_free(pr);
  db_rtr_free(pr);
  db_free(d.coh); db_free(d.x); db_free(d.flag); db_free(d.pp); db_free(d.clus);
  db_free(d.chunk_poff); db_free(d.tiles); db_free(d.blpq); db_free(d.scal); db_free(d.counters);
  db_free(pr->partials); db_free(pr->res); db_free(pr->g); db_free(pr->vis_stage);
  if (pr->pm) db_free(pr->pm);
  if (pr->xb) { db_free(pr->xb); db_free(pr->pp_start); }
  if (pr->E0) db_free(pr->E0);  // E1, E2 and poly_part live inside E0's allocation
  cudaFreeHost(d.h_scal);
  free(d.h_clus); free(d.h_chunk_poff);
  if (pr->own_stream) cudaStreamDestroy(d.stream);
  delete pr;
}

// host API-layout vector (8R doubles) -> planar device vector
void db_upload_vis(dirac_b200_problem *pr, const double *h, double2 *dst) {
  DevProblem &d = pr->d;
  DB_CHECK(cudaMemcpyAsync(pr->vis_stage, h, (size_t)d.R * 64, cudaMemcpyHostToDevice, d.stream));
  db_launch_vis_to_planar(pr->vis_stage, dst, d.R, d.stream);
  db_count_launch(1);
}
// planar device vector -> host API-layout vector
void db_download_vis(dirac_b200_problem *pr, const double2 *src, double *h) {
  DevProblem &d = pr->d;
  db_launch_vis_from_planar(src, pr->vis_stage, d.R, d.stream);
  db_count_launch(1);
  DB_CHECK(cudaMemcpyAsync(h, pr->vis_stage, (size_t)d.R * 64, cudaMemcpyDeviceToHost, d.stream));
  db_stream_sync(d.stream);
}

extern "C" void dirac_b200_set_data(dirac_b200_problem *pr, const double *x) {
  db_upload_vis(pr, x, pr->d.x);
  db_stream_sync(pr->d.stream);
}

void db_download_coh(const double2 *coh, double *x, int M, long long R, cudaStream_t st) {
  long long rows_per = (128ll << 20) / ((long long)M * 64);
  if (rows_per < 1) rows_per = 1;
  if (rows_per > R) rows_per = R;
  double2 *stage = dev_alloc<double2>((size_t)rows_per * M * 4);
  for (long long r0 = 0; r0 < R; r0 += rows_per) {
    int nr = (int)((R - r0 < rows_per) ? (R - r0) : rows_per);
    db_launch_coh_from_planar(coh, stage, r0, nr, M, R, st);
    db_count_launch(1);
    DB_CHECK(cudaMemcpyAsync(x + (size_t)r0 * M * 8, stage, (size_t)nr * M * 64,
                             cudaMemcpyDeviceToHost, st));
  }
  db_stream_sync(st);
  db_count_coh_host_bytes((size_t)R * M * 64);
  db_free(stage);
}

extern "C" void dirac_b200_get_coherencies(dirac_b200_problem *pr, double *coh) {
  db_download_coh(pr->d.coh, coh, pr->d.M, pr->d.R, pr->d.stream);
}

// ------------------------------------------------------------------------------------------------
// device-pointer primitives used by the solvers
// ------------------------------------------------------------------------------------------------
// model/residual/cost over all clusters at the Jones currently in d.pp; returns after queuing;
// the cost lands in d.scal[slot] (device)
void db_predict_dev(dirac_b200_problem *pr, const double *pp_dev, double2 *out, int out_mode,
                    int cost_mode, double nu, int slot) {
  DevProblem &d = pr->d;
  StreamAllArgs a;
  memset(&a, 0, sizeof(a));
  a.coh = d.coh; a.x = d.x; a.flag = d.flag; a.pp = pp_dev; a.clus = d.clus;
  a.chunk_poff = d.chunk_poff; a.blpq = d.blpq; a.out = out; a.partials = pr->partials;
  a.cost = d.scal + slot; a.counter = d.counters; a.R = d.R; a.N = d.N; a.Nbase = d.Nbase;
  a.tilesz = d.tilesz; a.M = d.M; a.out_mode = out_mode; a.cost_mode = cost_mode;
  a.inv_nu = (nu > 0.0) ? 1.0 / nu : 0.0;
  if (pr->world > 1) {
    // cluster-sharded: partial model of the local clusters, summed over the ranks, then residual
    // and cost from the sum (identical on every rank)
    if (!pr->pm) pr->pm = dev_alloc<double2>((size_t)4 * d.R);
    a.out = pr->pm; a.out_mode = 2; a.cost_mode = 0;
    db_prof_begin(0, (double)d.R * (64.0 * d.M + 65.0 + 64.0), d.stream);
    db_launch_predict_tma(&a, d.stream);
    db_prof_end(d.stream);
    db_allreduce(pr, pr->pm, 8 * d.R);
    db_launch_residual_cost(d.x, pr->pm, out, 4 * d.R, out ? out_mode : 0, cost_mode, a.inv_nu,
                            pr->partials, d.scal + slot, d.counters, d.stream);
    db_count_launch(2);
    return;
  }
  db_prof_begin(0, (double)d.R * (64.0 * d.M + 65.0 + (out_mode ? 64.0 : 0.0)), d.stream);
  db_launch_predict_tma(&a, d.stream);
  db_prof_end(d.stream);
  db_count_launch(1);
}

double db_read_scalar(dirac_b200_problem *pr, int slot) {
  DevProblem &d = pr->d;
  DB_CHECK(cudaMemcpyAsync(d.h_scal + slot, d.scal + slot, sizeof(double), cudaMemcpyDeviceToHost,
                           d.stream));
  db_stream_sync(d.stream);
  return d.h_scal[slot];
}

// gradient over all clusters from the residual in pr->res; g_dev (8*N*Mt) is overwritten
void db_grad_dev(dirac_b200_problem *pr, const double *pp_dev, double *g_dev, int robust,
                 double nu) {
  DevProblem &d = pr->d;
  DB_CHECK(cudaMemsetAsync(g_dev, 0, sizeof(double) * d.npar, d.stream));
  GradArgs a;
  a.coh = d.coh; a.res = pr->res; a.flag = d.flag; a.pp = pp_dev; a.clus = d.clus;
  a.chunk_poff = d.chunk_poff; a.tiles = d.tiles; a.g = g_dev; a.R = d.R; a.N = d.N;
  a.Nbase = d.Nbase; a.tilesz = d.tilesz; a.M = d.M; a.robust = robust; a.nu = nu;
  // sign conventions of the reference: Gaussian g = -2 Re(conj(f-d) . df) (robust_lbfgs.c:554),
  // robust g = +2 (f-d) df/(nu+(f-d)^2) (robust_lbfgs.c:286-299); here e = d-f
  a.scale = robust ? -2.0 : 2.0;
  db_prof_begin(1, (double)d.R * (64.0 * d.M + 65.0) + 64.0 * d.N * d.Mt, d.stream);
  db_launch_grad_tma(&a, d.ntile, d.stream);
  db_prof_end(d.stream);
  db_count_launch(1);
  // sharded: every rank filled the blocks of its own clusters; the sum is the full gradient
  db_allreduce(pr, g_dev, d.npar);
}

// Student's-t cost of the rows [r_lo, r_hi) alone at pp_dev (robust_cost_func_batch,
// robust_batchmode_lbfgs.c:822-846): only the timeslots that overlap the window are streamed, rows of
// the first and last of them outside it are skipped.  out != null: the residual e = x - V of the
// window's rows is written there (the other rows of out are left as they are).  Returns the cost.
double db_cost_window_dev(dirac_b200_problem *pr, const double *pp_dev, double2 *out, double nu,
                          long long r_lo, long long r_hi) {
  DevProblem &d = pr->d;
  if (r_lo < 0) r_lo = 0;
  if (r_hi > d.R) r_hi = d.R;
  if (r_hi <= r_lo) return 0.0;  // an empty window of the batch table
  const long long t_lo = r_lo / d.Nbase, t_hi = (r_hi + d.Nbase - 1) / d.Nbase;
  const long long r0 = t_lo * d.Nbase, len = r_hi - r_lo;
  StreamAllArgs a;
  memset(&a, 0, sizeof(a));
  a.coh = d.coh + r0; a.x = d.x + r0; a.flag = d.flag + r0; a.pp = pp_dev; a.clus = d.clus;
  a.chunk_poff = d.chunk_poff; a.blpq = d.blpq; a.partials = pr->partials;
  a.cost = d.scal; a.counter = d.counters; a.R = d.R; a.N = d.N; a.Nbase = d.Nbase;
  a.tilesz = (int)(t_hi - t_lo); a.M = d.M; a.row0 = r0;
  a.w_lo = r_lo - r0; a.w_hi = r_hi - r0;
  a.inv_nu = (nu > 0.0) ? 1.0 / nu : 0.0;
  const double bytes = (double)len * (64.0 * d.M + 65.0 + (out ? 64.0 : 0.0));
  if (pr->world <= 1) {
    a.out = out ? out + r0 : nullptr;
    a.out_mode = out ? 1 : 0;
    a.cost_mode = 2;
    db_prof_begin(0, bytes, d.stream);
    db_launch_cost_window_tma(&a, d.stream);
    db_prof_end(d.stream);
    db_count_launch(1);
    return db_read_scalar(pr, 0);
  }
  // cluster-sharded: partial model of the local clusters over the window, its 8 len doubles summed
  // over the ranks, then residual and cost of each polarisation plane from the sum (identical on
  // every rank; the four plane costs are added on the host in plane order)
  if (!pr->pm) pr->pm = dev_alloc<double2>((size_t)4 * d.R);
  a.out = pr->pm + r0; a.out_mode = 2; a.cost_mode = 0;
  db_prof_begin(0, bytes, d.stream);
  db_launch_cost_window_tma(&a, d.stream);
  db_prof_end(d.stream);
  for (int c = 0; c < 4; c++) db_allreduce(pr, pr->pm + (long long)c * d.R + r_lo, 2 * len);
  for (int c = 0; c < 4; c++) {
    const long long off = (long long)c * d.R + r_lo;
    db_launch_residual_cost(d.x + off, pr->pm + off, out ? out + off : nullptr, len, out ? 1 : 0, 2,
                            a.inv_nu, pr->partials, d.scal + 32 + c, d.counters, d.stream);
  }
  db_count_launch(5);
  DB_CHECK(cudaMemcpyAsync(d.h_scal + 32, d.scal + 32, 4 * sizeof(double), cudaMemcpyDeviceToHost,
                           d.stream));
  db_stream_sync(d.stream);
  return ((d.h_scal[32] + d.h_scal[33]) + d.h_scal[34]) + d.h_scal[35];
}

// gradient of the Student's-t cost over the rows [r_lo, r_hi) alone, from the residual of those rows
// in pr->res, with the sign of the reference's minibatch gradient (func_grad_robust_batch,
// robust_batchmode_lbfgs.c:489: -2 sum xr dV/(nu + xr^2) with xr = model - data, the NEGATED true
// gradient); g_dev (npar) is overwritten
void db_grad_window_dev(dirac_b200_problem *pr, const double *pp_dev, double *g_dev, double nu,
                        long long r_lo, long long r_hi) {
  DevProblem &d = pr->d;
  if (r_lo < 0) r_lo = 0;
  if (r_hi > d.R) r_hi = d.R;
  DB_CHECK(cudaMemsetAsync(g_dev, 0, sizeof(double) * d.npar, d.stream));
  if (r_hi <= r_lo) return;  // (the same window on every rank)
  GradArgs a;
  memset(&a, 0, sizeof(a));
  a.coh = d.coh; a.res = pr->res; a.flag = d.flag; a.pp = pp_dev; a.clus = d.clus;
  a.chunk_poff = d.chunk_poff; a.tiles = d.tiles; a.g = g_dev; a.R = d.R; a.N = d.N;
  a.Nbase = d.Nbase; a.tilesz = d.tilesz; a.M = d.M; a.robust = 1; a.nu = nu;
  a.scale = 2.0;  // e = d - f:  -2 (f - d) = +2 e
  db_prof_begin(1, (double)(r_hi - r_lo) * (64.0 * d.M + 65.0) + 64.0 * d.N * d.Mt, d.stream);
  db_launch_grad_window_tma(&a, d.ntile, r_lo, r_hi, d.stream);
  db_prof_end(d.stream);
  db_count_launch(1);
  db_allreduce(pr, g_dev, d.npar);
}

// ------------------------------------------------------------------------------------------------
// thin C-ABI
// ------------------------------------------------------------------------------------------------
extern "C" double dirac_b200_predict(dirac_b200_problem *pr, const double *pp, double *out,
                                     int out_mode, int cost_mode, double nu) {
  DevProblem &d = pr->d;
  DB_CHECK(cudaMemcpyAsync(d.pp, pp, sizeof(double) * d.npar, cudaMemcpyHostToDevice,
                           d.stream));
  if (!out) out_mode = 0;
  db_predict_dev(pr, d.pp, pr->res, out_mode, cost_mode, nu, 0);
  double c = 0.0;
  if (cost_mode) c = db_read_scalar(pr, 0);
  if (out_mode) db_download_vis(pr, pr->res, out);
  db_stream_sync(d.stream);
  DB_CHECK(cudaGetLastError());
  return c;
}

extern "C" void dirac_b200_grad(dirac_b200_problem *pr, const double *pp, double *g, int robust,
                                double nu) {
  DevProblem &d = pr->d;
  DB_CHECK(cudaMemcpyAsync(d.pp, pp, sizeof(double) * d.npar, cudaMemcpyHostToDevice,
                           d.stream));
  db_predict_dev(pr, d.pp, pr->res, 1, 0, 0.0, 0);  // residual e = x - V
  db_grad_dev(pr, d.pp, pr->g, robust, nu);
  DB_CHECK(cudaMemcpyAsync(g, pr->g, sizeof(double) * d.npar, cudaMemcpyDeviceToHost,
                           d.stream));
  db_stream_sync(d.stream);
  DB_CHECK(cudaGetLastError());
}

extern "C" double dirac_b200_cost_window(dirac_b200_problem *pr, const double *pp, long long row0,
                                         long long nrows, double nu) {
  DevProblem &d = pr->d;
  DB_CHECK(cudaMemcpyAsync(d.pp, pp, sizeof(double) * d.npar, cudaMemcpyHostToDevice, d.stream));
  const double c = db_cost_window_dev(pr, d.pp, nullptr, nu, row0, row0 + nrows);
  db_stream_sync(d.stream);
  DB_CHECK(cudaGetLastError());
  return c;
}

extern "C" void dirac_b200_grad_window(dirac_b200_problem *pr, const double *pp, double *g,
                                       long long row0, long long nrows, double nu) {
  DevProblem &d = pr->d;
  DB_CHECK(cudaMemcpyAsync(d.pp, pp, sizeof(double) * d.npar, cudaMemcpyHostToDevice, d.stream));
  db_cost_window_dev(pr, d.pp, pr->res, nu, row0, row0 + nrows);  // residual of the window's rows
  db_grad_window_dev(pr, d.pp, pr->g, nu, row0, row0 + nrows);
  DB_CHECK(cudaMemcpyAsync(g, pr->g, sizeof(double) * d.npar, cudaMemcpyDeviceToHost, d.stream));
  db_stream_sync(d.stream);
  DB_CHECK(cudaGetLastError());
}
