// Host side of the diffuse-cluster coherencies: recalculate_diffuse_coherencies with the reference's
// signature (Dirac_radio.h:228, diffuse_predict.c:295-586) and dirac_b200_diffuse_coherencies on a
// resident problem.  The host packs the sources (Stokes-weighted modes, product tensors) and the
// per-station spatial modes; kernels_diffuse.cu does the products and the rows.
#include <string.h>
#include <vector>

#include "../../include/dirac_b200.h"
#include "coh.h"
#include "diffuse_math.cuh"
#include "problem.h"

namespace {

struct DiffusePlan {
  std::vector<DiffuseSource> src;
  std::vector<double2> scoh, Zt;
  std::vector<double> cf;
  long long ncjq = 0;
  int max_n0 = 0;
};

void refuse_tensor(int L, int M, int N) {
  fprintf(stderr, "dirac_b200: the shapelet product tensor of orders (%d, %d, %d) leaves the double "
                  "range\n", L, M, N);
  exit(1);
}

// the sources of cluster c and the spatial model Z (2N x 2G, column major) as the kernels take them
void diffuse_plan(const clus_source_t &c, int N, int sh_n0, double sh_beta, const double2 *Z,
                  DiffusePlan *pl) {
  if (sh_n0 < 1 || sh_n0 > DIFFUSE_MAX_ORDER) {
    fprintf(stderr, "dirac_b200: spatial model order %d is outside 1..%d\n", sh_n0, DIFFUSE_MAX_ORDER);
    exit(1);
  }
  const int G = sh_n0 * sh_n0;
  // Zt: rows 2n, 2n+1 of Z as station n's modes, each 2x2 block transposed (:374-383)
  pl->Zt.resize((size_t)4 * G * N);
  for (int n = 0; n < N; n++)
    for (int g = 0; g < G; g++)
      for (int c2 = 0; c2 < 4; c2++)
        pl->Zt[((size_t)n * G + g) * 4 + c2] = Z[(size_t)(2 * n + (c2 & 1)) + (size_t)(2 * g + (c2 >> 1)) * 2 * N];
  for (int s = 0; s < c.N; s++) {
    if (c.stype[s] != STYPE_SHAPELET) {  // (:393-397)
      fprintf(stderr, "%s: %d: invalid source type, must be shapelet\n", __FILE__, __LINE__);
      exit(1);
    }
    const exinfo_shapelet *sp = (const exinfo_shapelet *)c.ex[s];
    const int n0 = sp->n0;
    if (n0 < 1 || n0 > COH_SHAPELET_MAX_N0) {
      fprintf(stderr, "dirac_b200: shapelet order %d of diffuse source %d is outside 1..%d\n", n0, s,
              COH_SHAPELET_MAX_N0);
      exit(1);
    }
    DiffuseSource d;
    memset(&d, 0, sizeof(d));
    d.ll = c.ll[s]; d.mm = c.mm[s]; d.nn = c.nn[s]; d.beta = sp->beta; d.n0 = n0;
    // Stokes-weighted modes [I+Q, U+iV, U-iV, I-Q] modes[mode] (:437-449)
    d.scoh = (long long)pl->scoh.size();
    const double2 xxyy[4] = {make_double2(c.sI[s] + c.sQ[s], 0.0), make_double2(c.sU[s], c.sV[s]),
                             make_double2(c.sU[s], -c.sV[s]), make_double2(c.sI[s] - c.sQ[s], 0.0)};
    for (int m = 0; m < n0 * n0; m++)
      for (int k = 0; k < 4; k++)
        pl->scoh.push_back(make_double2(xxyy[k].x * sp->modes[m], xxyy[k].y * sp->modes[m]));
    // product tensors at the image-plane scale beta / 2 pi (:403, :411, :487)
    const double bimg = sp->beta / (2.0 * M_PI);
    d.cf1 = (long long)pl->cf.size();
    pl->cf.resize(pl->cf.size() + (size_t)n0 * n0 * sh_n0);
    if (diffuse_product_tensor(n0, n0, sh_n0, bimg, bimg, sh_beta, pl->cf.data() + d.cf1))
      refuse_tensor(n0, n0, sh_n0);
    d.cf2 = (long long)pl->cf.size();
    pl->cf.resize(pl->cf.size() + (size_t)n0 * sh_n0 * n0);
    if (diffuse_product_tensor(n0, sh_n0, n0, bimg, sh_beta, bimg, pl->cf.data() + d.cf2))
      refuse_tensor(n0, sh_n0, n0);
    d.cjq = pl->ncjq;
    pl->ncjq += (long long)4 * n0 * n0 * N;
    if (n0 > pl->max_n0) pl->max_n0 = n0;
    pl->src.push_back(d);
  }
}

// a.pairs / rows / u, v, w / coh / R set by the caller; runs the kernels and waits for them
void diffuse_run(DeviceScope &ds, const DiffusePlan &pl, DiffuseArgs a) {
  a.src = ds.upload(pl.src); a.ns = (int)pl.src.size(); a.scoh = ds.upload(pl.scoh);
  a.Zt = ds.upload(pl.Zt); a.cf = ds.upload(pl.cf); a.cjq = ds.alloc<double2>(pl.ncjq);
  db_launch_diffuse(&a, pl.max_n0, ds.st);
  ds.sync();
}

void check_cluster(int cid, int M) {
  if (cid < 0 || cid >= M) {  // (:388-391)
    fprintf(stderr, "%s: %d: invalid cluster id\n", __FILE__, __LINE__);
    exit(1);
  }
}

}  // namespace

// Dirac_radio.h:228.  Nbase counts rows (baselines x timeslots), in any order; x is [row][M][4]
// complex and only its cluster cid is written, flagged rows included.  tdelta, dec0, uvmin, uvmax,
// Nt and use_cuda are not used: the computation always runs on the GPU, in fp64.
extern "C" int recalculate_diffuse_coherencies(double *u, double *v, double *w, double *x, int N,
                                               int Nbase, baseline_t *barr, clus_source_t *carr,
                                               int M, double freq0, double fdelta, double tdelta,
                                               double dec0, double uvmin, double uvmax, int cid,
                                               int sh_n0, double sh_beta, double *Z, int Nt,
                                               int use_cuda) {
  (void)tdelta; (void)dec0; (void)uvmin; (void)uvmax; (void)Nt; (void)use_cuda;
  check_cluster(cid, M);
  DiffusePlan pl;
  diffuse_plan(carr[cid], N, sh_n0, sh_beta, reinterpret_cast<const double2 *>(Z), &pl);
  if (pl.src.empty() || Nbase <= 0) return 0;  // no source: the slot is left as it is
  DeviceScope ds;
  const long long R = Nbase;
  // rows grouped by station pair (counting sort); rows naming a station outside 0..N-1 share one
  // group that gets zeros
  const long long NN = (long long)N * N;
  std::vector<long long> cnt(NN + 2, 0), key(R);
  for (long long r = 0; r < R; r++) {
    const int p = barr[r].sta1, q = barr[r].sta2;
    key[r] = (p >= 0 && p < N && q >= 0 && q < N) ? (long long)p * N + q : NN;
    cnt[key[r] + 1]++;
  }
  for (long long k = 0; k < NN + 1; k++) cnt[k + 1] += cnt[k];
  std::vector<long long> rows(R), pos(cnt.begin(), cnt.end() - 1);
  for (long long r = 0; r < R; r++) rows[pos[key[r]]++] = r;
  std::vector<short2> pairs;
  std::vector<long long> row_off;
  for (long long k = 0; k <= NN; k++) {
    if (cnt[k + 1] == cnt[k]) continue;
    pairs.push_back(k < NN ? make_short2((short)(k / N), (short)(k % N)) : make_short2(-1, -1));
    row_off.push_back(cnt[k]);
  }
  row_off.push_back(R);
  DiffuseArgs a;
  memset(&a, 0, sizeof(a));
  a.N = N; a.sh = sh_n0;
  a.pairs = ds.upload(pairs); a.npairs = (int)pairs.size();
  a.row_off = ds.upload(row_off); a.rows = ds.upload(rows);
  a.u = ds.upload(u, R); a.v = ds.upload(v, R); a.w = ds.upload(w, R);
  a.freq0 = freq0; a.fdelta2 = fdelta * 0.5; a.R = R;
  a.coh = ds.alloc<double2>(4 * R);
  diffuse_run(ds, pl, a);
  // only cluster cid's slice comes back: planar [4][R] -> x[row][cid][4]
  std::vector<double2> h((size_t)4 * R);
  DB_CHECK(cudaMemcpy(h.data(), a.coh, sizeof(double2) * 4 * R, cudaMemcpyDeviceToHost));
  double2 *X = reinterpret_cast<double2 *>(x);
  for (long long r = 0; r < R; r++)
    for (int c = 0; c < 4; c++) X[((size_t)r * M + cid) * 4 + c] = h[(size_t)c * R + r];
  return 0;
}

// the same computation into local cluster cid of a resident problem; the coherencies stay on the device
extern "C" int dirac_b200_diffuse_coherencies(dirac_b200_problem *pr, const double *u, const double *v,
                                              const double *w, const clus_source_t *carr, double freq0,
                                              double fdelta, int cid, int sh_n0, double sh_beta,
                                              const double *Z) {
  DevProblem &d = pr->d;
  check_cluster(cid, d.M);
  DiffusePlan pl;
  diffuse_plan(carr[cid], d.N, sh_n0, sh_beta, reinterpret_cast<const double2 *>(Z), &pl);
  if (pl.src.empty()) return 0;
  DiffuseArgs a;
  memset(&a, 0, sizeof(a));
  a.N = d.N; a.sh = sh_n0;
  a.pairs = d.blpq; a.npairs = d.Nbase; a.ntime = d.tilesz; a.Nbase = d.Nbase;
  DeviceScope ds(d.stream);
  a.u = ds.upload(u, d.R); a.v = ds.upload(v, d.R); a.w = ds.upload(w, d.R);
  a.freq0 = freq0; a.fdelta2 = fdelta * 0.5; a.R = d.R;
  a.coh = d.coh + (size_t)cid * 4 * d.R;
  diffuse_run(ds, pl, a);
  // the Gram tensors cached for LM belong to the old coherencies (every solve also rebuilds them)
  if (pr->lm.ready) memset(pr->lm.T_valid, 0, d.Mt);
  return 0;
}
