// Host flow of calculate_diagnostics_gpu (diagnostics.c:620-1182 of the reference): the residual and the
// channel-0 coherencies of every cluster, then per cluster the Hessian and right-hand side, the
// conditioning, an LU solve, the sum over clusters of the residual derivatives dR and the
// eigenvalues of its four correlations.  One DeviceScope per call; everything stays on the device
// until x goes back.
#include <math.h>
#include <string.h>
#include <vector>

#include <cusolverDn.h>

#include "../../include/dirac_b200.h"
#include "influence.h"
#include "problem.h"

#define INFL_CS(call)                                                                         \
  do {                                                                                        \
    cusolverStatus_t s__ = (call);                                                            \
    if (s__ != CUSOLVER_STATUS_SUCCESS) {                                                     \
      fprintf(stderr, "dirac_b200: cuSOLVER status %d at %s:%d\n", (int)s__, __FILE__, __LINE__); \
      exit(1);                                                                                \
    }                                                                                         \
  } while (0)

namespace {

// the stations of every baseline index, checked on every timeslot, and the baselines of every
// station (CSR, 2*b + side); false with a message when the rows do not have that structure
bool station_tables(const char *fn, const baseline_t *barr, int N, int Nbase, int tilesz,
                    std::vector<int> &sta1, std::vector<int> &sta2, std::vector<int> &st_off,
                    std::vector<int> &st_bl) {
  sta1.resize(Nbase); sta2.resize(Nbase);
  std::vector<char> seen((size_t)N * N, 0);
  for (int b = 0; b < Nbase; b++) {
    const int p = barr[b].sta1, q = barr[b].sta2;
    if (p < 0 || q < 0 || p >= N || q >= N || p == q || seen[(size_t)p * N + q] || seen[(size_t)q * N + p]) {
      fprintf(stderr, "%s: baseline %d joins stations (%d, %d): every baseline must join two distinct "
                      "stations in [0, %d), each pair once\n", fn, b, p, q, N);
      return false;
    }
    seen[(size_t)p * N + q] = 1;
    sta1[b] = p; sta2[b] = q;
  }
  for (long long n = Nbase; n < (long long)Nbase * tilesz; n++) {
    const int b = (int)(n % Nbase);
    if (barr[n].sta1 != sta1[b] || barr[n].sta2 != sta2[b]) {
      fprintf(stderr, "%s: row %lld joins stations (%d, %d), row %d of the first timeslot (%d, %d): "
                      "every timeslot must list the baselines in the same order\n", fn, n,
              barr[n].sta1, barr[n].sta2, b, sta1[b], sta2[b]);
      return false;
    }
  }
  st_off.assign(N + 1, 0);
  for (int b = 0; b < Nbase; b++) { st_off[sta1[b] + 1]++; st_off[sta2[b] + 1]++; }
  for (int s = 0; s < N; s++) st_off[s + 1] += st_off[s];
  st_bl.resize(2 * (size_t)Nbase);
  std::vector<int> fill(st_off.begin(), st_off.end() - 1);
  for (int b = 0; b < Nbase; b++) {
    st_bl[fill[sta1[b]]++] = 2 * b;
    st_bl[fill[sta2[b]]++] = 2 * b + 1;
  }
  return true;
}

struct InflTables {
  std::vector<int> sta1, sta2, st_off, st_bl;
  std::vector<unsigned char> flag;
};

// InflArgs of M clusters on ds, with H, AdV and S allocated; coh, res, p and the chunk tables are the
// caller's
InflArgs infl_args(DeviceScope &ds, const InflTables &t, int N, int Nbase, int tilesz, int M) {
  InflArgs a;
  memset(&a, 0, sizeof(a));
  a.N = N; a.Nbase = Nbase; a.T = tilesz; a.M = M; a.R = (long long)Nbase * tilesz;
  a.sta1 = ds.upload(t.sta1); a.sta2 = ds.upload(t.sta2);
  a.st_off = ds.upload(t.st_off); a.st_bl = ds.upload(t.st_bl);
  a.flag = ds.upload(t.flag);
  const size_t n4 = 4 * (size_t)N;
  a.H = ds.alloc<double2>(n4 * n4 * M);
  a.AdV = ds.alloc<double2>(n4 * Nbase * M);
  a.S = ds.alloc<double2>((size_t)Nbase * 4 * M);
  a.dR = ds.alloc<double2>((size_t)Nbase * Nbase * 4);
  return a;
}

void geev_buffer(cusolverDnHandle_t cs, cusolverDnParams_t prm, int n, size_t *dev, size_t *host) {
  INFL_CS(cusolverDnXgeev_bufferSize(cs, prm, CUSOLVER_EIG_MODE_NOVECTOR, CUSOLVER_EIG_MODE_NOVECTOR, n,
                                     CUDA_C_64F, nullptr, n, CUDA_C_64F, nullptr, CUDA_C_64F, nullptr, 1,
                                     CUDA_C_64F, nullptr, 1, CUDA_C_64F, dev, host));
}

}  // namespace

extern "C" int calculate_diagnostics_gpu(double *u, double *v, double *w, double *p, double *x, int N,
                                         int Nbase, int tilesz, baseline_t *barr, clus_source_t *carr,
                                         int M, double *freqs, int Nchan, double fdelta, double tdelta,
                                         double dec0, int bf_type, double b_ra0, double b_dec0,
                                         double ph_ra0, double ph_dec0, double ph_freq0,
                                         double *longitude, double *latitude, double *time_utc,
                                         int *Nelem, double **xx, double **yy, double **zz,
                                         elementcoeff *ecoeff, int dobeam, double *rho, double *Bpoly,
                                         double *Bi, int Mt, int Npoly, int Nf, int Nt) {
  (void)tdelta; (void)dec0; (void)Mt; (void)Nf; (void)Nt;
  const char *fn = "calculate_diagnostics_gpu";
  if (N < 2 || M < 1 || tilesz < 1 || Nchan < 1 || Nbase != N * (N - 1) / 2) {
    fprintf(stderr, "%s: N = %d, Nbase = %d, tilesz = %d, M = %d, Nchan = %d: the call takes N >= 2, "
                    "Nbase = N(N-1)/2 and positive tilesz, M and Nchan\n", fn, N, Nbase, tilesz, M, Nchan);
    return -1;
  }
  for (int k = 0; k < M; k++)
    if (carr[k].nchunk < 1) {
      fprintf(stderr, "%s: cluster %d has nchunk = %d\n", fn, k, carr[k].nchunk);
      return -1;
    }
  InflTables tb;
  if (!station_tables(fn, barr, N, Nbase, tilesz, tb.sta1, tb.sta2, tb.st_off, tb.st_bl)) return -1;
  BeamSpec beam = {bf_type, b_ra0, b_dec0, ph_ra0, ph_dec0, ph_freq0, longitude, latitude, time_utc,
                   tilesz, Nelem, xx, yy, zz, ecoeff, dobeam};
  if (beam_refused(fn, beam, N, Nchan)) return -1;
  // the consensus term of the Hessian's diagonal (diagnostics.c:717-751): 0.5 rho_k Fd1 with
  // Fd = 1 - Bpoly^T Bi_k Bpoly and Fd1 = Fd^2 (1 + Fd^2 / (1 - Fd^2))
  std::vector<double> hadd;
  if (rho && Bpoly && Bi) {
    hadd.resize(M);
    for (int k = 0; k < M; k++) {
      const double *B = Bi + (size_t)k * Npoly * Npoly;
      double bb = 0.0;
      for (int i = 0; i < Npoly; i++) {
        double s = 0.0;
        for (int j = 0; j < Npoly; j++) s += B[i + (size_t)j * Npoly] * Bpoly[j];
        bb += Bpoly[i] * s;
      }
      const double Fd = 1.0 - bb, Fdd = Fd * Fd;
      hadd[k] = 0.5 * rho[k] * (Fdd * (1.0 + Fdd / (1.0 - Fdd)));
    }
  }
  const long long R = (long long)Nbase * tilesz;
  tb.flag.resize(R);
  for (long long n = 0; n < R; n++) tb.flag[n] = barr[n].flag ? 1 : 0;

  require_gpu();
  const int n4 = 4 * N;
  // everything the call allocates, before any of it; the solver workspaces are asked for only when
  // the rest fits
  double need = 16.0 * ((double)Nchan * R * 4 + (double)M * 4 * R + (double)M * n4 * n4 +
                        (double)M * n4 * Nbase + (double)M * Nbase * 4 + 4.0 * Nbase * Nbase +
                        4.0 * Nbase) + 8.0 * n4 + 64.0 * (R + Nbase);
  size_t free_b = 0, total_b = 0;
  DB_CHECK(cudaMemGetInfo(&free_b, &total_b));
  cusolverDnHandle_t cs = nullptr;
  cusolverDnParams_t prm = nullptr;
  size_t geev_dev = 0, geev_host = 0, lu_dev = 0, lu_host = 0;
  if (need <= (double)free_b) {
    INFL_CS(cusolverDnCreate(&cs));
    INFL_CS(cusolverDnCreateParams(&prm));
    geev_buffer(cs, prm, Nbase, &geev_dev, &geev_host);
    INFL_CS(cusolverDnXgetrf_bufferSize(cs, prm, n4, n4, CUDA_C_64F, nullptr, n4, CUDA_C_64F, &lu_dev,
                                        &lu_host));
    need += (double)(geev_dev > lu_dev ? geev_dev : lu_dev);
  }
  if (need > (double)free_b) {
    fprintf(stderr, "%s: N = %d stations, M = %d clusters need %.3g GB of device memory (the four "
                    "Nbase x Nbase dR matrices alone %.3g GB), %.3g GB are free\n", fn, N, M,
            need / 1e9, 64.0 * Nbase * (double)Nbase / 1e9, (double)free_b / 1e9);
    if (prm) cusolverDnDestroyParams(prm);
    if (cs) cusolverDnDestroy(cs);
    return -1;
  }
  {
    DeviceScope ds;
    INFL_CS(cusolverDnSetStream(cs, ds.st));
    const int rec_call = db_prof_open(23, 0.0, ds.st);  // kind 23: the device work of the call
    const int rec_model = db_prof_open(18, 0.0, ds.st);  // kind 18: the model stage
    DiagModel md;
    db_diagnostics_model(ds, u, v, w, p, x, N, Nbase, tilesz, barr, carr, M, freqs, Nchan, fdelta, &beam,
                         &md);
    db_prof_close(rec_model, ds.st);
    InflArgs a = infl_args(ds, tb, N, Nbase, tilesz, M);
    a.coh = md.coh; a.res = md.x; a.p = md.p;
    a.clus_nchunk = md.clus_nchunk; a.clus_chunk0 = md.clus_chunk0; a.chunk_poff = md.chunk_poff;
    a.X = a.AdV;
    const double *hadd_d = hadd.empty() ? nullptr : ds.upload(hadd);
    db_prof_begin(19, 0.0, ds.st);  // kind 19: Hessian and right-hand side
    db_launch_infl_assemble(&a, ds.st);
    db_launch_infl_condition(&a, hadd_d, ds.st);
    db_prof_end(ds.st);
    db_count_launch(3);
    int64_t *piv = ds.alloc<int64_t>(n4);
    int *info = ds.alloc<int>(M + 4);
    void *work = ds.alloc<char>(lu_dev > geev_dev ? lu_dev : geev_dev);
    std::vector<char> hwork(lu_host > geev_host ? lu_host : geev_host);
    db_prof_begin(20, 0.0, ds.st);  // kind 20: the LU solves
    for (int k = 0; k < M; k++) {
      double2 *Hk = a.H + (size_t)k * n4 * n4;
      double2 *Bk = a.AdV + (size_t)k * n4 * Nbase;
      INFL_CS(cusolverDnXgetrf(cs, prm, n4, n4, CUDA_C_64F, Hk, n4, piv, CUDA_C_64F, work, lu_dev,
                               hwork.data(), lu_host, info + k));
      INFL_CS(cusolverDnXgetrs(cs, prm, CUBLAS_OP_N, n4, Nbase, CUDA_C_64F, Hk, n4, piv, CUDA_C_64F, Bk,
                               n4, info + k));
    }
    db_prof_end(ds.st);
    db_prof_begin(21, 64.0 * Nbase * (double)Nbase, ds.st);  // kind 21: dR
    db_launch_infl_dr(&a, ds.st);
    db_prof_end(ds.st);
    db_count_launch(1);
    double2 *W = ds.alloc<double2>(4 * (size_t)Nbase);
    db_prof_begin(22, 0.0, ds.st);  // kind 22: the four eigenvalue problems
    for (int c = 0; c < 4; c++)
      INFL_CS(cusolverDnXgeev(cs, prm, CUSOLVER_EIG_MODE_NOVECTOR, CUSOLVER_EIG_MODE_NOVECTOR, Nbase,
                              CUDA_C_64F, a.dR + (size_t)c * Nbase * Nbase, Nbase, CUDA_C_64F,
                              W + (size_t)c * Nbase, CUDA_C_64F, nullptr, 1, CUDA_C_64F, nullptr, 1,
                              CUDA_C_64F, work, geev_dev, hwork.data(), geev_host, info + M + c));
    db_prof_end(ds.st);
    db_launch_infl_eigs(W, md.x, Nbase, tilesz, ds.st);
    db_count_launch(1);
    db_prof_close(rec_call, ds.st);
    std::vector<int> hinfo(M + 4);
    DB_CHECK(cudaMemcpyAsync(hinfo.data(), info, sizeof(int) * (M + 4), cudaMemcpyDeviceToHost, ds.st));
    DB_CHECK(cudaMemcpyAsync(x, md.x, sizeof(double2) * Nchan * R * 4, cudaMemcpyDeviceToHost, ds.st));
    ds.sync();
    for (int k = 0; k < M; k++)
      if (hinfo[k]) fprintf(stderr, "%s: cluster %d: the LU of the Hessian reports info %d\n", fn, k, hinfo[k]);
    for (int c = 0; c < 4; c++)
      if (hinfo[M + c]) fprintf(stderr, "%s: correlation %d: geev reports info %d\n", fn, c, hinfo[M + c]);
  }
  cusolverDnDestroyParams(prm);
  cusolverDnDestroy(cs);
  return 0;
}

// TEST HOOK (not in the headers): the kernels of one cluster on host arrays.  coh and res: channel 0,
// [R][8]; p: [nchunk][N][8]; X: 4N x Nbase complex, column major.  Out: the Hessian before the
// conditioning (4N x 4N complex), AdV (4N x Nbase complex) and the dR of X ([4][Nbase][Nbase]
// complex, column major).  Returns 0, or -1 when the rows are refused.
extern "C" int dirac_b200_diagnostics_eval(int N, int Nbase, int tilesz, const baseline_t *barr,
                                           const double *p, int nchunk, const double *coh,
                                           const double *res, const double *X, double *hess,
                                           double *AdV, double *dR) {
  const char *fn = "dirac_b200_diagnostics_eval";
  if (N < 2 || tilesz < 1 || nchunk < 1 || Nbase != N * (N - 1) / 2) return -1;
  InflTables tb;
  if (!station_tables(fn, barr, N, Nbase, tilesz, tb.sta1, tb.sta2, tb.st_off, tb.st_bl)) return -1;
  const long long R = (long long)Nbase * tilesz;
  tb.flag.resize(R);
  for (long long n = 0; n < R; n++) tb.flag[n] = barr[n].flag ? 1 : 0;
  require_gpu();
  std::vector<int> nch(1, nchunk), ch0(1, 0), poff(nchunk);
  for (int c = 0; c < nchunk; c++) poff[c] = 8 * N * c;
  const int n4 = 4 * N;
  DeviceScope ds;
  InflArgs a = infl_args(ds, tb, N, Nbase, tilesz, 1);
  a.coh = (const double2 *)ds.upload(coh, (size_t)8 * R);
  a.res = (const double2 *)ds.upload(res, (size_t)8 * R);
  a.p = ds.upload(p, (size_t)8 * N * nchunk);
  a.clus_nchunk = ds.upload(nch); a.clus_chunk0 = ds.upload(ch0); a.chunk_poff = ds.upload(poff);
  a.X = (const double2 *)ds.upload(X, (size_t)2 * n4 * Nbase);
  db_launch_infl_assemble(&a, ds.st);
  db_launch_infl_dr(&a, ds.st);
  DB_CHECK(cudaMemcpyAsync(hess, a.H, sizeof(double2) * n4 * n4, cudaMemcpyDeviceToHost, ds.st));
  DB_CHECK(cudaMemcpyAsync(AdV, a.AdV, sizeof(double2) * n4 * Nbase, cudaMemcpyDeviceToHost, ds.st));
  DB_CHECK(cudaMemcpyAsync(dR, a.dR, sizeof(double2) * 4 * Nbase * Nbase, cudaMemcpyDeviceToHost, ds.st));
  ds.sync();
  return 0;
}
