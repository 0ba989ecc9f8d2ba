// Host side of the device coherency prediction: packs clus_source_t into the flat device sky,
// and implements precalculate_coherencies / predict_visibilities_multifreq of the Dirac radio API.
#include <math.h>
#include <string.h>
#include <vector>

#include "../../include/dirac_b200.h"
#include "../../include/dirac_b200_channels.h"
#include "../../include/dirac_b200_stochastic.h"
#include "coh.h"
#include "influence.h"
#include "problem.h"

// the sky of M clusters, u, v, w of R rows and Nchan channel frequencies on the device through ds, and
// the CohArgs fields every sky entry point shares; fdelta_ch: the smearing width of one channel
static CohArgs stage_sky(DeviceScope &ds, const clus_source_t *carr, int M, const double *u,
                         const double *v, const double *w, long long R, const double *freqs,
                         int Nchan, double fdelta_ch) {
  std::vector<DevSource> src;
  std::vector<double> modes;
  std::vector<CohSegment> segs;
  for (int k = 0; k < M; k++) {
    const clus_source_t &c = carr[k];
    const int first = (int)src.size();
    for (int s = 0; s < c.N; s++) {
      DevSource d;
      memset(&d, 0, sizeof(d));
      d.ll = c.ll[s]; d.mm = c.mm[s]; d.nn = c.nn[s];
      d.sI = c.sI[s]; d.sQ = c.sQ[s]; d.sU = c.sU[s]; d.sV = c.sV[s];
      d.stype = (double)c.stype[s];
      d.ra = c.ra ? c.ra[s] : 0.0;
      d.dec = c.dec ? c.dec[s] : 0.0;
      if (c.stype[s] == STYPE_SHAPELET && c.ex && c.ex[s]) {
        const exinfo_shapelet *g = (const exinfo_shapelet *)c.ex[s];
        if (g->n0 < 1 || g->n0 > COH_SHAPELET_MAX_N0) {
          fprintf(stderr, "dirac_b200: shapelet order %d of cluster %d source %d is outside 1..%d\n",
                  g->n0, k, s, COH_SHAPELET_MAX_N0);
          exit(1);
        }
        d.eX = g->eX; d.eY = g->eY; d.eP = g->eP; d.cxi = g->cxi; d.sxi = g->sxi;
        d.cphi = g->cphi; d.sphi = g->sphi; d.use_projection = (double)g->use_projection;
        d.sh_n0 = (double)g->n0; d.sh_beta = g->beta; d.sh_off = (double)modes.size();
        modes.insert(modes.end(), g->modes, g->modes + (size_t)g->n0 * g->n0);
      } else if (c.stype[s] == STYPE_SHAPELET) {
        fprintf(stderr, "dirac_b200: shapelet source without exinfo (cluster %d source %d)\n", k, s);
        exit(1);
      }
      if (c.stype[s] == STYPE_GAUSSIAN && c.ex && c.ex[s]) {
        const exinfo_gaussian *g = (const exinfo_gaussian *)c.ex[s];
        d.eX = g->eX; d.eY = g->eY; d.eP = g->eP; d.cxi = g->cxi; d.sxi = g->sxi;
        d.cphi = g->cphi; d.sphi = g->sphi; d.use_projection = (double)g->use_projection;
      } else if ((c.stype[s] == STYPE_DISK || c.stype[s] == STYPE_RING) && c.ex && c.ex[s]) {
        // exinfo_disk / exinfo_ring: { eX; cxi, sxi, cphi, sphi; use_projection }
        const double *g = (const double *)c.ex[s];
        d.eX = g[0]; d.cxi = g[1]; d.sxi = g[2]; d.cphi = g[3]; d.sphi = g[4];
        d.use_projection = 1.0;
      }
      d.sI0 = c.sI0 ? c.sI0[s] : c.sI[s];
      d.sQ0 = c.sQ0 ? c.sQ0[s] : c.sQ[s];
      d.sU0 = c.sU0 ? c.sU0[s] : c.sU[s];
      d.sV0 = c.sV0 ? c.sV0[s] : c.sV[s];
      d.f0 = c.f0 ? c.f0[s] : 1.0;
      d.spec_idx = c.spec_idx ? c.spec_idx[s] : 0.0;
      d.spec_idx1 = c.spec_idx1 ? c.spec_idx1[s] : 0.0;
      d.spec_idx2 = c.spec_idx2 ? c.spec_idx2[s] : 0.0;
      src.push_back(d);
    }
    int done = 0;
    do {  // an empty cluster still yields one (empty, closing) segment
      CohSegment sg;
      sg.first = first + done;
      sg.count = c.N - done;
      if (sg.count > COH_SEG_MAX) sg.count = COH_SEG_MAX;
      sg.cluster = k;
      done += sg.count;
      sg.last = (done >= c.N) ? 1 : 0;
      segs.push_back(sg);
    } while (done < c.N);
  }
  if (src.empty()) src.resize(1);
  if (modes.empty()) modes.resize(2, 0.0);
  CohArgs a;
  memset(&a, 0, sizeof(a));
  a.modes = ds.upload(modes);
  a.src = ds.upload(src);
  a.segs = ds.upload(segs);
  db_stream_sync(ds.st);  // the vectors go out of scope
  a.nseg = (int)segs.size();
  a.beam_S = (int)src.size();  // the stride of the beam tables, read only with them
  db_count_sky_upload();
  a.u = ds.upload(u, R); a.v = ds.upload(v, R); a.w = ds.upload(w, R);
  a.freqs = ds.upload(freqs, Nchan); a.Nchan = Nchan; a.fdelta2 = fdelta_ch * 0.5; a.R = R;
  return a;
}

// the stations of every row, for the kernel modes that index Jones or beams by station; h holds the
// host copy until the caller's next wait
static void upload_row_stations(DeviceScope &ds, const baseline_t *barr, long long R,
                                std::vector<int> &h, CohArgs *a) {
  h.resize(2 * R);
  for (long long r = 0; r < R; r++) {
    h[r] = barr[r].sta1;
    h[R + r] = barr[r].sta2;
  }
  a->sta1 = ds.upload(h.data(), R);
  a->sta2 = ds.upload(h.data() + R, R);
}


// ---- station beams (precalculate_coherencies_withbeam & co, predict_withbeam.c) -----------------------
// doBeam: Dirac_common.h:120-151
static bool beam_wide(int doBeam) {
  return doBeam == DOBEAM_ARRAY_WB || doBeam == DOBEAM_FULL_WB || doBeam == DOBEAM_ELEMENT_WB;
}
static bool beam_array(int doBeam) {
  return doBeam == DOBEAM_ARRAY || doBeam == DOBEAM_FULL || doBeam == DOBEAM_ARRAY_WB ||
         doBeam == DOBEAM_FULL_WB;
}
static bool beam_element(int doBeam) {
  return doBeam == DOBEAM_ELEMENT || doBeam == DOBEAM_FULL || doBeam == DOBEAM_ELEMENT_WB ||
         doBeam == DOBEAM_FULL_WB;
}
// the first entry (in complex coefficients) of the coefficient set channel c is predicted with: a
// wide-band element table holds one set per channel (predict_withbeam.c:842, Nf = Nchan), the other
// modes one set for all channels
static size_t beam_channel_set(const BeamSpec *b, int c) {
  return beam_wide(b->doBeam) && b->ecoeff ? (size_t)b->ecoeff->Nmodes * c : 0;
}
// a row outside [uvmin, uvmax] at the beam-former's reference frequency (predict_withbeam.c:474-476
// with freq0 = ph_freq0, :784)
static bool beam_uv_outside(double u, double v, double ph_freq0, double uvmin, double uvmax) {
  const double uvdist = sqrt(u * u + v * v) * ph_freq0;
  return uvdist < uvmin || uvdist > uvmax;
}
// what the beam tables read that depends on neither time nor channel, on the device: stations,
// element layouts and every coefficient set; the array factor and E-Jones buffers hold ntab entries.
// The caller fills in the sky, the channels and the timeslots of each launch.
static BeamArgs beam_upload(DeviceScope &ds, const BeamSpec *b, int N, size_t ntab) {
  const bool do_array = beam_array(b->doBeam), do_elem = beam_element(b->doBeam);
  if (!do_array && !do_elem) {
    fprintf(stderr, "dirac_b200: beam mode %d is not supported (the lunar element beam needs "
                    "CSPICE)\n", b->doBeam);
    exit(1);
  }
  BeamArgs g;
  memset(&g, 0, sizeof(g));
  g.f0 = b->ph_freq0;
  g.N = N; g.bf_type = b->bf_type; g.b_ra0 = b->b_ra0; g.b_dec0 = b->b_dec0;
  g.ra0 = b->ph_ra0; g.dec0 = b->ph_dec0; g.wideband = beam_wide(b->doBeam) ? 1 : 0;
  g.lon = ds.upload(b->longitude, N);
  g.lat = ds.upload(b->latitude, N);
  if (do_array) {
    if (b->bf_type != STAT_SINGLE && b->bf_type != STAT_TILE) {
      fprintf(stderr, "dirac_b200: array beam needs bf_type STAT_SINGLE or STAT_TILE\n");
      exit(1);
    }
    std::vector<int> off(N), ne(N);
    std::vector<double> ex, ey, ez;
    for (int n = 0; n < N; n++) {
      off[n] = (int)ex.size();
      ne[n] = b->Nelem[n];
      const int len = b->Nelem[n] + (b->bf_type == STAT_TILE ? HBA_TILE_SIZE : 0);
      ex.insert(ex.end(), b->xx[n], b->xx[n] + len);
      ey.insert(ey.end(), b->yy[n], b->yy[n] + len);
      ez.insert(ez.end(), b->zz[n], b->zz[n] + len);
    }
    g.elem_off = ds.upload(off);
    g.Nelem = ds.upload(ne);
    g.ex = ds.upload(ex);
    g.ey = ds.upload(ey);
    g.ez = ds.upload(ez);
    g.af = ds.alloc<double>(ntab);
    db_stream_sync(ds.st);  // the host vectors go out of scope
  }
  if (do_elem) {
    const elementcoeff *ec = b->ecoeff;
    if (!ec || !ec->pattern_phi || !ec->pattern_theta || !ec->preamble) {
      fprintf(stderr, "dirac_b200: element beam requested (doBeam %d) without coefficient tables "
                      "(set_elementcoeffs)\n", b->doBeam);
      exit(1);
    }
    const int nfc = g.wideband ? ec->Nf : 1;
    g.ecM = ec->M; g.ecNmodes = ec->Nmodes; g.ecbeta = ec->beta;
    g.pat_phi = (const double2 *)ds.upload(ec->pattern_phi, 2ll * ec->Nmodes * nfc);
    g.pat_theta = (const double2 *)ds.upload(ec->pattern_theta, 2ll * ec->Nmodes * nfc);
    g.preamble = ds.upload(ec->preamble, ec->Nmodes);
    g.E = ds.alloc<double2>(4 * ntab);
  }
  return g;
}
// one launch of k_beam_tables over g.T timeslots and g.Nf channels (profile kind 15: the tables
// written once)
static void beam_tables(const BeamArgs &g, cudaStream_t st) {
  const double ntab = (double)g.T * g.Nf * g.S * g.N;
  db_prof_begin(15, ntab * ((g.af ? 8.0 : 0.0) + (g.E ? 64.0 : 0.0)), st);
  db_launch_beam_tables(&g, st);
  db_prof_end(st);
  db_count_launch(1);
}
// builds the per (timeslot, channel, source, station) tables on the device for the sky and channels
// staged in a and points the coherency kernel at them
static void beam_prepare(DeviceScope &ds, const BeamSpec *b, int N, int Nbase_slot,
                         const baseline_t *barr, CohArgs *a) {
  if (!b || b->doBeam == DOBEAM_NONE) return;
  BeamArgs g = beam_upload(ds, b, N, (size_t)b->tilesz * a->Nchan * a->beam_S * N);
  g.src = a->src; g.S = a->beam_S; g.freqs = a->freqs; g.Nf = a->Nchan;
  g.T = b->tilesz;
  g.time_jd = ds.upload(b->time_utc, b->tilesz);
  beam_tables(g, ds.st);
  // the coherency kernel needs the stations of every row now
  if (!a->sta1) {
    std::vector<int> sta;
    upload_row_stations(ds, barr, a->R, sta, a);
    db_stream_sync(ds.st);
  }
  a->beam_af = g.af; a->beam_E = g.E; a->Nbase = Nbase_slot; a->N = N;
}

extern "C" void dirac_b200_precalculate(dirac_b200_problem *pr, const double *u, const double *v,
                                        const double *w, const clus_source_t *carr, double freq0,
                                        double fdelta, double uvmin, double uvmax,
                                        baseline_t *barr) {
  DevProblem &d = pr->d;
  DeviceScope ds(d.stream);
  CohArgs a = stage_sky(ds, carr, d.M, u, v, w, d.R, &freq0, 1, fdelta);
  a.uvmin = uvmin; a.uvmax = uvmax; a.coh = d.coh; a.flag = d.flag;
  db_launch_coherencies(&a, ds.st);
  db_count_launch(1);
  if (barr) {
    std::vector<unsigned char> hf(d.R);
    DB_CHECK(cudaMemcpyAsync(hf.data(), d.flag, d.R, cudaMemcpyDeviceToHost, ds.st));
    db_stream_sync(ds.st);
    for (long long r = 0; r < d.R; r++) barr[r].flag = hf[r];
  }
  ds.sync();
  // the Gram tensors cached for LM belong to the old coherencies
  if (pr->lm.ready) memset(pr->lm.T_valid, 0, d.Mt);
}

// Dirac_radio.h:209 — here Nbase is already Nbase*tilesz (predict.c:503-578); rows need not be in
// canonical order for this call (no station indexing), only flags are read/written.
static int precalculate_impl(double *u, double *v, double *w, double *x, int N, int Nbase,
                            baseline_t *barr, clus_source_t *carr, int M, double freq0,
                            double fdelta, double uvmin, double uvmax, const BeamSpec *beam) {
  DeviceScope ds;
  const long long R = Nbase;
  CohArgs a = stage_sky(ds, carr, M, u, v, w, R, &freq0, 1, fdelta);
  std::vector<unsigned char> hf(R);
  for (long long r = 0; r < R; r++) hf[r] = barr[r].flag;
  a.flag = ds.alloc<unsigned char>(R + 16);
  DB_CHECK(cudaMemcpyAsync(a.flag, hf.data(), R, cudaMemcpyHostToDevice, ds.st));
  a.coh = ds.alloc<double2>((size_t)M * 4 * R);
  a.uvmin = uvmin; a.uvmax = uvmax;
  beam_prepare(ds, beam, N, N * (N - 1) / 2, barr, &a);
  db_launch_coherencies(&a, ds.st);
  db_count_launch(1);
  DB_CHECK(cudaMemcpyAsync(hf.data(), a.flag, R, cudaMemcpyDeviceToHost, ds.st));
  db_download_coh(a.coh, x, M, R, ds.st);  // waits for the flags too
  DB_CHECK(cudaGetLastError());
  for (long long r = 0; r < R; r++) barr[r].flag = hf[r];
  return 0;
}
extern "C" int precalculate_coherencies(double *u, double *v, double *w, double *x, int N,
                                        int Nbase, baseline_t *barr, clus_source_t *carr, int M,
                                        double freq0, double fdelta, double tdelta, double dec0,
                                        double uvmin, double uvmax, int Nt) {
  (void)tdelta; (void)dec0; (void)Nt;
  return precalculate_impl(u, v, w, x, N, Nbase, barr, carr, M, freq0, fdelta, uvmin, uvmax, nullptr);
}
// Dirac_radio.h:472,516 (predict_withbeam.c:553-723): the same with the station beam towards every
// source folded in: array factor (a real gain per station) and / or element beam (a 2x2 E-Jones per
// station), evaluated per timeslot.  Nbase is Nbase*tilesz here too; rows in time order.
extern "C" int precalculate_coherencies_withbeam(
    double *u, double *v, double *w, double *x, int N, int Nbase, baseline_t *barr,
    clus_source_t *carr, int M, double freq0, double fdelta, double tdelta, double dec0, double uvmin,
    double uvmax, int bf_type, double b_ra0, double b_dec0, double ph_ra0, double ph_dec0,
    double ph_freq0, double *longitude, double *latitude, double *time_utc, int tilesz, int *Nelem,
    double **xx, double **yy, double **zz, elementcoeff *ecoeff, int doBeam, int Nt) {
  (void)tdelta; (void)dec0; (void)Nt;
  BeamSpec b = {bf_type, b_ra0, b_dec0, ph_ra0, ph_dec0, ph_freq0, longitude, latitude, time_utc,
                tilesz, Nelem, xx, yy, zz, ecoeff, doBeam};
  return precalculate_impl(u, v, w, x, N, Nbase, barr, carr, M, freq0, fdelta, uvmin, uvmax, &b);
}
extern "C" int precalculate_coherencies_withbeam_gpu(
    double *u, double *v, double *w, double *x, int N, int Nbase, baseline_t *barr,
    clus_source_t *carr, int M, double freq0, double fdelta, double tdelta, double dec0, double uvmin,
    double uvmax, int bf_type, double b_ra0, double b_dec0, double ph_ra0, double ph_dec0,
    double ph_freq0, double *longitude, double *latitude, double *time_utc, int tilesz, int *Nelem,
    double **xx, double **yy, double **zz, elementcoeff *ecoeff, int doBeam, int Nt) {
  return precalculate_coherencies_withbeam(u, v, w, x, N, Nbase, barr, carr, M, freq0, fdelta, tdelta,
                                           dec0, uvmin, uvmax, bf_type, b_ra0, b_dec0, ph_ra0,
                                           ph_dec0, ph_freq0, longitude, latitude, time_utc, tilesz,
                                           Nelem, xx, yy, zz, ecoeff, doBeam, Nt);
}

// Dirac_radio.h:221,479,534 (predict.c:745-816, predict_withbeam.c:726-900): coherencies of Nchan
// channels, x[chan][row][cluster][4] -- what the minibatch drivers feed bfgsfit_minibatch_*.  Fluxes
// are the catalogue's (no spectral index here, predict.c:690-696), the smearing width is
// fdelta / Nchan per channel (:792), a row gets flag 2 if it is shorter than uvmin at the first
// channel or longer than uvmax at the last (:731-735); the beam variant cuts both ways at the
// beam-former's reference frequency instead (predict_withbeam.c:456-463,784).  One pass of the single-channel kernel per
// channel; wide-band element beams see their channel's coefficient set.
static int precalculate_multifreq_impl(double *u, double *v, double *w, double *x, int N, int Nbase,
                                       baseline_t *barr, clus_source_t *carr, int M, double *freqs,
                                       int Nchan, double fdelta, double uvmin, double uvmax,
                                       const BeamSpec *beam) {
  const double HUGE_UV = 1e300;
  for (int c = 0; c < Nchan; c++) {
    // (the beam variant cuts on ONE frequency, ph_freq0: done on the host below)
    const double lo = (c == 0 && !beam) ? uvmin : 0.0;
    const double hi = (c == Nchan - 1 && !beam) ? uvmax : HUGE_UV;
    BeamSpec bc;
    elementcoeff ec;
    const BeamSpec *bp = nullptr;
    if (beam) {
      bc = *beam;
      if (beam_wide(beam->doBeam) && beam->ecoeff) {  // this channel's set as a one-frequency table
        ec = *beam->ecoeff;
        ec.pattern_phi = beam->ecoeff->pattern_phi + 2 * beam_channel_set(beam, c);
        ec.pattern_theta = beam->ecoeff->pattern_theta + 2 * beam_channel_set(beam, c);
        ec.Nf = 1;
        bc.ecoeff = &ec;
      }
      bp = &bc;
    }
    const int rv = precalculate_impl(u, v, w, x + (size_t)c * 8 * M * Nbase, N, Nbase, barr, carr, M,
                                     freqs[c], fdelta / (double)Nchan, lo, hi, bp);
    if (rv) return rv;
  }
  if (beam)
    for (long long r = 0; r < Nbase; r++)
      if (!barr[r].flag && beam_uv_outside(u[r], v[r], beam->ph_freq0, uvmin, uvmax)) barr[r].flag = 2;
  return 0;
}
extern "C" int precalculate_coherencies_multifreq(double *u, double *v, double *w, double *x, int N,
                                                  int Nbase, baseline_t *barr, clus_source_t *carr,
                                                  int M, double *freqs, int Nchan, double fdelta,
                                                  double tdelta, double dec0, double uvmin,
                                                  double uvmax, int Nt) {
  (void)tdelta; (void)dec0; (void)Nt;
  return precalculate_multifreq_impl(u, v, w, x, N, Nbase, barr, carr, M, freqs, Nchan, fdelta, uvmin,
                                     uvmax, nullptr);
}
extern "C" int precalculate_coherencies_multifreq_withbeam(
    double *u, double *v, double *w, double *x, int N, int Nbase, baseline_t *barr,
    clus_source_t *carr, int M, double *freqs, int Nchan, double fdelta, double tdelta, double dec0,
    double uvmin, double uvmax, int bf_type, double b_ra0, double b_dec0, double ph_ra0,
    double ph_dec0, double ph_freq0, double *longitude, double *latitude, double *time_utc, int tilesz,
    int *Nelem, double **xx, double **yy, double **zz, elementcoeff *ecoeff, int doBeam, int Nt) {
  (void)tdelta; (void)dec0; (void)Nt;
  BeamSpec b = {bf_type, b_ra0, b_dec0, ph_ra0, ph_dec0, ph_freq0, longitude, latitude, time_utc,
                tilesz, Nelem, xx, yy, zz, ecoeff, doBeam};
  return precalculate_multifreq_impl(u, v, w, x, N, Nbase, barr, carr, M, freqs, Nchan, fdelta, uvmin,
                                     uvmax, &b);
}
extern "C" int precalculate_coherencies_multifreq_withbeam_gpu(
    double *u, double *v, double *w, double *x, int N, int Nbase, baseline_t *barr,
    clus_source_t *carr, int M, double *freqs, int Nchan, double fdelta, double tdelta, double dec0,
    double uvmin, double uvmax, int bf_type, double b_ra0, double b_dec0, double ph_ra0,
    double ph_dec0, double ph_freq0, double *longitude, double *latitude, double *time_utc, int tilesz,
    int *Nelem, double **xx, double **yy, double **zz, elementcoeff *ecoeff, int doBeam, int Nt) {
  return precalculate_coherencies_multifreq_withbeam(u, v, w, x, N, Nbase, barr, carr, M, freqs, Nchan,
                                                     fdelta, tdelta, dec0, uvmin, uvmax, bf_type,
                                                     b_ra0, b_dec0, ph_ra0, ph_dec0, ph_freq0,
                                                     longitude, latitude, time_utc, tilesz, Nelem, xx,
                                                     yy, zz, ecoeff, doBeam, Nt);
}

// Dirac_radio.h:659 (residual.c:1257-1340): x[chan][row][8] += sum over clusters; add_to_data ==
// SIMUL_ONLY (1, Dirac_radio.h:78) clears x first, every other value accumulates onto the input
// (the thread function only ever adds, residual.c:1238-1245).  No Jones, no flags.
static int predict_multifreq_impl(double *u, double *v, double *w, double *x, int N, int Nbase,
                                  int tilesz, baseline_t *barr, clus_source_t *carr, int M,
                                  double *freqs, int Nchan, double fdelta, int add_to_data,
                                  const BeamSpec *beam) {
  DeviceScope ds;
  const long long R = (long long)Nbase * tilesz;
  CohArgs a = stage_sky(ds, carr, M, u, v, w, R, freqs, Nchan, fdelta / (double)Nchan);
  const size_t nx = (size_t)Nchan * R * 4;
  a.xout = ds.alloc<double2>(nx);
  if (add_to_data == 1) {  // SIMUL_ONLY
    DB_CHECK(cudaMemsetAsync(a.xout, 0, sizeof(double2) * nx, ds.st));
  } else {
    DB_CHECK(cudaMemcpyAsync(a.xout, x, sizeof(double2) * nx, cudaMemcpyHostToDevice, ds.st));
  }
  beam_prepare(ds, beam, N, Nbase, barr, &a);
  db_launch_predict_multifreq(&a, ds.st);
  db_count_launch(1);
  DB_CHECK(cudaMemcpyAsync(x, a.xout, sizeof(double2) * nx, cudaMemcpyDeviceToHost, ds.st));
  ds.sync();
  return 0;
}
extern "C" int predict_visibilities_multifreq(double *u, double *v, double *w, double *x, int N,
                                              int Nbase, int tilesz, baseline_t *barr,
                                              clus_source_t *carr, int M, double *freqs, int Nchan,
                                              double fdelta, double tdelta, double dec0, int Nt,
                                              int add_to_data) {
  (void)tdelta; (void)dec0; (void)Nt;
  return predict_multifreq_impl(u, v, w, x, N, Nbase, tilesz, barr, carr, M, freqs, Nchan, fdelta,
                                add_to_data, nullptr);
}
// Dirac_radio.h:485,521 (predict_withbeam.c:1219-1440): per-channel station beams
extern "C" int predict_visibilities_multifreq_withbeam(
    double *u, double *v, double *w, double *x, int N, int Nbase, int tilesz, baseline_t *barr,
    clus_source_t *carr, int M, double *freqs, int Nchan, double fdelta, double tdelta, double dec0,
    int bf_type, double b_ra0, double b_dec0, double ph_ra0, double ph_dec0, double ph_freq0,
    double *longitude, double *latitude, double *time_utc, int *Nelem, double **xx, double **yy,
    double **zz, elementcoeff *ecoeff, int doBeam, int Nt, int add_to_data) {
  (void)tdelta; (void)dec0; (void)Nt;
  BeamSpec b = {bf_type, b_ra0, b_dec0, ph_ra0, ph_dec0, ph_freq0, longitude, latitude, time_utc,
                tilesz, Nelem, xx, yy, zz, ecoeff, doBeam};
  return predict_multifreq_impl(u, v, w, x, N, Nbase, tilesz, barr, carr, M, freqs, Nchan, fdelta,
                                add_to_data, &b);
}
extern "C" int predict_visibilities_multifreq_withbeam_gpu(
    double *u, double *v, double *w, double *x, int N, int Nbase, int tilesz, baseline_t *barr,
    clus_source_t *carr, int M, double *freqs, int Nchan, double fdelta, double tdelta, double dec0,
    int bf_type, double b_ra0, double b_dec0, double ph_ra0, double ph_dec0, double ph_freq0,
    double *longitude, double *latitude, double *time_utc, int *Nelem, double **xx, double **yy,
    double **zz, elementcoeff *ecoeff, int doBeam, int Nt, int add_to_data) {
  return predict_visibilities_multifreq_withbeam(u, v, w, x, N, Nbase, tilesz, barr, carr, M, freqs,
                                                 Nchan, fdelta, tdelta, dec0, bf_type, b_ra0, b_dec0,
                                                 ph_ra0, ph_dec0, ph_freq0, longitude, latitude,
                                                 time_utc, Nelem, xx, yy, zz, ecoeff, doBeam, Nt,
                                                 add_to_data);
}

// 2x2 inverse of (J + rho I) with the reference's guard on a small determinant (mat_invert,
// residual.c:162-199)
static void jones_invert(const double xx[8], double yy[8], double rho) {
  const double a0r = xx[0] + rho, a0i = xx[1], a1r = xx[2], a1i = xx[3];
  const double a2r = xx[4], a2i = xx[5], a3r = xx[6] + rho, a3i = xx[7];
  double dr = (a0r * a3r - a0i * a3i) - (a1r * a2r - a1i * a2i);
  double di = (a0r * a3i + a0i * a3r) - (a1r * a2i + a1i * a2r);
  if (sqrt(sqrt(dr * dr + di * di)) <= rho) dr += rho;
  const double den = dr * dr + di * di;
  const double ir = dr / den, ii = -di / den;  // 1/det
  yy[0] = a3r * ir - a3i * ii;      yy[1] = a3r * ii + a3i * ir;
  yy[2] = -(a1r * ir - a1i * ii);   yy[3] = -(a1r * ii + a1i * ir);
  yy[4] = -(a2r * ir - a2i * ii);   yy[5] = -(a2r * ii + a2i * ir);
  yy[6] = a0r * ir - a0i * ii;      yy[7] = a0r * ii + a0i * ir;
}

// eigenvector of the largest eigenvalue of a real symmetric 3x3 matrix by cyclic Jacobi rotations
// (stands in for dsyevx with IL = IU = 3, manifold_average.c:470,541)
static void sym3_top_eigvec(const double Hin[3][3], double z[3]) {
  double A[3][3], V[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) A[i][j] = Hin[i][j];
  for (int sweep = 0; sweep < 60; sweep++) {
    const double off = A[0][1] * A[0][1] + A[0][2] * A[0][2] + A[1][2] * A[1][2];
    const double dg = A[0][0] * A[0][0] + A[1][1] * A[1][1] + A[2][2] * A[2][2];
    if (off <= 1e-34 * dg || off == 0.0) break;
    for (int p = 0; p < 2; p++)
      for (int q = p + 1; q < 3; q++) {
        if (A[p][q] == 0.0) continue;
        const double theta = (A[q][q] - A[p][p]) / (2.0 * A[p][q]);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), sn = t * c;
        for (int k = 0; k < 3; k++) {  // A <- A R
          const double akp = A[k][p], akq = A[k][q];
          A[k][p] = c * akp - sn * akq;
          A[k][q] = sn * akp + c * akq;
        }
        for (int k = 0; k < 3; k++) {  // A <- R^T A
          const double apk = A[p][k], aqk = A[q][k];
          A[p][k] = c * apk - sn * aqk;
          A[q][k] = sn * apk + c * aqk;
        }
        for (int k = 0; k < 3; k++) {
          const double vkp = V[k][p], vkq = V[k][q];
          V[k][p] = c * vkp - sn * vkq;
          V[k][q] = sn * vkp + c * vkq;
        }
      }
  }
  int top = 0;
  for (int i = 1; i < 3; i++)
    if (A[i][i] > A[top][top]) top = i;
  const double nrm = sqrt(V[0][top] * V[0][top] + V[1][top] * V[1][top] + V[2][top] * V[2][top]);
  for (int i = 0; i < 3; i++) z[i] = V[i][top] / nrm;
}

// phases of the jointly diagonalised solutions of one (cluster, chunk): niter rounds of two Jacobi
// rotations J <- J G^H common to all stations (towards diagonal J), then the unit-modulus diagonal
// (extract_phases, manifold_average.c:399-610).  pin / pout: N x 8 doubles in the pp layout.
static void extract_phases_host(const double *pin, double *pout, int N, int niter) {
  struct cd { double r, i; };
  auto mul = [](cd a, cd b) { return cd{a.r * b.r - a.i * b.i, a.r * b.i + a.i * b.r}; };
  auto conj = [](cd a) { return cd{a.r, -a.i}; };
  std::vector<cd> J00(N), J01(N), J10(N), J11(N);
  for (int s = 0; s < N; s++) {
    J00[s] = {pin[8 * s + 0], pin[8 * s + 1]};
    J01[s] = {pin[8 * s + 2], pin[8 * s + 3]};
    J10[s] = {pin[8 * s + 4], pin[8 * s + 5]};
    J11[s] = {pin[8 * s + 6], pin[8 * s + 7]};
  }
  for (int ni = 0; ni < niter; ni++)
    for (int pass = 0; pass < 2; pass++) {
      double H[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
      for (int s = 0; s < N; s++) {
        // pass 0: h = conj[a - d, b + c, i (c - b)]; pass 1: h = conj[d - a, c + b, i (b - c)]
        const cd a = J00[s], b = J01[s], c = J10[s], d = J11[s];
        const double sg = pass == 0 ? 1.0 : -1.0;
        cd h[3];
        h[0] = conj(cd{sg * (a.r - d.r), sg * (a.i - d.i)});
        h[1] = conj(cd{b.r + c.r, b.i + c.i});
        const cd cmb = {sg * (c.r - b.r), sg * (c.i - b.i)};
        h[2] = conj(cd{-cmb.i, cmb.r});  // i (c - b)
        for (int i = 0; i < 3; i++)
          for (int j = 0; j < 3; j++) H[i][j] += h[i].r * h[j].r + h[i].i * h[j].i;  // Re(h h^H)
      }
      double Z[3];
      sym3_top_eigvec(H, Z);
      cd cc, ss;
      if (Z[0] >= 0.0) {
        cc = {sqrt(0.5 + Z[0] * 0.5), 0.0};
        ss = {0.5 * Z[1] / cc.r, -0.5 * Z[2] / cc.r};
      } else {
        cc = {sqrt(0.5 - Z[0] * 0.5), 0.0};
        ss = {-0.5 * Z[1] / cc.r, 0.5 * Z[2] / cc.r};
      }
      // G = [c, conj(s); -s, conj(c)] (column-major [c, -s, conj(s), conj(c)]);  J <- J G^H
      // (G^H)(0,0) = conj(c), (G^H)(0,1) = conj(-s), (G^H)(1,0) = s, (G^H)(1,1) = c
      const cd g00 = conj(cc), g01 = conj(cd{-ss.r, -ss.i}), g10 = ss, g11 = cc;
      for (int s = 0; s < N; s++) {
        const cd a = J00[s], b = J01[s], c = J10[s], d = J11[s];
        const cd t0 = mul(a, g00), t1 = mul(b, g10), t2 = mul(a, g01), t3 = mul(b, g11);
        const cd u0 = mul(c, g00), u1 = mul(d, g10), u2 = mul(c, g01), u3 = mul(d, g11);
        J00[s] = {t0.r + t1.r, t0.i + t1.i};
        J01[s] = {t2.r + t3.r, t2.i + t3.i};
        J10[s] = {u0.r + u1.r, u0.i + u1.i};
        J11[s] = {u2.r + u3.r, u2.i + u3.i};
      }
    }
  memset(pout, 0, sizeof(double) * 8 * N);
  for (int s = 0; s < N; s++) {
    const double m0 = sqrt(J00[s].r * J00[s].r + J00[s].i * J00[s].i);
    const double m1 = sqrt(J11[s].r * J11[s].r + J11[s].i * J11[s].i);
    pout[8 * s + 0] = J00[s].r / m0;
    pout[8 * s + 1] = J00[s].i / m0;
    pout[8 * s + 6] = J11[s].r / m1;
    pout[8 * s + 7] = J11[s].i / m1;
  }
}

// host arithmetic, no GPU needed: exposed so that the CPU tests can pin it against the reference
extern "C" int dirac_b200_extract_phases(const double *p, double *pout, int N, int niter) {
  extract_phases_host(p, pout, N, niter);
  return 0;
}

// what MODE 2 of the sky kernel reads besides the sky, pointed to from a: chunk tables, the stations
// of every row and the sign of every cluster.  cm: the LAST cluster with id == ccid
// (residual.c:584-590), or -1; npar: doubles of p the chunk offsets reach
struct ResidualTables {
  int cm;
  long long npar;
};
static ResidualTables residual_tables(DeviceScope &ds, const baseline_t *barr,
                                      const clus_source_t *carr, int N, int M,
                                      const std::vector<signed char> &coef, int ccid, CohArgs *a) {
  ResidualTables t = {-1, 0};
  std::vector<int> nchunk(M), chunk0(M), poff, sta;
  int mt = 0;
  for (int k = 0; k < M; k++) {
    nchunk[k] = carr[k].nchunk;
    chunk0[k] = mt;
    if (carr[k].id == ccid) t.cm = k;
    for (int c = 0; c < carr[k].nchunk; c++) {
      poff.push_back(carr[k].p[c]);
      if ((long long)carr[k].p[c] + 8ll * N > t.npar) t.npar = (long long)carr[k].p[c] + 8ll * N;
    }
    mt += carr[k].nchunk;
  }
  a->clus_nchunk = ds.upload(nchunk);
  a->clus_chunk0 = ds.upload(chunk0);
  a->chunk_poff = ds.upload(poff);
  upload_row_stations(ds, barr, a->R, sta, a);
  a->clus_coef = ds.upload(coef);
  db_stream_sync(ds.st);  // the vectors go out of scope
  return t;
}
// (J + rho I)^-1 of every station and chunk of the correction cluster, [nchunk][N][8]; phase_only: of
// the phases of its jointly diagonalised solutions (residual.c:975-990)
static void correction_inverse(const double *p, const clus_source_t &c, int N, double rho,
                               int phase_only, std::vector<double> &pinv) {
  pinv.resize((size_t)8 * N * c.nchunk);
  std::vector<double> pphase(phase_only ? (size_t)8 * N : 0);
  for (int ck = 0; ck < c.nchunk; ck++) {
    const double *pm = p + c.p[ck];
    if (phase_only) {
      extract_phases_host(pm, pphase.data(), N, 10);
      pm = pphase.data();
    }
    for (int s = 0; s < N; s++) jones_invert(pm + 8 * s, pinv.data() + (size_t)8 * N * ck + 8 * s, rho);
  }
}

// Dirac_radio.h:652,666 (residual.c:940-1061,1620-1740): the model of every cluster with the solved
// Jones, per channel, x[chan][row][8] += coef[k] J_p C_k(chan) J_q^H (coef -1, 0 or +1 per cluster;
// clear_x: x starts from zero instead of the caller's data), the coherencies re-predicted from the
// sources at every channel frequency; then, if a cluster has id == ccid, every row is corrected by
// that cluster's inverse Jones (J + rho I)^-1; phase_only != 0: by the inverse of the phases of its
// jointly diagonalised solutions (extract_phases, manifold_average.c:399-610).  Rows are predicted
// whatever their flag.
// residuals_stage: the same up to the launch, the result left in a.xout on the device (pinv holds
// the host copy of the correction until the caller's next wait; correct false: no correction)
static CohArgs residuals_stage(DeviceScope &ds, const double *u, const double *v, const double *w,
                               const double *p, const double *x, int N, int Nbase, int tilesz,
                               const baseline_t *barr, const clus_source_t *carr, int M,
                               const double *freqs, int Nchan, double fdelta,
                               const std::vector<signed char> &coef, bool clear_x, bool correct,
                               int ccid, double rho, int phase_only, const BeamSpec *beam,
                               std::vector<double> &pinv) {
  const long long R = (long long)Nbase * tilesz;
  CohArgs a = stage_sky(ds, carr, M, u, v, w, R, freqs, Nchan, fdelta / (double)Nchan);
  const ResidualTables tb = residual_tables(ds, barr, carr, N, M, coef, ccid, &a);
  const int cm = correct ? tb.cm : -1;
  if (cm >= 0) correction_inverse(p, carr[cm], N, rho, phase_only, pinv);
  a.p = ds.upload(p, tb.npar);
  a.pinv = cm >= 0 ? ds.upload(pinv) : nullptr;
  a.pinv_nchunk = cm >= 0 ? carr[cm].nchunk : 1; a.N = N;
  const size_t nx = (size_t)Nchan * R * 4;
  a.xout = ds.alloc<double2>(nx);
  if (clear_x) {
    DB_CHECK(cudaMemsetAsync(a.xout, 0, sizeof(double2) * nx, ds.st));
  } else {
    DB_CHECK(cudaMemcpyAsync(a.xout, x, sizeof(double2) * nx, cudaMemcpyHostToDevice, ds.st));
  }
  beam_prepare(ds, beam, N, Nbase, barr, &a);
  db_prof_begin(11, 128.0 * (double)nx / 4.0, ds.st);  // profile kind 11: x read and written once
  db_launch_residual_multifreq(&a, ds.st);
  db_prof_end(ds.st);
  db_count_launch(1);
  return a;
}
static int residuals_multifreq_impl(double *u, double *v, double *w, double *p, double *x, int N,
                                    int Nbase, int tilesz, baseline_t *barr, clus_source_t *carr,
                                    int M, double *freqs, int Nchan, double fdelta,
                                    const std::vector<signed char> &coef, bool clear_x, int ccid,
                                    double rho, int phase_only, const BeamSpec *beam) {
  DeviceScope ds;
  std::vector<double> pinv;
  CohArgs a = residuals_stage(ds, u, v, w, p, x, N, Nbase, tilesz, barr, carr, M, freqs, Nchan, fdelta,
                              coef, clear_x, true, ccid, rho, phase_only, beam, pinv);
  const size_t nx = (size_t)Nchan * Nbase * tilesz * 4;
  DB_CHECK(cudaMemcpyAsync(x, a.xout, sizeof(double2) * nx, cudaMemcpyDeviceToHost, ds.st));
  ds.sync();
  return 0;
}

// Step 1 of calculate_diagnostics_gpu (diagnostics_host.cu): x[chan][row][4] on the device minus the
// model of every cluster, whatever its id, without correction (diagnostics.c:243-246), and the
// coherencies of every cluster at channel 0, [M][R][4], by the multi-channel prediction one cluster
// at a time: the same fluxes (spectral indices included), smearing width and beams as the model
int db_diagnostics_model(DeviceScope &ds, const double *u, const double *v, const double *w,
                         const double *p, const double *x, int N, int Nbase, int tilesz,
                         const baseline_t *barr, const clus_source_t *carr, int M,
                         const double *freqs, int Nchan, double fdelta, const BeamSpec *beam,
                         DiagModel *out) {
  std::vector<double> pinv;
  const std::vector<signed char> coef(M, -1);
  const CohArgs r = residuals_stage(ds, u, v, w, p, x, N, Nbase, tilesz, barr, carr, M, freqs, Nchan,
                                    fdelta, coef, false, false, 0, 0.0, 0, beam, pinv);
  const long long R = (long long)Nbase * tilesz;
  CohArgs a = stage_sky(ds, carr, M, u, v, w, R, freqs, 1, fdelta / (double)Nchan);
  beam_prepare(ds, beam, N, Nbase, barr, &a);
  double2 *coh = ds.alloc<double2>((size_t)M * 4 * R);
  DB_CHECK(cudaMemsetAsync(coh, 0, sizeof(double2) * M * 4 * R, ds.st));
  int seg0 = 0;
  for (int k = 0; k < M; k++) {  // stage_sky's segments of cluster k (at least one)
    const int nseg = carr[k].N > COH_SEG_MAX ? (carr[k].N + COH_SEG_MAX - 1) / COH_SEG_MAX : 1;
    CohArgs ak = a;
    ak.segs = a.segs + seg0; ak.nseg = nseg; ak.xout = coh + (size_t)k * 4 * R;
    db_launch_predict_multifreq(&ak, ds.st);
    seg0 += nseg;
  }
  db_count_launch(M);
  out->x = r.xout; out->coh = coh; out->p = r.p; out->clus_nchunk = r.clus_nchunk;
  out->clus_chunk0 = r.clus_chunk0; out->chunk_poff = r.chunk_poff;
  return 0;
}
// the residual subtracts the clusters with id >= 0 (residual.c:704)
static std::vector<signed char> residual_coef(const clus_source_t *carr, int M) {
  std::vector<signed char> coef(M);
  for (int k = 0; k < M; k++) coef[k] = carr[k].id >= 0 ? -1 : 0;
  return coef;
}
// the simulation predicts every cluster at a position k with ignorelist[k] == 0, whatever its id
// (residual.c:1373); add_to_data (Dirac_radio.h:78-80): SIMUL_ONLY 1 and SIMUL_ADD 2 add, SIMUL_SUB 3
// subtracts, any other value leaves x as the caller gave it (residual.c:1556-1576)
static std::vector<signed char> simul_coef(const int *ignorelist, int M, int add_to_data) {
  const signed char s = (add_to_data == 1 || add_to_data == 2) ? 1 : (add_to_data == 3 ? -1 : 0);
  std::vector<signed char> coef(M);
  for (int k = 0; k < M; k++) coef[k] = ignorelist[k] ? 0 : s;
  return coef;
}
extern "C" int calculate_residuals_multifreq(double *u, double *v, double *w, double *p, double *x,
                                             int N, int Nbase, int tilesz, baseline_t *barr,
                                             clus_source_t *carr, int M, double *freqs, int Nchan,
                                             double fdelta, double tdelta, double dec0, int Nt,
                                             int ccid, double rho, int phase_only) {
  (void)tdelta; (void)dec0; (void)Nt;
  return residuals_multifreq_impl(u, v, w, p, x, N, Nbase, tilesz, barr, carr, M, freqs, Nchan, fdelta,
                                  residual_coef(carr, M), false, ccid, rho, phase_only, nullptr);
}
// Dirac_radio.h:639 (residual.c:314-674): one channel at freq0; the worker is the multi-channel one
// with the channel loop taken out (no phase_only here)
extern "C" int calculate_residuals(double *u, double *v, double *w, double *p, double *x, int N,
                                   int Nbase, int tilesz, baseline_t *barr, clus_source_t *carr,
                                   int M, double freq0, double fdelta, double tdelta, double dec0,
                                   int Nt, int ccid, double rho) {
  (void)tdelta; (void)dec0; (void)Nt;
  return residuals_multifreq_impl(u, v, w, p, x, N, Nbase, tilesz, barr, carr, M, &freq0, 1, fdelta,
                                  residual_coef(carr, M), false, ccid, rho, 0, nullptr);
}

// The per-channel refinement of one interval (driver option -b 1, fullbatch_mode.cpp:464-497) on ONE
// resident problem.  Per channel: coherencies at the channel straight into the planar storage (with
// the uv cut accumulating in the resident flags, predict.c:489-495), LBFGS from the start Jones, then
// the residual re-predicted from the sky with the channel's spectral fluxes and the solved Jones, on
// the channel's data kept in API layout on the device.  Only the data of a channel go up and its
// residual comes down.
extern "C" int dirac_b200_bfgsfit_channels(double *u, double *v, double *w, double *xo, int N,
                                           int Nbase, int tilesz, baseline_t *barr,
                                           clus_source_t *carr, int M, int Mt, double *freqs,
                                           int Nchan, double deltafch, double uvmin, double uvmax,
                                           double *p, int max_lbfgs, int lbfgs_m, int solver_mode,
                                           double mean_nu, int ccid, double rho, double *res_00,
                                           double *res_01, double *pfreq) {
  if (Nchan < 1) return 0;
  dirac_b200_problem *pr = dirac_b200_create(N, Nbase, tilesz, barr, carr, M, Mt, nullptr, nullptr);
  DevProblem &d = pr->d;
  const long long R = d.R;
  const size_t m = (size_t)8 * N * Mt;
  {  // the scope ends before the problem whose stream it borrows
    DeviceScope ds(d.stream);
    CohArgs a = stage_sky(ds, carr, M, u, v, w, R, freqs, Nchan, deltafch);
    const double *df = a.freqs;
    const int cm = residual_tables(ds, barr, carr, N, M, residual_coef(carr, M), ccid, &a).cm;
    std::vector<double> pinv, pown(pfreq ? 0 : m);
    double *dpinv = cm >= 0 ? ds.alloc<double>((size_t)8 * N * carr[cm].nchunk) : nullptr;
    double2 *dx = (double2 *)db_malloc(sizeof(double2) * 4 * (size_t)R);  // [R][4]: data in, residual out
    a.Nchan = 1; a.uvmin = uvmin; a.uvmax = uvmax; a.N = N;
    a.pinv_nchunk = cm >= 0 ? carr[cm].nchunk : 1;
    double *pc = pown.data();
    for (int ci = 0; ci < Nchan; ci++) {
      double *xc = xo + (size_t)ci * 8 * R;
      DB_CHECK(cudaMemcpyAsync(dx, xc, (size_t)R * 64, cudaMemcpyHostToDevice, ds.st));
      db_launch_vis_to_planar(dx, d.x, R, ds.st);
      a.freqs = df + ci;
      a.coh = d.coh; a.flag = d.flag; a.xout = nullptr; a.p = nullptr; a.pinv = nullptr;
      db_launch_coherencies(&a, ds.st);
      db_count_launch(2);
      if (pfreq) pc = pfreq + (size_t)ci * m;
      memcpy(pc, p, sizeof(double) * m);
      db_bfgsfit_dev(pr, pc, max_lbfgs, lbfgs_m, solver_mode, mean_nu, res_00 + ci, res_01 + ci, false);
      // the fit left the solution in d.pp
      if (cm >= 0) {
        correction_inverse(pc, carr[cm], N, rho, 0, pinv);
        DB_CHECK(cudaMemcpyAsync(dpinv, pinv.data(), sizeof(double) * pinv.size(),
                                 cudaMemcpyHostToDevice, ds.st));
      }
      a.coh = nullptr; a.flag = nullptr; a.xout = dx; a.p = d.pp; a.pinv = dpinv;
      db_prof_begin(11, 128.0 * (double)R, ds.st);
      db_launch_residual_multifreq(&a, ds.st);
      db_prof_end(ds.st);
      db_count_launch(1);
      DB_CHECK(cudaMemcpyAsync(xc, dx, (size_t)R * 64, cudaMemcpyDeviceToHost, ds.st));
      db_stream_sync(ds.st);  // pinv is rewritten by the next channel
    }
    memcpy(p, pc, sizeof(double) * m);
    std::vector<unsigned char> hf(R);
    DB_CHECK(cudaMemcpyAsync(hf.data(), d.flag, R, cudaMemcpyDeviceToHost, ds.st));
    ds.sync();
    for (long long r = 0; r < R; r++) barr[r].flag = hf[r];
    db_free(dx);
  }
  dirac_b200_destroy(pr);
  return 0;
}
// ---- stochastic calibration of one interval ----------------------------------------------------------
// Device storage for a whole interval (minibatch_mode.cpp:368-506, minibatch_consensus_mode.cpp:453-672):
// the coherencies coh[minibatch][chan][M][4][R] (planar, so that a band of a minibatch is one contiguous
// [nc][M][4][R] block), the data twice, [minibatch][chan][R][4] for the residual kernel and planar
// [minibatch][chan][4][R] for the fits, and two sets of flags: as preset (every later pass re-presets
// the flags on each load) and with the uv cut of the first pass.  With station beams, the beam inputs
// and one set of tables, rebuilt for every (minibatch, channel) and every (minibatch, band).
struct IntervalDev {
  long long R;
  int M, Nchan, tmb;
  // bands (minibatch_mode.cpp:93-116): nper = ceil(Nchan / nsolbw) channels from c0[b], the last the rest
  std::vector<int> c0, nc;
  int nper;
  CohArgs a;                // the staged sky; u, v, w and freqs of the whole interval below
  const double *du, *dv, *dw, *df;
  unsigned char *flag_preset, *flag_cut;
  double2 *xapi, *xpl, *coh;
  size_t nvis;
  const BeamSpec *beam;     // or null
  BeamArgs bg;              // the beam inputs on the device, tables for tmb x nper channels
  const double *tjd;        // [minibatches][tmb] the timeslots' JD
  // band b of minibatch mb, with the uv cut (first pass) or the preset flags
  BandView band(int mb, int b, bool cut) const {
    const size_t mc = (size_t)mb * Nchan + c0[b];
    return {coh + mc * M * 4 * R, xpl + mc * 4 * R, (cut ? flag_cut : flag_preset) + (size_t)mb * R,
            nc[b]};
  }
};

// the bands of one minibatch's tables from the interval's beam inputs: timeslots of minibatch mb,
// channels [c, c + nc) with the coefficient sets from set `set` on
static void interval_beam_tables(DeviceScope &ds, const IntervalDev &iv, int mb, int c, int nc,
                                 size_t set) {
  BeamArgs g = iv.bg;
  g.time_jd = iv.tjd + (size_t)mb * iv.tmb;
  g.freqs = iv.df + c;
  g.Nf = nc;
  if (g.pat_phi) {
    g.pat_phi += set;
    g.pat_theta += set;
  }
  beam_tables(g, ds.st);
}

// the bands, one sky upload, u, v, w, both sets of flags and the data; the coherencies of every
// (minibatch, channel) predicted into device storage with the uv cut of
// precalculate_coherencies_multifreq (predict.c:731-735), or with station beams (beam != null) as
// precalculate_coherencies_multifreq_withbeam predicts them: per channel its own beam tables and
// coefficient set, the uv cut both ways at ph_freq0
static void interval_stage(DeviceScope &ds, IntervalDev &iv, const double *u, const double *v,
                           const double *w, const double *xo, int N, int Nbase, int tmb,
                           int minibatches, const baseline_t *barr, const clus_source_t *carr, int M,
                           const double *freqs, int Nchan, double deltaf, double uvmin, double uvmax,
                           int nsolbw, const BeamSpec *beam) {
  const long long R = (long long)Nbase * tmb;
  iv.R = R; iv.M = M; iv.Nchan = Nchan; iv.tmb = tmb; iv.beam = beam;
  iv.nper = (Nchan + nsolbw - 1) / nsolbw;
  iv.c0.assign(nsolbw, 0);
  iv.nc.assign(nsolbw, 0);
  for (int b = 0, count = 0; b < nsolbw; b++) {
    iv.nc[b] = count + iv.nper < Nchan ? iv.nper : Nchan - count;
    iv.c0[b] = count;
    count += iv.nc[b];
  }
  std::vector<unsigned char> hflag((size_t)minibatches * R);
  for (int mb = 0; mb < minibatches; mb++)
    db_canonical_flags(N, Nbase, tmb, barr + (size_t)mb * R, hflag.data() + (size_t)mb * R);
  CohArgs &a = iv.a;
  a = stage_sky(ds, carr, M, u, v, w, (long long)minibatches * R, freqs, Nchan,
                deltaf / (double)Nchan);
  iv.du = a.u; iv.dv = a.v; iv.dw = a.w; iv.df = a.freqs;
  a.R = R; a.N = N;
  iv.flag_preset = ds.upload(hflag);
  std::vector<unsigned char> hcut;
  if (beam) {  // the beam's uv cut, on the host as the reference-named call makes it
    hcut = hflag;
    for (long long r = 0; r < (long long)minibatches * R; r++)
      if (!hcut[r] && beam_uv_outside(u[r], v[r], beam->ph_freq0, uvmin, uvmax)) hcut[r] = 2;
  }
  iv.flag_cut = ds.upload(beam ? hcut : hflag);
  iv.nvis = (size_t)minibatches * Nchan * R * 4;
  iv.xapi = ds.upload((const double2 *)xo, iv.nvis);
  iv.xpl = ds.alloc<double2>(iv.nvis);
  if (beam) {
    // one set of tables, for the widest band: tmb x nper x S x N entries (72 bytes each at most)
    iv.bg = beam_upload(ds, beam, N, (size_t)tmb * iv.nper * a.beam_S * N);
    iv.bg.src = a.src; iv.bg.S = a.beam_S; iv.bg.T = tmb;
    iv.tjd = ds.upload(beam->time_utc, (size_t)minibatches * tmb);
    // every minibatch has the canonical rows (db_canonical_flags), so one upload of the stations
    std::vector<int> sta;
    upload_row_stations(ds, barr, R, sta, &a);
    db_stream_sync(ds.st);
    a.beam_af = iv.bg.af; a.beam_E = iv.bg.E; a.Nbase = Nbase;
  }
  iv.coh = (double2 *)db_malloc(sizeof(double2) * (size_t)M * iv.nvis);
  for (int mb = 0; mb < minibatches; mb++) {
    a.u = iv.du + (size_t)mb * R; a.v = iv.dv + (size_t)mb * R; a.w = iv.dw + (size_t)mb * R;
    a.flag = beam ? nullptr : iv.flag_cut + (size_t)mb * R;
    for (int c = 0; c < Nchan; c++) {
      const size_t mc = (size_t)mb * Nchan + c;
      db_launch_vis_to_planar(iv.xapi + mc * 4 * R, iv.xpl + mc * 4 * R, R, ds.st);
      if (beam) interval_beam_tables(ds, iv, mb, c, 1, beam_channel_set(beam, c));
      a.freqs = iv.df + c;
      a.Nchan = 1;
      a.uvmin = c == 0 ? uvmin : 0.0;
      a.uvmax = c == Nchan - 1 ? uvmax : 1e300;
      a.coh = iv.coh + mc * M * 4 * R;
      // profile kind 16: u, v, w read and the coherencies written once
      db_prof_begin(16, (double)R * (24.0 + 64.0 * M), ds.st);
      db_launch_coherencies(&a, ds.st);
      db_prof_end(ds.st);
      db_count_launch(2);
    }
  }
}

// residuals of every minibatch and band with the band's solution (calculate_residuals_multifreq) and
// the ccid / rho / phase_only correction, downloaded into xo; frees the coherencies.  With station
// beams, each (minibatch, band) gets the tables calculate_residuals_multifreq_withbeam builds for the
// band's channels: wide-band element beams use the coefficient sets 0 .. nc-1, the band's own channel
// numbers, whatever channel the band starts at (predict_withbeam.c:516,527; DESIGN.md §7 item 19)
static void interval_residuals(DeviceScope &ds, IntervalDev &iv, const baseline_t *barr,
                               const clus_source_t *carr, int N, int M, int minibatches, int nsolbw,
                               const double *pfreq, size_t m, int ccid, double rho, int phase_only,
                               double *xo) {
  CohArgs &a = iv.a;
  const long long R = iv.R;
  a.coh = nullptr; a.flag = nullptr;
  const ResidualTables tb = residual_tables(ds, barr, carr, N, M, residual_coef(carr, M), ccid, &a);
  const int cm = tb.cm;
  a.pinv_nchunk = cm >= 0 ? carr[cm].nchunk : 1;
  double *dp = ds.alloc<double>(tb.npar > 0 ? (size_t)tb.npar : 1);
  double *dpinv = cm >= 0 ? ds.alloc<double>((size_t)8 * N * carr[cm].nchunk) : nullptr;
  std::vector<double> pinv;
  for (int b = 0; b < nsolbw; b++) {
    if (iv.nc[b] == 0) continue;
    DB_CHECK(cudaMemcpyAsync(dp, pfreq + b * m, sizeof(double) * tb.npar, cudaMemcpyHostToDevice,
                             ds.st));
    if (cm >= 0) {
      correction_inverse(pfreq + b * m, carr[cm], N, rho, phase_only, pinv);
      DB_CHECK(cudaMemcpyAsync(dpinv, pinv.data(), sizeof(double) * pinv.size(),
                               cudaMemcpyHostToDevice, ds.st));
    }
    a.p = dp; a.pinv = dpinv; a.freqs = iv.df + iv.c0[b]; a.Nchan = iv.nc[b];
    for (int mb = 0; mb < minibatches; mb++) {
      a.u = iv.du + (size_t)mb * R; a.v = iv.dv + (size_t)mb * R; a.w = iv.dw + (size_t)mb * R;
      a.xout = iv.xapi + ((size_t)mb * iv.Nchan + iv.c0[b]) * 4 * R;
      if (iv.beam) interval_beam_tables(ds, iv, mb, iv.c0[b], iv.nc[b], 0);
      db_prof_begin(11, 128.0 * (double)R * iv.nc[b], ds.st);
      db_launch_residual_multifreq(&a, ds.st);
      db_prof_end(ds.st);
      db_count_launch(1);
    }
    db_stream_sync(ds.st);  // dp and dpinv are rewritten by the next band
  }
  DB_CHECK(cudaMemcpyAsync(xo, iv.xapi, sizeof(double2) * iv.nvis, cudaMemcpyDeviceToHost, ds.st));
  ds.sync();
  db_free(iv.coh);
  iv.coh = nullptr;
}

static bool bands_refused(const char *fn, int nsolbw, int Nchan) {
  if (nsolbw >= 1 && nsolbw <= Nchan) return false;
  fprintf(stderr, "%s: nsolbw = %d bands of Nchan = %d channels; the driver clamps nsolbw to Nchan, "
                  "this call takes 1 <= nsolbw <= Nchan\n", fn, nsolbw, Nchan);
  return true;
}

// the beam arguments of the _withbeam interval calls, checked before any device work: -1 with a
// message (the reference-named _withbeam calls exit instead)
bool beam_refused(const char *fn, const BeamSpec &b, int N, int Nchan) {
  if (b.doBeam == DOBEAM_NONE) return false;
  if (b.doBeam < DOBEAM_NONE || b.doBeam > DOBEAM_ELEMENT_WB) {
    fprintf(stderr, "%s: doBeam = %d is not a beam mode this call takes (0..6; the lunar element "
                    "beam needs CSPICE)\n", fn, b.doBeam);
    return true;
  }
  if (!b.longitude || !b.latitude || !b.time_utc) {
    fprintf(stderr, "%s: doBeam = %d without station longitudes, latitudes or timeslot times\n", fn,
            b.doBeam);
    return true;
  }
  if (beam_array(b.doBeam)) {
    if (b.bf_type != STAT_SINGLE && b.bf_type != STAT_TILE) {
      fprintf(stderr, "%s: the array beam (doBeam = %d) needs bf_type STAT_SINGLE or STAT_TILE, "
                      "not %d\n", fn, b.doBeam, b.bf_type);
      return true;
    }
    bool missing = !b.Nelem || !b.xx || !b.yy || !b.zz;
    for (int n = 0; n < N && !missing; n++) missing = !b.xx[n] || !b.yy[n] || !b.zz[n];
    if (missing) {
      fprintf(stderr, "%s: the array beam (doBeam = %d) needs Nelem and the element positions xx, "
                      "yy, zz of every station\n", fn, b.doBeam);
      return true;
    }
  }
  if (beam_element(b.doBeam)) {
    const elementcoeff *ec = b.ecoeff;
    if (!ec || !ec->pattern_phi || !ec->pattern_theta || !ec->preamble) {
      fprintf(stderr, "%s: the element beam (doBeam = %d) needs coefficient tables "
                      "(set_elementcoeffs)\n", fn, b.doBeam);
      return true;
    }
    if (beam_wide(b.doBeam) && ec->Nf < Nchan) {
      fprintf(stderr, "%s: the wide-band element beam (doBeam = %d) needs one coefficient set per "
                      "channel (set_elementcoeffs_wb over %d channels), the tables hold %d\n", fn,
              b.doBeam, Nchan, ec->Nf);
      return true;
    }
  }
  return false;
}

// The stochastic calibration of one interval (minibatch_mode.cpp:368-506) in one call: epochs x
// minibatches x bands of the minibatch LBFGS; the uv cut holds in the first epoch only.
static int stochastic_interval_impl(const char *fn, double *u, double *v, double *w, double *xo, int N,
                                    int Nbase, int tmb, int minibatches, baseline_t *barr,
                                    clus_source_t *carr, int M, int Mt, double *freqs, int Nchan,
                                    double deltaf, double uvmin, double uvmax, const BeamSpec *beam,
                                    int nsolbw, int nepochs, int max_lbfgs, int lbfgs_m,
                                    double robust_nu, persistent_data_t *pt, double *pfreq, int ccid,
                                    double rho, int phase_only, double *res_00, double *res_01) {
  if (bands_refused(fn, nsolbw, Nchan)) return -1;
  if (beam && beam_refused(fn, *beam, N, Nchan)) return -1;
  if (beam && beam->doBeam == DOBEAM_NONE) beam = nullptr;
  const size_t m = (size_t)8 * N * Mt;
  DeviceScope ds;
  IntervalDev iv;
  interval_stage(ds, iv, u, v, w, xo, N, Nbase, tmb, minibatches, barr, carr, M, freqs, Nchan, deltaf,
                 uvmin, uvmax, nsolbw, beam);
  BandDev *bd = db_band_create(N, Nbase, tmb, carr, M, Mt, iv.nper, ds.st);
  for (int ep = 0; ep < nepochs; ep++)
    for (int mb = 0; mb < minibatches; mb++)
      for (int b = 0; b < nsolbw; b++) {
        const size_t o = ((size_t)ep * minibatches + mb) * nsolbw + b;
        db_band_fit(bd, iv.band(mb, b, ep == 0), pfreq + b * m, nullptr, nullptr, nullptr, max_lbfgs,
                    lbfgs_m, robust_nu, res_00 + o, res_01 + o, pt + b);
      }
  db_band_destroy(bd);
  interval_residuals(ds, iv, barr, carr, N, M, minibatches, nsolbw, pfreq, m, ccid, rho, phase_only,
                     xo);
  return 0;
}
extern "C" int dirac_b200_stochastic_interval(double *u, double *v, double *w, double *xo, int N,
                                              int Nbase, int tmb, int minibatches, baseline_t *barr,
                                              clus_source_t *carr, int M, int Mt, double *freqs,
                                              int Nchan, double deltaf, double uvmin, double uvmax,
                                              int nsolbw, int nepochs, int max_lbfgs, int lbfgs_m,
                                              double robust_nu, persistent_data_t *pt,
                                              double *pfreq, int ccid, double rho, int phase_only,
                                              double *res_00, double *res_01) {
  return stochastic_interval_impl("dirac_b200_stochastic_interval", u, v, w, xo, N, Nbase, tmb,
                                  minibatches, barr, carr, M, Mt, freqs, Nchan, deltaf, uvmin, uvmax,
                                  nullptr, nsolbw, nepochs, max_lbfgs, lbfgs_m, robust_nu, pt, pfreq,
                                  ccid, rho, phase_only, res_00, res_01);
}
// the same with station beams (minibatch_mode.cpp:403-427,485-500 with doBeam > 0); time_utc
// [minibatches][tmb]
extern "C" int dirac_b200_stochastic_interval_withbeam(
    double *u, double *v, double *w, double *xo, int N, int Nbase, int tmb, int minibatches,
    baseline_t *barr, clus_source_t *carr, int M, int Mt, double *freqs, int Nchan, double deltaf,
    double uvmin, double uvmax, int bf_type, double b_ra0, double b_dec0, double ph_ra0,
    double ph_dec0, double ph_freq0, double *longitude, double *latitude, double *time_utc,
    int *Nelem, double **xx, double **yy, double **zz, elementcoeff *ecoeff, int doBeam, int nsolbw,
    int nepochs, int max_lbfgs, int lbfgs_m, double robust_nu, persistent_data_t *pt, double *pfreq,
    int ccid, double rho, int phase_only, double *res_00, double *res_01) {
  const BeamSpec b = {bf_type, b_ra0, b_dec0, ph_ra0, ph_dec0, ph_freq0, longitude, latitude,
                      time_utc, tmb, Nelem, xx, yy, zz, ecoeff, doBeam};
  return stochastic_interval_impl("dirac_b200_stochastic_interval_withbeam", u, v, w, xo, N, Nbase,
                                  tmb, minibatches, barr, carr, M, Mt, freqs, Nchan, deltaf, uvmin,
                                  uvmax, &b, nsolbw, nepochs, max_lbfgs, lbfgs_m, robust_nu, pt, pfreq,
                                  ccid, rho, phase_only, res_00, res_01);
}

// The stochastic calibration with spectral consensus over the bands (minibatch_consensus_mode.cpp:
// 453-672) in one call: nadmm x epochs x minibatches; per minibatch every band's fit with the
// consensus terms y = Y_b, z = B_b Z, rho_b, then the ADMM step of dirac_b200_consensus_bands_update.
// The coherencies are predicted once, with the uv cut, in (admm 0, epoch 0) (:491); Y starts from zero
// and res_0 / res_1 from 0 (:453-454); Z is the caller's.
static int stochastic_consensus_interval_impl(
    const char *fn, double *u, double *v, double *w, double *xo, int N, int Nbase, int tmb,
    int minibatches, baseline_t *barr, clus_source_t *carr, int M, int Mt, double *freqs, int Nchan,
    double deltaf, double uvmin, double uvmax, const BeamSpec *beam, int nsolbw, int nepochs,
    int max_lbfgs, int lbfgs_m, double robust_nu, persistent_data_t *pt, double *pfreq, int ccid,
    double rho, int phase_only, int nadmm, int Npoly, double *B, double *Bi, double *rhok, double *Z,
    int use_global, double *res_00, double *res_01, double *res_0, double *res_1, int *fband) {
  if (bands_refused(fn, nsolbw, Nchan)) return -1;
  if (nadmm < 1 || Npoly < 1) {
    fprintf(stderr, "%s: nadmm = %d ADMM iterations, Npoly = %d polynomial terms; each must be at "
                    "least 1\n", fn, nadmm, Npoly);
    return -1;
  }
  if (beam && beam_refused(fn, *beam, N, Nchan)) return -1;
  if (beam && beam->doBeam == DOBEAM_NONE) beam = nullptr;
  const size_t m = (size_t)8 * N * Mt;
  DeviceScope ds;
  IntervalDev iv;
  interval_stage(ds, iv, u, v, w, xo, N, Nbase, tmb, minibatches, barr, carr, M, freqs, Nchan, deltaf,
                 uvmin, uvmax, nsolbw, beam);
  std::vector<double> Y((size_t)nsolbw * m, 0.0), z(m);
  *res_0 = *res_1 = 0.0;
  BandDev *bd = db_band_create(N, Nbase, tmb, carr, M, Mt, iv.nper, ds.st);
  for (int ad = 0; ad < nadmm; ad++)
    for (int ep = 0; ep < nepochs; ep++)
      for (int mb = 0; mb < minibatches; mb++) {
        const size_t o = (((size_t)ad * nepochs + ep) * minibatches + mb) * nsolbw;
        for (int b = 0; b < nsolbw; b++) {
          db_consensus_bz(Z, B + (size_t)b * Npoly, N, Mt, Npoly, z.data());
          db_band_fit(bd, iv.band(mb, b, ad == 0 && ep == 0), pfreq + b * m, Y.data() + b * m,
                      z.data(), rhok + (size_t)b * Mt, max_lbfgs, lbfgs_m, robust_nu, res_00 + o + b,
                      res_01 + o + b, pt + b);
        }
        dirac_b200_consensus_bands_update(N, Mt, nsolbw, Npoly, res_00 + o, res_01 + o, pfreq, B, Bi,
                                          rhok, res_0, res_1, Y.data(), Z, fband);
      }
  db_band_destroy(bd);
  if (use_global)  // -U: every band's solution is its B_b Z (:608-620)
    for (int b = 0; b < nsolbw; b++)
      db_consensus_bz(Z, B + (size_t)b * Npoly, N, Mt, Npoly, pfreq + b * m);
  interval_residuals(ds, iv, barr, carr, N, M, minibatches, nsolbw, pfreq, m, ccid, rho, phase_only,
                     xo);
  return 0;
}
extern "C" int dirac_b200_stochastic_consensus_interval(
    double *u, double *v, double *w, double *xo, int N, int Nbase, int tmb, int minibatches,
    baseline_t *barr, clus_source_t *carr, int M, int Mt, double *freqs, int Nchan, double deltaf,
    double uvmin, double uvmax, int nsolbw, int nepochs, int max_lbfgs, int lbfgs_m, double robust_nu,
    persistent_data_t *pt, double *pfreq, int ccid, double rho, int phase_only, int nadmm, int Npoly,
    double *B, double *Bi, double *rhok, double *Z, int use_global, double *res_00, double *res_01,
    double *res_0, double *res_1, int *fband) {
  return stochastic_consensus_interval_impl(
      "dirac_b200_stochastic_consensus_interval", u, v, w, xo, N, Nbase, tmb, minibatches, barr, carr,
      M, Mt, freqs, Nchan, deltaf, uvmin, uvmax, nullptr, nsolbw, nepochs, max_lbfgs, lbfgs_m,
      robust_nu, pt, pfreq, ccid, rho, phase_only, nadmm, Npoly, B, Bi, rhok, Z, use_global, res_00,
      res_01, res_0, res_1, fband);
}
// the same with station beams (minibatch_consensus_mode.cpp:493-506,648-663 with doBeam > 0)
extern "C" int dirac_b200_stochastic_consensus_interval_withbeam(
    double *u, double *v, double *w, double *xo, int N, int Nbase, int tmb, int minibatches,
    baseline_t *barr, clus_source_t *carr, int M, int Mt, double *freqs, int Nchan, double deltaf,
    double uvmin, double uvmax, int bf_type, double b_ra0, double b_dec0, double ph_ra0,
    double ph_dec0, double ph_freq0, double *longitude, double *latitude, double *time_utc,
    int *Nelem, double **xx, double **yy, double **zz, elementcoeff *ecoeff, int doBeam, int nsolbw,
    int nepochs, int max_lbfgs, int lbfgs_m, double robust_nu, persistent_data_t *pt, double *pfreq,
    int ccid, double rho, int phase_only, int nadmm, int Npoly, double *B, double *Bi, double *rhok,
    double *Z, int use_global, double *res_00, double *res_01, double *res_0, double *res_1,
    int *fband) {
  const BeamSpec b = {bf_type, b_ra0, b_dec0, ph_ra0, ph_dec0, ph_freq0, longitude, latitude,
                      time_utc, tmb, Nelem, xx, yy, zz, ecoeff, doBeam};
  return stochastic_consensus_interval_impl(
      "dirac_b200_stochastic_consensus_interval_withbeam", u, v, w, xo, N, Nbase, tmb, minibatches,
      barr, carr, M, Mt, freqs, Nchan, deltaf, uvmin, uvmax, &b, nsolbw, nepochs, max_lbfgs, lbfgs_m,
      robust_nu, pt, pfreq, ccid, rho, phase_only, nadmm, Npoly, B, Bi, rhok, Z, use_global, res_00,
      res_01, res_0, res_1, fband);
}
// Dirac_radio.h:666 (residual.c:1620-1740): simulation with solutions

// The federated stochastic slave's interval (sagecal_stochastic_slave.cpp:650-881) for one measurement
// set on this rank, with the master's exchange (sagecal_stochastic_master.cpp:334-354) done on every
// rank after one all-reduce.  The coherencies are predicted once; the slave predicts them in every
// pass with the reloaded flags and the uv cut (:675-723), so every pass here fits the cut rows' flags
// (DESIGN.md 7 items 24, 25).  Y, X and Zavg start from zero; Z is the caller's.
extern "C" int dirac_b200_stochastic_federated_interval(
    double *u, double *v, double *w, double *xo, int N, int Nbase, int tmb, int minibatches,
    baseline_t *barr, clus_source_t *carr, int M, int Mt, double *freqs, int Nchan, double deltaf,
    double uvmin, double uvmax, int nsolbw, int nepochs, int max_lbfgs, int lbfgs_m, double robust_nu,
    persistent_data_t *pt, double *pfreq, int ccid, double rho, int phase_only, int nadmm, int Npoly,
    double *B, double *Bi, double *rhok, double *alphak, double *Z, int use_global, int randomize,
    int rank, int world, dirac_b200_allreduce_fn allreduce, void *user, double *res_00,
    double *res_01, double *res_0, double *res_1, int *fband) {
  const char *fn = "dirac_b200_stochastic_federated_interval";
  if (bands_refused(fn, nsolbw, Nchan)) return -1;
  if (nadmm < 1 || Npoly < 1) {
    fprintf(stderr, "%s: nadmm = %d ADMM iterations, Npoly = %d polynomial terms; each must be at "
                    "least 1\n", fn, nadmm, Npoly);
    return -1;
  }
  if (world < 1 || world > 64 || rank < 0 || rank >= world) {
    fprintf(stderr, "%s: rank %d of world %d; 0 <= rank < world <= 64\n", fn, rank, world);
    return -1;
  }
  if (world > 1 && !allreduce && db_nccl_world() != world) {
    fprintf(stderr, "%s: world %d without an exchange: give a callback or call dirac_b200_nccl_init "
                    "with %d ranks first\n", fn, world, world);
    return -1;
  }
  const size_t m = (size_t)8 * N * Mt, L = m * Npoly;
  DeviceScope ds;
  IntervalDev iv;
  interval_stage(ds, iv, u, v, w, xo, N, Nbase, tmb, minibatches, barr, carr, M, freqs, Nchan, deltaf,
                 uvmin, uvmax, nsolbw, nullptr);
  std::vector<double> Y((size_t)nsolbw * m, 0.0), z(m), X(L, 0.0), Zavg(L, 0.0), ex((size_t)world * L + Mt);
  // [world][L] solutions | [Mt] rank 0's draws
  double *dex = ds.alloc<double>(ex.size());
  int *dcr = ds.alloc<int>(Mt);
  std::vector<int> cr(Mt);
  BandDev *bd = db_band_create(N, Nbase, tmb, carr, M, Mt, iv.nper, ds.st);
  for (int ad = 0; ad < nadmm; ad++) {
    for (int ep = 0; ep < nepochs; ep++)
      for (int mb = 0; mb < minibatches; mb++) {
        const size_t o = (((size_t)ad * nepochs + ep) * minibatches + mb) * nsolbw;
        for (int b = 0; b < nsolbw; b++) {
          db_consensus_bz(Z, B + (size_t)b * Npoly, N, Mt, Npoly, z.data());
          db_band_fit(bd, iv.band(mb, b, true), pfreq + b * m, Y.data() + b * m, z.data(),
                      rhok + (size_t)b * Mt, max_lbfgs, lbfgs_m, robust_nu, res_00 + o + b,
                      res_01 + o + b, pt + b);
        }
        dirac_b200_federated_bands_update(N, Mt, nsolbw, Npoly, ad, res_00 + o, res_01 + o, pfreq, B,
                                          Bi, rhok, alphak, Zavg.data(), X.data(), res_0, res_1,
                                          Y.data(), Z, fband);
      }
    // the exchange (:857-880): gather every rank's Z and rank 0's draws, average on every rank
    std::fill(ex.begin(), ex.end(), 0.0);
    std::copy(Z, Z + L, ex.begin() + (size_t)rank * L);
    if (rank == 0)
      for (int k = 0; k < Mt; k++) ex[(size_t)world * L + k] = randomize ? (double)(rand() % world) : 0.0;
    DB_CHECK(cudaMemcpyAsync(dex, ex.data(), sizeof(double) * ex.size(), cudaMemcpyHostToDevice, ds.st));
    if (world > 1) db_allreduce_stream(allreduce, user, dex, (long long)ex.size(), ds.st);
    DB_CHECK(cudaMemcpyAsync(ex.data() + (size_t)world * L, dex + (size_t)world * L,
                             sizeof(double) * Mt, cudaMemcpyDeviceToHost, ds.st));
    db_stream_sync(ds.st);
    for (int k = 0; k < Mt; k++) cr[k] = (int)ex[(size_t)world * L + k];
    DB_CHECK(cudaMemcpyAsync(dcr, cr.data(), sizeof(int) * Mt, cudaMemcpyHostToDevice, ds.st));
    if (db_manifold_projectback(dex, N * Npoly, Mt, world, ad == 0 ? 10 : 2, dcr, ds.st)) exit(1);
    DB_CHECK(cudaMemcpyAsync(Zavg.data(), dex + (size_t)rank * L, sizeof(double) * L,
                             cudaMemcpyDeviceToHost, ds.st));
    db_stream_sync(ds.st);
    // X_k += alpha_k (Z_k - Zavg_k)
    for (int k = 0; k < Mt; k++)
      for (size_t i = 0; i < (size_t)8 * N * Npoly; i++) {
        const size_t j = (size_t)k * 8 * N * Npoly + i;
        X[j] += alphak[k] * (Z[j] - Zavg[j]);
      }
  }
  db_band_destroy(bd);
  if (use_global)
    for (int b = 0; b < nsolbw; b++)
      db_consensus_bz(Z, B + (size_t)b * Npoly, N, Mt, Npoly, pfreq + b * m);
  interval_residuals(ds, iv, barr, carr, N, M, minibatches, nsolbw, pfreq, m, ccid, rho, phase_only,
                     xo);
  return 0;
}

extern "C" int predict_visibilities_multifreq_withsol(double *u, double *v, double *w, double *p,
                                                      double *x, int *ignorelist, int N, int Nbase,
                                                      int tilesz, baseline_t *barr,
                                                      clus_source_t *carr, int M, double *freqs,
                                                      int Nchan, double fdelta, double tdelta,
                                                      double dec0, int Nt, int add_to_data, int ccid,
                                                      double rho, int phase_only) {
  (void)tdelta; (void)dec0; (void)Nt;
  return residuals_multifreq_impl(u, v, w, p, x, N, Nbase, tilesz, barr, carr, M, freqs, Nchan, fdelta,
                                  simul_coef(ignorelist, M, add_to_data), add_to_data == 1, ccid,
                                  rho, phase_only, nullptr);
}
// Dirac_radio.h:490,529 (predict_withbeam.c:1452-1680, predict_withbeam_cuda.c:2905-3130): the same
// with per-channel station beams; the correction by cluster ccid is applied once, after all clusters
extern "C" int predict_visibilities_multifreq_withsol_withbeam(
    double *u, double *v, double *w, double *p, double *x, int *ignorelist, int N, int Nbase,
    int tilesz, baseline_t *barr, clus_source_t *carr, int M, double *freqs, int Nchan, double fdelta,
    double tdelta, double dec0, int bf_type, double b_ra0, double b_dec0, double ph_ra0,
    double ph_dec0, double ph_freq0, double *longitude, double *latitude, double *time_utc,
    int *Nelem, double **xx, double **yy, double **zz, elementcoeff *ecoeff, int doBeam, int Nt,
    int add_to_data, int ccid, double rho, int phase_only) {
  (void)tdelta; (void)dec0; (void)Nt;
  BeamSpec b = {bf_type, b_ra0, b_dec0, ph_ra0, ph_dec0, ph_freq0, longitude, latitude, time_utc,
                tilesz, Nelem, xx, yy, zz, ecoeff, doBeam};
  return residuals_multifreq_impl(u, v, w, p, x, N, Nbase, tilesz, barr, carr, M, freqs, Nchan, fdelta,
                                  simul_coef(ignorelist, M, add_to_data), add_to_data == 1, ccid,
                                  rho, phase_only, &b);
}
extern "C" int predict_visibilities_withsol_withbeam_gpu(
    double *u, double *v, double *w, double *p, double *x, int *ignorelist, int N, int Nbase,
    int tilesz, baseline_t *barr, clus_source_t *carr, int M, double *freqs, int Nchan, double fdelta,
    double tdelta, double dec0, int bf_type, double b_ra0, double b_dec0, double ph_ra0,
    double ph_dec0, double ph_freq0, double *longitude, double *latitude, double *time_utc,
    int *Nelem, double **xx, double **yy, double **zz, elementcoeff *ecoeff, int doBeam, int Nt,
    int add_to_data, int ccid, double rho, int phase_only) {
  return predict_visibilities_multifreq_withsol_withbeam(
      u, v, w, p, x, ignorelist, N, Nbase, tilesz, barr, carr, M, freqs, Nchan, fdelta, tdelta, dec0,
      bf_type, b_ra0, b_dec0, ph_ra0, ph_dec0, ph_freq0, longitude, latitude, time_utc, Nelem, xx, yy,
      zz, ecoeff, doBeam, Nt, add_to_data, ccid, rho, phase_only);
}
// Dirac_radio.h:489,525 (predict_withbeam.c:1989-2315): per-channel station beams in the re-prediction
extern "C" int calculate_residuals_multifreq_withbeam(
    double *u, double *v, double *w, double *p, double *x, int N, int Nbase, int tilesz,
    baseline_t *barr, clus_source_t *carr, int M, double *freqs, int Nchan, double fdelta,
    double tdelta, double dec0, int bf_type, double b_ra0, double b_dec0, double ph_ra0,
    double ph_dec0, double ph_freq0, double *longitude, double *latitude, double *time_utc,
    int *Nelem, double **xx, double **yy, double **zz, elementcoeff *ecoeff, int doBeam, int Nt,
    int ccid, double rho, int phase_only) {
  (void)tdelta; (void)dec0; (void)Nt;
  BeamSpec b = {bf_type, b_ra0, b_dec0, ph_ra0, ph_dec0, ph_freq0, longitude, latitude, time_utc,
                tilesz, Nelem, xx, yy, zz, ecoeff, doBeam};
  return residuals_multifreq_impl(u, v, w, p, x, N, Nbase, tilesz, barr, carr, M, freqs, Nchan, fdelta,
                                  residual_coef(carr, M), false, ccid, rho, phase_only, &b);
}
extern "C" int calculate_residuals_multifreq_withbeam_gpu(
    double *u, double *v, double *w, double *p, double *x, int N, int Nbase, int tilesz,
    baseline_t *barr, clus_source_t *carr, int M, double *freqs, int Nchan, double fdelta,
    double tdelta, double dec0, int bf_type, double b_ra0, double b_dec0, double ph_ra0,
    double ph_dec0, double ph_freq0, double *longitude, double *latitude, double *time_utc,
    int *Nelem, double **xx, double **yy, double **zz, elementcoeff *ecoeff, int doBeam, int Nt,
    int ccid, double rho, int phase_only) {
  return calculate_residuals_multifreq_withbeam(u, v, w, p, x, N, Nbase, tilesz, barr, carr, M, freqs,
                                                Nchan, fdelta, tdelta, dec0, bf_type, b_ra0, b_dec0,
                                                ph_ra0, ph_dec0, ph_freq0, longitude, latitude,
                                                time_utc, Nelem, xx, yy, zz, ecoeff, doBeam, Nt, ccid,
                                                rho, phase_only);
}
