// Per-source and per-station arithmetic of the coherency kernels (kernels_coh.cu), host-callable so
// that oracle/coh_math_check.cu can run exactly this code on the CPU against the reference's
// shapelet_contrib / arraybeam / element_beam (test infrastructure; the product only runs it on the
// device).
#pragma once
#include <math.h>

#include "internal.cuh"
#include "coh.h"

#ifdef __CUDA_ARCH__
#define COH_UNROLL1 _Pragma("unroll 1")
#else
#define COH_UNROLL1
#endif

// ---- per-source term ------------------------------------------------------------------------------
// bb[n] = phi_n(x) = H_n(x) exp(-x^2/2) / sqrt(2^(n+1) n!), n < n0 (calculate_uv_mode_vectors_scalar,
// shapelet.c:84-95): the recursion of shapelet_factor below, for the diffuse cluster's rows
// (diffuse_math.cuh).  shapelet_factor keeps its own copy: routed through this helper, nvcc schedules
// the sky-prediction kernel differently.
__host__ __device__ __forceinline__ void shapelet_basis(double x, int n0, double *bb) {
  const double ex = exp(-0.5 * x * x);
  double hm2 = 1.0, hm1 = 2.0 * x, fact = 1.0, p2 = 2.0;  // H_0, H_1, n!, 2^(n+1)
  for (int n = 0; n < n0; n++) {
    double h;
    if (n == 0) h = 1.0;
    else if (n == 1) h = hm1;
    else {
      h = 2.0 * x * hm1 - 2.0 * (double)(n - 1) * hm2;
      hm2 = hm1;
      hm1 = h;
    }
    if (n > 0) fact *= (double)n;
    bb[n] = h * ex / sqrt(p2 * fact);
    p2 *= 2.0;
  }
}
// mode vector entry of mode (n1, n2): sign * phi_n1(-u beta) phi_n2(v beta); *odd: the mode is
// imaginary (calculate_uv_mode_vectors_scalar, shapelet.c:109-127)
__host__ __device__ __forceinline__ double shapelet_mode_coeff(const double *bu, const double *bv, int n1,
                                                      int n2, int *odd) {
  *odd = (n1 + n2) & 1;
  const int sg = (((n1 + n2 - *odd) / 2) & 1) ? -1 : 1;
  return (sg < 0 ? -bu[n1] : bu[n1]) * bv[n2];
}

// phase * |sinc| smearing * shape factor for one source at one frequency (predict.c:411-470)
// Fourier-plane value of a shapelet source (shapelet_contrib + calculate_uv_mode_vectors_scalar,
// shapelet.c:50-190): sum over the n0 x n0 modes of coeff * phi_n1(-ut beta) phi_n2(vt beta), odd
// n1+n2 imaginary, phi_n(x) = H_n(x) exp(-x^2/2) / sqrt(2^(n+1) n!), times 2 pi / (eX eY)
static __host__ __device__ __noinline__ double2 shapelet_factor(const DevSource &s, const double *modes, double uf,
                                                double vf, double wf) {
  double up, vp;
  if (s.use_projection != 0.0) {
    up = -uf * s.cxi + vf * s.cphi * s.sxi - wf * s.sphi * s.sxi;
    vp = -uf * s.sxi - vf * s.cphi * s.cxi + wf * s.sphi * s.cxi;
  } else {
    up = uf;
    vp = vf;
  }
  const double a = 1.0 / s.eX, b = 1.0 / s.eY;
  double sph, cph;
  sincos(s.eP, &sph, &cph);
  const double ut = a * (cph * up - sph * vp);
  const double vt = b * (sph * up + cph * vp);
  const int n0 = (int)s.sh_n0;
  double bu[COH_SHAPELET_MAX_N0], bv[COH_SHAPELET_MAX_N0];
COH_UNROLL1
  for (int side = 0; side < 2; side++) {
    const double x = (side == 0 ? -ut : vt) * s.sh_beta;
    const double ex = exp(-0.5 * x * x);
    double *bb = side == 0 ? bu : bv;
    double hm2 = 1.0, hm1 = 2.0 * x, fact = 1.0, p2 = 2.0;  // H_0, H_1, n!, 2^(n+1)
    for (int n = 0; n < n0; n++) {
      double h;
      if (n == 0) h = 1.0;
      else if (n == 1) h = hm1;
      else {
        h = 2.0 * x * hm1 - 2.0 * (double)(n - 1) * hm2;
        hm2 = hm1;
        hm1 = h;
      }
      if (n > 0) fact *= (double)n;
      bb[n] = h * ex / sqrt(p2 * fact);
      p2 *= 2.0;
    }
  }
  const double *md = modes + (long long)s.sh_off;
  double re = 0.0, im = 0.0;
  for (int n2 = 0; n2 < n0; n2++)
    for (int n1 = 0; n1 < n0; n1++) {
      const int odd = (n1 + n2) & 1;
      const int sg = (((n1 + n2 - odd) / 2) & 1) ? -1 : 1;
      const double av = (sg < 0 ? -bu[n1] : bu[n1]) * bv[n2];
      const double c = md[n2 * n0 + n1] * av;
      if (odd) im += c;
      else re += c;
    }
  const double sc = 2.0 * M_PI * a * b;
  return make_double2(sc * re, sc * im);
}

__host__ __device__ __forceinline__ double2 source_phase(const DevSource &s, const double *modes, double u,
                                                double v, double w, double freq, double fdelta2) {
  const double G = 2.0 * M_PI * (u * s.ll + v * s.mm + w * s.nn);
  double sp, cp;
  sincos(G * freq, &sp, &cp);
  double fac = 1.0;
  if (G != 0.0) {
    const double sm = G * fdelta2;
    fac = fabs(sin(sm) / sm);
  }
  double2 ph = make_double2(cp * fac, sp * fac);
  const int st = (int)s.stype;
  if (st == STYPE_SHAPELET_) {
    const double2 sf = shapelet_factor(s, modes, u * freq, v * freq, w * freq);
    ph = make_double2(ph.x * sf.x - ph.y * sf.y, ph.x * sf.y + ph.y * sf.x);
  } else if (st != STYPE_POINT_) {
    const double uf = u * freq, vf = v * freq, wf = w * freq;
    double up, vp;
    if (st == STYPE_GAUSSIAN_ && s.use_projection == 0.0) {
      up = uf;
      vp = vf;
    } else {
      up = uf * s.cxi - vf * s.cphi * s.sxi + wf * s.sphi * s.sxi;
      vp = uf * s.sxi + vf * s.cphi * s.cxi - wf * s.sphi * s.cxi;
    }
    double shape = 1.0;
    if (st == STYPE_GAUSSIAN_) {
      double sph, cph;
      sincos(s.eP, &sph, &cph);
      const double ut = s.eX * (cph * up - sph * vp);
      const double vt = s.eY * (sph * up + cph * vp);
      shape = exp(-2.0 * M_PI * M_PI * (ut * ut + vt * vt));
    } else if (st == STYPE_DISK_) {
      shape = j1(sqrt(up * up + vp * vp) * s.eX * 2.0 * M_PI);
    } else if (st == STYPE_RING_) {
      shape = j0(sqrt(up * up + vp * vp) * s.eX * 2.0 * M_PI);
    }
    ph.x *= shape;
    ph.y *= shape;
  }
  return ph;
}

__host__ __device__ __forceinline__ void add_stokes(double2 *C, double2 ph, double I, double Q, double U,
                                           double V) {
  // C0 += ph (I+Q); C1 += ph (U + iV); C2 += ph (U - iV); C3 += ph (I-Q)   (predict.c:466-476)
  const double2 II = make_double2(ph.x * I, ph.y * I), QQ = make_double2(ph.x * Q, ph.y * Q);
  const double2 UU = make_double2(ph.x * U, ph.y * U), VV = make_double2(ph.x * V, ph.y * V);
  C[0].x += II.x + QQ.x;  C[0].y += II.y + QQ.y;
  C[1].x += UU.x - VV.y;  C[1].y += UU.y + VV.x;
  C[2].x += UU.x + VV.y;  C[2].y += UU.y - VV.x;
  C[3].x += II.x - QQ.x;  C[3].y += II.y - QQ.y;
}

// flux at frequency f with the three-term log-spectral index (residual.c:1177-1210)
__host__ __device__ __forceinline__ double spec_flux(double s0, double tempfr) {
  if (s0 > 0.0) return exp(log(s0) + tempfr);
  return (s0 == 0.0) ? 0.0 : -exp(log(-s0) + tempfr);
}

// ---- station beam tables ----------------------------------------------------------------------------
// JD -> Greenwich mean sidereal angle in degrees (jd2gmst, transforms.c:139-146)
__host__ __device__ __forceinline__ double jd2gmst_deg(double time_jd) {
  const double t = (time_jd - 2451545.0) / 36525.0;
  const double theta =
      67310.54841 + t * ((876600.0 * 3600.0 + 8640184.812866) + t * (0.093104 - (6.2 * 10e-6) * t));
  return fmod(fmod(theta, 86400.0 * (theta / fabs(theta))) / 240.0, 360.0);
}
// (ra, dec) -> (az, el) at a station (radec2azel_gmst, transforms.c:157-180)
__host__ __device__ __forceinline__ void radec2azel(double ra, double dec, double lon, double lat,
                                           double gmst, double *az, double *el) {
  const double lst = gmst + lon * 180.0 * M_1_PI;
  const double LHA = fmod(lst - ra * 180.0 * M_1_PI, 360.0);
  double sinlat, coslat, sindec, cosdec, sinL, cosL;
  sincos(lat, &sinlat, &coslat);
  sincos(dec, &sindec, &cosdec);
  sincos(LHA * M_PI / 180.0, &sinL, &cosL);
  const double tmp = sinlat * sindec + coslat * cosdec * cosL;
  *el = asin(tmp);
  double sinel, cosel;
  sincos(*el, &sinel, &cosel);
  double a = fmod(atan2(-sinL * cosdec / cosel, (sindec - sinel * sinlat) / (cosel * coslat)),
                  2.0 * M_PI);
  if (a < 0) a += 2.0 * M_PI;
  *az = a;
}
// generalised Laguerre polynomial L_p^q(x) (L_g1, elementbeam.c:341-356)
__host__ __device__ __forceinline__ double laguerre(int p, int q, double x) {
  if (p == 0) return 1.0;
  if (p == 1) return 1.0 - x + (double)q;
  double Lp = 0.0, Lp1 = 1.0 - x + (double)q, Lp2 = 1.0;
  for (int i = 2; i <= p; i++) {
    const double p1 = 1.0 / (double)i;
    Lp = (2.0 + p1 * ((double)q - 1.0 - x)) * Lp1 - (1.0 + p1 * (q - 1)) * Lp2;
    Lp2 = Lp1;
    Lp1 = Lp;
  }
  return Lp;
}
// element pattern (theta, phi components) at zenith angle r and azimuth th (eval_elementcoeffs[_wb],
// elementbeam.c:384-460); coefficient set `fi` of the wide-band tables
__host__ __device__ __forceinline__ void element_eval(const BeamArgs &a, double r, double th, int fi,
                                             double2 *e_theta, double2 *e_phi) {
  const double rb = pow(r / a.ecbeta, 2);
  const double ex = exp(-0.5 * rb);
  double2 ph = make_double2(0.0, 0.0), tt = make_double2(0.0, 0.0);
  int idx = 0;
  for (int n = 0; n < a.ecM; n++)
    for (int m = -n; m <= n; m += 2) {
      const int absm = m >= 0 ? m : -m;
      const double Lg = laguerre((n - absm) / 2, absm, rb);
      const double rm = pow(M_PI_4 + r, (double)absm);
      double s, c;
      sincos(-(double)m * th, &s, &c);
      const double pr = rm * Lg * ex * a.preamble[idx];
      const double2 basis = make_double2(pr * c, pr * s);
      cfma(ph, a.pat_phi[(size_t)fi * a.ecNmodes + idx], basis);
      cfma(tt, a.pat_theta[(size_t)fi * a.ecNmodes + idx], basis);
      idx++;
    }
  *e_theta = tt;
  *e_phi = ph;
}

// one thread per (timeslot, channel, source, station): array factor (arraybeam / array_element_beam,
// stationbeam.c:49-330) and element E-Jones (element_beam, :372-430)
__host__ __host__ __device__ __forceinline__ void beam_table_entry(const BeamArgs &a, size_t gid) {
  const int sta = (int)(gid % a.N);
  size_t q = gid / a.N;
  const int s = (int)(q % a.S);
  q /= a.S;
  const int cf = (int)(q % a.Nf);
  const int t = (int)(q / a.Nf);
  const double gmst = jd2gmst_deg(a.time_jd[t]);
  const double ra = a.src[s].ra, dec = a.src[s].dec;
  const double f = a.freqs[cf];
  double az, el;
  radec2azel(ra, dec, a.lon[sta], a.lat[sta], gmst, &az, &el);
  const double theta = M_PI_2 - el;
  if (a.af) {
    double gain = 0.0;
    if (el >= 0.0) {
      const double tpc = 2.0 * M_PI / 299792458.0;
      const double beam_f = a.wideband ? f : a.f0;
      double az0, el0;
      radec2azel(a.ra0, a.dec0, a.lon[sta], a.lat[sta], gmst, &az0, &el0);
      double sint, cost, sinph, cosph, sint0, cost0, sinph0, cosph0;
      sincos(theta, &sint, &cost);
      sincos(-az, &sinph, &cosph);
      sincos(M_PI_2 - el0, &sint0, &cost0);
      sincos(-az0, &sinph0, &cosph0);
      double rat1 = beam_f * sint0;
      const double rat2 = f * sint;
      double r1 = rat1 * cosph0 - rat2 * cosph, r2 = rat1 * sinph0 - rat2 * sinph;
      double r3 = beam_f * cost0 - f * cost;
      const int K = a.Nelem[sta];
      const double *px = a.ex + a.elem_off[sta], *py = a.ey + a.elem_off[sta];
      const double *pz = a.ez + a.elem_off[sta];
      const int skip = a.bf_type == 2 ? 16 : 0;  // STAT_TILE: tile centroids follow the 16 dipoles
      double csum = 0.0, ssum = 0.0;
      for (int j = 0; j < K; j++) {
        double sn, cs;
        sincos(-tpc * (r1 * px[j + skip] + r2 * py[j + skip] + r3 * pz[j + skip]), &sn, &cs);
        ssum += sn;
        csum += cs;
      }
      if (a.bf_type == 2) {
        double azb, elb;
        radec2azel(a.b_ra0, a.b_dec0, a.lon[sta], a.lat[sta], gmst, &azb, &elb);
        sincos(M_PI_2 - elb, &sint0, &cost0);
        sincos(-azb, &sinph0, &cosph0);
        rat1 = beam_f * sint0;
        r1 = rat1 * cosph0 - rat2 * cosph;
        r2 = rat1 * sinph0 - rat2 * sinph;
        r3 = beam_f * cost0 - f * cost;
        double cb = 0.0, sb = 0.0;
        for (int j = 0; j < 16; j++) {
          double sn, cs;
          sincos(-tpc * (r1 * px[j] + r2 * py[j] + r3 * pz[j]), &sn, &cs);
          sb += sn;
          cb += cs;
        }
        gain = sqrt(csum * csum + ssum * ssum) * sqrt(cb * cb + sb * sb) / (double)(K * 16);
      } else {
        gain = sqrt(csum * csum + ssum * ssum) / (double)K;
      }
    }
    a.af[gid] = gain;
  }
  if (a.E) {
    double2 e[4];
    e[0] = e[1] = e[2] = e[3] = make_double2(0.0, 0.0);
    if (el >= 0.0) {
      const int fi = a.wideband ? cf : 0;
      // E = [E_theta(az - pi/4) E_phi(az - pi/4); E_theta(az + pi/4) E_phi(az + pi/4)]
      element_eval(a, theta, az - M_PI_4, fi, &e[0], &e[1]);
      element_eval(a, theta, az - M_PI_4 + M_PI_2, fi, &e[2], &e[3]);
    }
    for (int c = 0; c < 4; c++) a.E[gid * 4 + c] = e[c];
  }
}

