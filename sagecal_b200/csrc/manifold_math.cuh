// Arithmetic of the projectback manifold average (calculate_manifold_average_projectback,
// manifold_average.c:641-867).  Host-callable so that oracle/manifold_math_check.cu runs exactly this
// code on the CPU against the compiled reference (test infrastructure); the product runs it on the
// device in k_manifold_projectback (kernels_manifold.cu).
//
// One solution block of a chunk is the 2n x 2 complex matrix J (n = N Npoly stations) of the
// reference's copy_1col_2col ordering.  Its rows 2i and 2i+1 are the 2x2 Jones matrix of station i,
// which is the 8 doubles pp[8i..8i+7] read as a row-major double2[4] (the layout of internal.cuh's
// 2x2 algebra).  So every product the reference forms with zgemm over 2n rows is a sum over stations
// of 2x2 products:
//   Gram  A^H B  = sum_i A_i^H B_i                 (mat_ahb per station)
//   block update J <- J W  is  J_i <- J_i W         (mat_ab per station)
#pragma once
#include <math.h>

#include "internal.cuh"

// ---- the unitary polar factor U V^H of a 2x2 complex Gram ---------------------------------------
// The reference takes it from LAPACK's zgesvd('A','A') followed by U*VT.  For a nonsingular Gram this
// is the unique unitary polar factor.  For a singular one it is not unique: the part that maps the
// null spaces onto each other is whatever zgesvd's reduction leaves there.  The reference's answers
// (tests/test_oracle_manifold_math.py) are:
//   zero Gram                          -> the identity;
//   rank 1, e.g. a zero row or column  -> u1 v1^H + u2 v2^H, where the phase of u2 v2^H depends on
//                                         the entries and no simple rule gives it.
// So the factor below is zgesvd's own sequence on a 2x2 matrix, in closed form: zgebd2's three
// Householder reflections (zlarfg) reduce G to a real upper bidiagonal [[d1, e1], [0, d2]] = Q^H G P;
// zungbr forms Q and P^H; zbdsqr splits off a negligible e1 or takes one dlasv2 rotation pair, makes
// the singular values positive by negating rows of V^H, and sorts them; the result is U V^H.  On a
// nonsingular Gram it agrees with any SVD to rounding; on a singular one it gives zgesvd's choice.
// G is row-major [00, 01, 10, 11].  Inputs far outside [1e-139, 1e139], which zgesvd rescales first,
// are not rescaled here.

// Fortran SIGN(a, b) as gfortran evaluates it: |a| with the sign bit of b
__host__ __device__ __forceinline__ double mf_sign(double a, double b) { return copysign(fabs(a), b); }

// zlarfg on (alpha, x) with x of length 0 or 1: beta (real), tau and the scaled x.  With no x to
// annihilate and a real alpha the reflector is the identity (tau = 0, beta = alpha).
__host__ __device__ __forceinline__ void mf_zlarfg(double2 alpha, double2 *x, double2 &tau,
                                                   double &beta) {
  const double xnorm = x ? hypot(x->x, x->y) : 0.0;
  if (xnorm == 0.0 && alpha.y == 0.0) {
    tau = make_double2(0.0, 0.0);
    beta = alpha.x;
    return;
  }
  beta = -mf_sign(sqrt(alpha.x * alpha.x + alpha.y * alpha.y + xnorm * xnorm), alpha.x);
  tau = make_double2((beta - alpha.x) / beta, -alpha.y / beta);
  if (x) {  // x <- x / (alpha - beta)
    const double2 den = make_double2(alpha.x - beta, alpha.y);
    const double inv = 1.0 / (den.x * den.x + den.y * den.y);
    const double2 s = make_double2(den.x * inv, -den.y * inv);
    *x = cmul(s, *x);
  }
}

// dlasv2: SVD of the real upper triangular [[f, g], [0, h]]
__host__ __device__ __forceinline__ void mf_dlasv2(double f, double g, double h, double &ssmin,
                                                   double &ssmax, double &snr, double &csr,
                                                   double &snl, double &csl) {
  const double eps = 1.1102230246251565e-16;  // dlamch('EPS')
  double ft = f, fa = fabs(f), ht = h, ha = fabs(h);
  int pmax = 1;
  const bool swap = ha > fa;
  if (swap) {
    pmax = 3;
    double t = ft; ft = ht; ht = t;
    t = fa; fa = ha; ha = t;
  }
  const double gt = g, ga = fabs(g);
  double clt, crt, slt, srt;
  if (ga == 0.0) {
    ssmin = ha;
    ssmax = fa;
    clt = 1.0; crt = 1.0; slt = 0.0; srt = 0.0;
  } else {
    bool gasmal = true;
    if (ga > fa) {
      pmax = 2;
      if (fa / ga < eps) {
        gasmal = false;
        ssmax = ga;
        ssmin = ha > 1.0 ? fa / (ga / ha) : (fa / ga) * ha;
        clt = 1.0;
        slt = ht / gt;
        srt = 1.0;
        crt = ft / gt;
      }
    }
    if (gasmal) {
      const double d = fa - ha;
      double l = d == fa ? 1.0 : d / fa;
      const double m = gt / ft;
      double t = 2.0 - l;
      const double mm = m * m, tt = t * t;
      const double s = sqrt(tt + mm);
      const double r = l == 0.0 ? fabs(m) : sqrt(l * l + mm);
      const double a = 0.5 * (s + r);
      ssmin = ha / a;
      ssmax = fa * a;
      if (mm == 0.0) {
        t = l == 0.0 ? mf_sign(2.0, ft) * mf_sign(1.0, gt) : gt / mf_sign(d, ft) + m / t;
      } else {
        t = (m / (s + t) + m / (r + l)) * (1.0 + a);
      }
      l = sqrt(t * t + 4.0);
      crt = 2.0 / l;
      srt = t / l;
      clt = (crt + srt * m) / a;
      slt = (ht / ft) * srt / a;
    }
  }
  if (swap) {
    csl = srt; snl = crt; csr = slt; snr = clt;
  } else {
    csl = clt; snl = slt; csr = crt; snr = srt;
  }
  double tsign;
  if (pmax == 1) tsign = mf_sign(1.0, csr) * mf_sign(1.0, csl) * mf_sign(1.0, f);
  else if (pmax == 2) tsign = mf_sign(1.0, snr) * mf_sign(1.0, csl) * mf_sign(1.0, g);
  else tsign = mf_sign(1.0, snr) * mf_sign(1.0, snl) * mf_sign(1.0, h);
  ssmax = mf_sign(ssmax, tsign);
  ssmin = mf_sign(ssmin, tsign * mf_sign(1.0, f) * mf_sign(1.0, h));
}

// W = U V^H of the SVD G = U S V^H as zgesvd('A','A') returns it (see above); G, W row-major
__host__ __device__ __forceinline__ void manifold_polar(const double2 *G, double2 *W) {
  const double2 one = make_double2(1.0, 0.0), zero = make_double2(0.0, 0.0);
  // zgebd2, column 1: H1 = I - tau1 v v^H, v = (1, v2), annihilates G[1][0]
  double2 v2 = G[2], tau1;
  double d1;
  mf_zlarfg(G[0], &v2, tau1, d1);
  // H1^H applied to column 2
  double2 a12 = G[1], a22 = G[3];
  if (tau1.x != 0.0 || tau1.y != 0.0) {
    const double2 w = cadd(a12, cmulcl(v2, a22));
    const double2 ct = make_double2(tau1.x, -tau1.y);
    a12 = csub(a12, cmul(ct, w));
    a22 = csub(a22, cmul(ct, cmul(v2, w)));
  }
  // row 1: G1 makes conj(a12) real; applied from the right to a22
  double2 taup;
  double e1;
  mf_zlarfg(make_double2(a12.x, -a12.y), nullptr, taup, e1);
  if (taup.x != 0.0 || taup.y != 0.0) a22 = cmul(a22, make_double2(1.0 - taup.x, -taup.y));
  // column 2: H2 makes a22 real
  double2 tau2;
  double d2;
  mf_zlarfg(a22, nullptr, tau2, d2);
  // zungbr('Q'): U = H1 diag(1, 1 - tau2); zungbr('P'): VT = diag(1, 1 - conj(taup))
  double2 U[4], VT[4];
  {
    const double2 q22 = make_double2(1.0 - tau2.x, -tau2.y);
    U[0] = make_double2(1.0 - tau1.x, -tau1.y);
    U[2] = make_double2(-(tau1.x * v2.x - tau1.y * v2.y), -(tau1.x * v2.y + tau1.y * v2.x));
    if (tau1.x != 0.0 || tau1.y != 0.0) {
      const double2 w = cmulcl(v2, q22);
      U[1] = csub(zero, cmul(tau1, w));
      U[3] = csub(q22, cmul(tau1, cmul(v2, w)));
    } else {
      U[1] = zero;
      U[3] = q22;
    }
    VT[0] = one;
    VT[1] = zero;
    VT[2] = zero;
    VT[3] = make_double2(1.0 - taup.x, taup.y);
  }
  // zbdsqr on [[d1, e1], [0, d2]]
  const double eps = 1.1102230246251565e-16, unfl = 2.2250738585072014e-308;
  const double tolmul = fmax(10.0, fmin(100.0, pow(eps, -0.125)));
  const double tol = tolmul * eps;
  double sminoa = fabs(d1);
  if (sminoa != 0.0) {
    const double mu = fabs(d2) * (sminoa / (sminoa + fabs(e1)));
    sminoa = fmin(sminoa, mu);
  }
  sminoa = sminoa / sqrt(2.0);
  const double thresh = fmax(tol * sminoa, 6.0 * 2.0 * 2.0 * unfl);
  if (!(fabs(e1) <= thresh)) {
    double sigmn, sigmx, sinr, cosr, sinl, cosl;
    mf_dlasv2(d1, e1, d2, sigmn, sigmx, sinr, cosr, sinl, cosl);
    d1 = sigmx;
    d2 = sigmn;
    for (int j = 0; j < 2; j++) {  // zdrot on the rows of VT
      const double2 x = VT[j], y = VT[2 + j];
      VT[j] = make_double2(cosr * x.x + sinr * y.x, cosr * x.y + sinr * y.y);
      VT[2 + j] = make_double2(cosr * y.x - sinr * x.x, cosr * y.y - sinr * x.y);
    }
    for (int i = 0; i < 2; i++) {  // zdrot on the columns of U
      const double2 x = U[2 * i], y = U[2 * i + 1];
      U[2 * i] = make_double2(cosl * x.x + sinl * y.x, cosl * x.y + sinl * y.y);
      U[2 * i + 1] = make_double2(cosl * y.x - sinl * x.x, cosl * y.y - sinl * x.y);
    }
  }
  if (d1 < 0.0) { d1 = -d1; VT[0] = make_double2(-VT[0].x, -VT[0].y); VT[1] = make_double2(-VT[1].x, -VT[1].y); }
  if (d2 < 0.0) { d2 = -d2; VT[2] = make_double2(-VT[2].x, -VT[2].y); VT[3] = make_double2(-VT[3].x, -VT[3].y); }
  if (!(d2 <= d1)) {  // sort decreasing: swap rows of VT and columns of U
    double2 t = VT[0]; VT[0] = VT[2]; VT[2] = t;
    t = VT[1]; VT[1] = VT[3]; VT[3] = t;
    t = U[0]; U[0] = U[1]; U[1] = t;
    t = U[2]; U[2] = U[3]; U[3] = t;
  }
  mat_ab(U, VT, W);
}

// ---- the average in the space of 2x2 rotations -------------------------------------------------
// Per chunk, every block stays its input block Y_f times a 2x2 unitary R_f, so each Gram the
// reference forms over 2n rows is a 2x2 product of the R's with the pairwise Grams C_fg = Y_f^H Y_g
// of the input blocks (kernels_manifold.cu).  C holds the f <= g half, pair p = (f, g) in row order.

// G += A_i^H B_i for one station (A, B: 8 doubles each, read as row-major double2[4])
__host__ __device__ __forceinline__ void manifold_gram_acc(const double2 *A, const double2 *B,
                                                           double2 *G) {
  double2 g[4];
  mat_ahb(A, B, g);
  for (int e = 0; e < 4; e++) G[e] = cadd(G[e], g[e]);
}

// pair index p -> (f, g), f <= g
__host__ __device__ __forceinline__ void manifold_pair(int p, int Nf, int &f, int &g) {
  f = 0;
  int row = Nf;
  while (p >= row) { p -= row; f++; row--; }
  g = f + p;
}

// C_fg for any f, g from the stored half (C_gf = C_fg^H)
__host__ __device__ __forceinline__ void manifold_cfg(const double2 *C, int Nf, int f, int g,
                                                      double2 *out) {
  if (f <= g) {
    const int p = f * Nf - f * (f - 1) / 2 + (g - f);
    for (int e = 0; e < 4; e++) out[e] = C[4 * p + e];
  } else {
    const int p = g * Nf - g * (g - 1) / 2 + (f - g);
    const double2 *c = C + 4 * p;
    out[0] = make_double2(c[0].x, -c[0].y);
    out[1] = make_double2(c[2].x, -c[2].y);
    out[2] = make_double2(c[1].x, -c[1].y);
    out[3] = make_double2(c[3].x, -c[3].y);
  }
}

// step 1, block f: project onto block cr (project_procrustes_block): R_f = polar(C_f,cr), R_cr = I
__host__ __device__ __forceinline__ void manifold_start(const double2 *C, int Nf, int f, int cr,
                                                        double2 *Rf) {
  if (f == cr) {
    Rf[0] = Rf[3] = make_double2(1.0, 0.0);
    Rf[1] = Rf[2] = make_double2(0.0, 0.0);
    return;
  }
  double2 G[4];
  manifold_cfg(C, Nf, f, cr, G);
  manifold_polar(G, Rf);
}

// one round of step 2 for block f, from the rotations R of the previous round:
// J3 = (sum_g Y_g R_g) / Nf, Gram (Y_f R_f)^H J3 = R_f^H (sum_g C_fg R_g) / Nf, Rn_f = R_f polar(Gram)
__host__ __device__ __forceinline__ void manifold_round(const double2 *C, int Nf, int f,
                                                        const double2 *R, double2 *Rnf) {
  const double a = 1.0 / (double)Nf;
  double2 S[4] = {make_double2(0.0, 0.0), make_double2(0.0, 0.0), make_double2(0.0, 0.0),
                  make_double2(0.0, 0.0)};
  for (int g = 0; g < Nf; g++) {
    double2 c[4], t[4];
    manifold_cfg(C, Nf, f, g, c);
    mat_ab(c, R + 4 * g, t);
    for (int e = 0; e < 4; e++) S[e] = cadd(S[e], t[e]);
  }
  for (int e = 0; e < 4; e++) S[e] = make_double2(S[e].x * a, S[e].y * a);
  double2 G[4], W[4];
  mat_ahb(R + 4 * f, S, G);
  manifold_polar(G, W);
  mat_ab(R + 4 * f, W, Rnf);
}

// step 4 for block f: P_f = polar(J3^H Y_f) = polar((sum_g R_g^H C_gf) / Nf)
__host__ __device__ __forceinline__ void manifold_final(const double2 *C, int Nf, int f,
                                                        const double2 *R, double2 *Pf) {
  const double a = 1.0 / (double)Nf;
  double2 S[4] = {make_double2(0.0, 0.0), make_double2(0.0, 0.0), make_double2(0.0, 0.0),
                  make_double2(0.0, 0.0)};
  for (int g = 0; g < Nf; g++) {
    double2 c[4], t[4];
    manifold_cfg(C, Nf, g, f, c);
    mat_ahb(R + 4 * g, c, t);
    for (int e = 0; e < 4; e++) S[e] = cadd(S[e], t[e]);
  }
  for (int e = 0; e < 4; e++) S[e] = make_double2(S[e].x * a, S[e].y * a);
  manifold_polar(S, Pf);
}

// steps 3 and 4 for station i: J3_i = (sum_g Y_g,i R_g) / Nf, Y_f,i <- J3_i P_f.  Y points at the
// station's 2x2 in block 0; blocks are fs double2 apart.
__host__ __device__ __forceinline__ void manifold_output(double2 *Y, size_t fs, int Nf,
                                                         const double2 *R, const double2 *P) {
  const double a = 1.0 / (double)Nf;
  double2 J3[4] = {make_double2(0.0, 0.0), make_double2(0.0, 0.0), make_double2(0.0, 0.0),
                   make_double2(0.0, 0.0)};
  for (int g = 0; g < Nf; g++) {
    double2 y[4], t[4];
    for (int e = 0; e < 4; e++) y[e] = Y[fs * g + e];
    mat_ab(y, R + 4 * g, t);
    for (int e = 0; e < 4; e++) J3[e] = cadd(J3[e], t[e]);
  }
  for (int e = 0; e < 4; e++) J3[e] = make_double2(J3[e].x * a, J3[e].y * a);
  for (int f = 0; f < Nf; f++) {
    double2 o[4];
    mat_ab(J3, P + 4 * f, o);
    for (int e = 0; e < 4; e++) Y[fs * f + e] = o[e];
  }
}
