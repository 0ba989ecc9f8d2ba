"""helpers shared by the tests: problems in API layout bound to ctypes structures"""
import numpy as np

from sagecal_b200 import synth
from sagecal_b200.dirac_api import SkyModel, make_barr


class Bound:
    """a synthetic problem plus the ctypes objects both libraries take"""

    def __init__(self, pr: synth.Problem):
        self.pr = pr
        self.barr = make_barr(pr.sta1, pr.sta2, pr.flag)
        self.sky = SkyModel(pr.clusters, pr.N)
        self.n = 8 * pr.Nbase1
        self.m = 8 * pr.N * pr.Mt

    def fresh_barr(self):
        return make_barr(self.pr.sta1, self.pr.sta2, self.pr.flag)


def small_problem(N=8, M=2, tilesz=10, seed=11, **kw):
    return Bound(synth.make_problem(N=N, M=M, tilesz=tilesz, seed=seed, **kw))


def perturbed_jones(pr, seed=3, amp=0.1):
    rng = np.random.default_rng(seed)
    return pr.pp0 + amp * rng.normal(0, 1, pr.pp0.shape)


def _api_layout(z):
    """[nrow, 2, 2] complex -> float64 [8 * nrow] (XX re, im, XY, YX, YY per row)"""
    o = np.empty((z.shape[0], 4, 2))
    o[:, :, 0] = z.reshape(-1, 4).real
    o[:, :, 1] = z.reshape(-1, 4).imag
    return o.reshape(-1)


def line_model_ref(pr, xk, pk):
    """plain numpy restatement of the LBFGS line model: with A = Jp + a Dp and B = Jq + a Dq of
    every cluster (Jones xk, direction pk, hybrid chunk of the row), sum_k A C B^H = V0 + a V1 + a^2 V2.
    returns (V0, V1, V2) in API layout, zero on flagged and uv-cut rows (they carry no model)"""
    nrow = pr.Nbase1
    c = pr.coh.reshape(nrow, pr.M, 2, 2)
    rows = np.arange(nrow)
    V = [np.zeros((nrow, 2, 2), dtype=np.complex128) for _ in range(3)]

    def jones(vec, off, nch):
        J = vec[off:off + nch * 8 * pr.N].reshape(nch, pr.N, 4, 2)
        return (J[..., 0] + 1j * J[..., 1]).reshape(nch, pr.N, 2, 2)

    off = 0
    for k in range(pr.M):
        nch = pr.nchunk[k]
        px = synth.chunk_index(rows, nrow, nch)
        J, D = jones(xk, off, nch), jones(pk, off, nch)
        Jp, Jq, Dp, Dq = J[px, pr.sta1], J[px, pr.sta2], D[px, pr.sta1], D[px, pr.sta2]
        H = lambda X: np.conj(np.swapaxes(X, 1, 2))
        JC, DC = Jp @ c[:, k], Dp @ c[:, k]
        V[0] += JC @ H(Jq)
        V[1] += DC @ H(Jq) + JC @ H(Dq)
        V[2] += DC @ H(Dq)
        off += nch * 8 * pr.N
    for v in V:
        v[pr.flag != 0] = 0.0
    return tuple(_api_layout(v) for v in V)


def _jones(vec, N):
    """8N parameter vector (station s: J[a][m] at 8s + 2(2a+m)) -> [N, 2, 2] complex"""
    J = np.asarray(vec, dtype=np.float64).reshape(N, 4, 2)
    return (J[..., 0] + 1j * J[..., 1]).reshape(N, 2, 2)


def _chunk_rows(pr, k, t0, nt, y):
    """hidden data d, coherencies C of cluster k, unflagged mask and stations of the chunk's rows"""
    r0, r1 = t0 * pr.Nbase, (t0 + nt) * pr.Nbase
    dd = np.asarray(y, dtype=np.float64)[8 * r0:8 * r1].reshape(-1, 4, 2)
    d = (dd[..., 0] + 1j * dd[..., 1]).reshape(-1, 2, 2)
    C = pr.coh.reshape(pr.Nbase1, pr.M, 2, 2)[r0:r1, k]
    return d, C, pr.flag[r0:r1] == 0, pr.sta1[r0:r1], pr.sta2[r0:r1]


def _station_sums(pr, nt, vp, vq):
    """per-row 2x2 terms of the p and q ends -> per-station sums [N, 2, 2]: summed over the timeslots
    of each baseline first, then over the baselines of each station"""
    Nb = pr.Nbase
    S = np.zeros((pr.N, 2, 2), dtype=vp.dtype)
    np.add.at(S, pr.sta1[:Nb], vp.reshape(nt, Nb, 2, 2).sum(axis=0))
    np.add.at(S, pr.sta2[:Nb], vq.reshape(nt, Nb, 2, 2).sum(axis=0))
    return S


def rtr_eval_ref(pr, k, t0, nt, x, eta=None, wt=None, y=None):
    """plain float64 per-row restatement of the RTR evaluator (rtr_algo.h, evaluator concept) on
    cluster k, tiles [t0, t0 + nt), hidden data y (default: the problem's data), row weights wt
    (one per row of the chunk, default 1), flagged rows skipped:
      cost   sum w |d - Gp C Gq^H|^2
      vec    station sums of w res Gq C^H (at p) and w res^H Gp C (at q); with eta their derivative
             along eta: w (res Eq - res1 Gq) C^H and w (res^H Ep - res1^H Gp) C, res1 = Gp C Eq^H + Ep C Gq^H
      counts unflagged rows per station
    Each value comes with a magnitude companion, the same sums over absolute values with res taken as
    |d| + |Gp||C||Gq|^T (the tensor form of the kernels subtracts those two): cost_scale
    sum w (|d|^2 + (|Gp||C||Gq|^T)^2), vec_scale [8N].  Vectors in the parameter layout."""
    N = pr.N
    d, C, ok, p, q = _chunk_rows(pr, k, t0, nt, pr.x if y is None else y)
    w = ok * (1.0 if wt is None else np.asarray(wt, dtype=np.float64))
    H = lambda A: np.conj(np.swapaxes(A, -1, -2))
    T = lambda A: np.swapaxes(A, -1, -2)
    A = np.abs
    G = _jones(x, N)
    Gp, Gq = G[p], G[q]
    V = Gp @ C @ H(Gq)
    Va = A(Gp) @ A(C) @ T(A(Gq))
    res = d - V
    ra = A(d) + Va
    wr = w[:, None, None]
    cost = float(np.sum(w * np.sum(np.abs(res) ** 2, axis=(1, 2))))
    cost_scale = float(np.sum(w * np.sum(np.abs(d) ** 2 + Va ** 2, axis=(1, 2))))
    if eta is None:
        vp = wr * (res @ Gq @ H(C))
        vq = wr * (H(res) @ Gp @ C)
        sp = wr * (ra @ A(Gq) @ T(A(C)))
        sq = wr * (T(ra) @ A(Gp) @ A(C))
    else:
        E = _jones(eta, N)
        Ep, Eq = E[p], E[q]
        res1 = Gp @ C @ H(Eq) + Ep @ C @ H(Gq)
        r1a = A(Gp) @ A(C) @ T(A(Eq)) + A(Ep) @ A(C) @ T(A(Gq))
        vp = wr * ((res @ Eq - res1 @ Gq) @ H(C))
        vq = wr * ((H(res) @ Ep - H(res1) @ Gp) @ C)
        sp = wr * ((ra @ A(Eq) + r1a @ A(Gq)) @ T(A(C)))
        sq = wr * ((T(ra) @ A(Ep) + T(r1a) @ A(Gp)) @ A(C))
    S = _station_sums(pr, nt, vp, vq)
    Sa = _station_sums(pr, nt, sp, sq)
    vec = np.stack([S.real, S.imag], axis=-1).reshape(-1)
    vec_scale = np.stack([Sa, Sa], axis=-1).reshape(-1)
    counts = (np.bincount(p, weights=ok.astype(float), minlength=N)
              + np.bincount(q, weights=ok.astype(float), minlength=N))
    return dict(cost=cost, cost_scale=cost_scale, vec=vec, vec_scale=vec_scale, counts=counts)


def rtr_weights_ref(pr, k, t0, nt, x, nu, y=None):
    """Student's-t row weights (nu+2)/(nu + max_c |res_c|^2) at x on the chunk's unflagged rows (0 on
    flagged ones) and sum(log w - w) over the unflagged rows divided by ALL rows of the chunk.
    returns (slw, w, slw_scale), slw_scale the same mean over |log w| + w"""
    d, C, ok, p, q = _chunk_rows(pr, k, t0, nt, pr.x if y is None else y)
    G = _jones(x, pr.N)
    res = d - G[p] @ C @ np.conj(np.swapaxes(G[q], -1, -2))
    e2 = np.max((np.abs(res) ** 2).reshape(-1, 4), axis=1)
    w = np.where(ok, (nu + 2.0) / (nu + e2), 0.0)
    lw = np.where(ok, np.log(np.where(ok, w, 1.0)), 0.0)
    n = len(ok)
    return float(np.sum(lw - w)) / n, w, float(np.sum(np.abs(lw) + w)) / n


def _digamma(x):
    """the reference's digamma series (updatenu.c:36-49)"""
    r = 0.0
    while x < 7.0:
        r -= 1.0 / x
        x += 1.0
    x -= 0.5
    xx = 1.0 / x
    xx2 = xx * xx
    xx4 = xx2 * xx2
    return (r + np.log(x) + (1. / 24.) * xx2 - (7.0 / 960.0) * xx4 + (31.0 / 8064.0) * xx4 * xx2
            - (127.0 / 30720.0) * xx4 * xx4)


def irls_ref(e, wt_old, nu0, nulow=2.0, nuhigh=30.0):
    """the update between two IRLS rounds of the robust LM, restated (robustlm.c:2533-2566,
    updatenu.c:86-104,137-262) for the chunk's residual e and its sqrt-weights wt_old (flat, 8 values
    per row): w = (nu0+1)/(nu0+e^2), q = |w - log w|, lambda = sum |wt_old|, sumq = sum q / ndata,
    nu = the point of the 30-point grid on [nulow, nuhigh) with the smallest
    |psi((nu+1)/2) - ln((nu+1)/2) - psi(nu/2) + ln(nu/2) - sumq + 1| (first one on a tie), new weights
    sqrt(w) lambda / ndata.  Sums in long double.  returns dict(w, lam, sumq, nu, margin: runner-up
    |value| minus the best one)"""
    e = np.asarray(e, dtype=np.float64)
    n = e.size
    w = (nu0 + 1.0) / (nu0 + e * e)
    lam = lsum(np.abs(wt_old))
    sumq = lsum(np.abs(w - np.log(w))) / n
    deltanu = (nuhigh - nulow) / 30.0
    nus = [nulow + float(ci) * deltanu for ci in range(30)]
    qs = np.array([abs(_digamma(t * 0.5 + 0.5) - np.log((t + 1.0) * 0.5) - _digamma(t * 0.5)
                       + np.log(t * 0.5) - sumq + 1.0) for t in nus])
    best = int(np.argmin(qs))
    return dict(w=np.sqrt(w) * (lam / n), lam=lam, sumq=sumq, nu=nus[best],
                margin=float(np.sort(qs)[1] - qs[best]))


def os_subset_ref(J, e, wt, ntiles, Nbase, l):
    """the system of ordered subset l as the reference's oslevmar / osrlevmar form it
    (clmfit.c:1313-1413, robustlm.c:2835-2935), built literally from the chunk's dense Jacobian J
    [8 ntiles Nbase, 8N], unweighted residual e and sqrt-weights wt (None: 1): the rows of the subset's
    Ntper tiles, cut or zero padded to Nos rows, paired with e[kl:kl+Nos] and wt[kl:kl+Nos].
    returns (JTJ, JTe, (kl, Nos, tl, tileI))"""
    n = 8 * ntiles * Nbase
    ns = min(10, ntiles)
    Nper = (n + ns - 1) // ns
    Ntper = (ntiles + ns - 1) // ns
    kl, tl = l * Nper, l * Ntper
    if tl + Ntper < ntiles:
        Nos, tileI = Nper, Ntper
    else:
        Nos, tileI = n - kl, ntiles - tl
    m8 = J.shape[1]
    Jos = np.zeros((max(Nos, 0), m8))
    if tileI > 0 and Nos > 0:
        Jl = J[8 * Nbase * tl:8 * Nbase * (tl + tileI)]
        m = min(Nos, len(Jl))
        Jos[:m] = Jl[:m]
    w = np.ones(n) if wt is None else np.asarray(wt, dtype=np.float64)
    ww = w[kl:kl + max(Nos, 0)]
    ew = (w * e)[kl:kl + max(Nos, 0)]
    Jw = Jos * ww[:, None]
    return Jw.T @ Jw, Jw.T @ ew, (kl, Nos, tl, tileI)


def big_cluster_sky(seed=7, sizes=(1, 95, 96, 97, 192, 200, 0)):
    """clusters of the given sizes (0: empty), half the sources Gaussian, spread over a few
    degrees, fluxes with a spectral index"""
    rng = np.random.default_rng(seed)
    clusters = []
    for k, K in enumerate(sizes):
        l0, m0 = np.deg2rad(rng.uniform(-3, 3, 2))
        ll = l0 + np.deg2rad(0.5) * rng.uniform(-1, 1, K)
        mm = m0 + np.deg2rad(0.5) * rng.uniform(-1, 1, K)
        sI = rng.lognormal(-1.0, 1.0, K)
        gauss = np.zeros((K, 8))
        gauss[:, 0] = np.deg2rad(rng.uniform(0.5, 3.0, K) / 60.0)
        gauss[:, 1] = np.deg2rad(rng.uniform(0.5, 3.0, K) / 60.0)
        gauss[:, 2] = rng.uniform(0, np.pi, K)
        gauss[:, 3] = 1.0
        gauss[:, 5] = 1.0
        clusters.append(dict(
            ll=ll, mm=mm, nn=np.sqrt(1.0 - ll * ll - mm * mm) - 1.0, sI=sI,
            sQ=0.1 * sI * rng.uniform(-1, 1, K), sU=0.1 * sI * rng.uniform(-1, 1, K),
            sV=0.02 * sI * rng.uniform(-1, 1, K), stype=(np.arange(K) % 2).astype(np.uint8),
            gauss=gauss, spec_idx=np.where(np.arange(K) % 3 == 0, -0.7, 0.0),
            spec_idx1=np.full(K, 0.05), spec_idx2=np.full(K, -0.01), f0=np.full(K, 140e6),
            nchunk=1, id=k))
    return clusters


def split_cluster(cl, parts):
    """the sources of one cluster as consecutive clusters of the given sizes"""
    out, s0 = [], 0
    for n in parts:
        sub = {}
        for key, v in cl.items():
            sub[key] = v[s0:s0 + n] if isinstance(v, np.ndarray) else v
        out.append(sub)
        s0 += n
    return out


#: element-wise error budget of the sky prediction: |got - want| <= SKY_C eps sum_s w_s per row,
#: correlation and channel, w_s from sky_predict_ref
SKY_C = 16.0


def sky_predict_ref(u, v, w, clusters, freq, fdelta2, spectral):
    """per-cluster coherencies of point, Gaussian, disk and ring sources at one frequency, restated in
    long double from predict.c:399-472 (spectral=False: the fluxes sI..sV as they are) and
    residual.c:1124-1226 (spectral=True: the three-term log spectral index from sI0..sV0 and f0 where
    spec_idx != 0).  M_PI is the double constant, as in both codes.  returns (C [nrow, M, 4] complex,
    budget [nrow, M]): budget is the sum over the cluster's sources of
      w_s = |flux_s| (|shape_s| (1 + phi_s) + 1 + sigma_s + lambda_s),
    |flux_s| = |I| + |Q| + |U| + |V|, phi_s = 2 pi f (|u l| + |v m| + |w n|) the size of the phase
    before cancellation (G is rounded before it is scaled by f, so a phase of 1e5 rad carries an error
    of about 1e5 eps), sigma_s the sensitivity of the shape factor to a relative error of its argument
    (Gaussian x e^-x with x = 2 pi^2 (ut^2 + vt^2) taken over absolute values, disk / ring the Bessel
    argument, |j0'|, |j1'| <= 1) and lambda_s = |log |s0|| + |tempfr| that of the spectral flux."""
    from scipy import special
    L = np.longdouble
    pi = L(np.pi)
    f = L(freq)
    u = np.asarray(u, dtype=L)[:, None]
    v = np.asarray(v, dtype=L)[:, None]
    w = np.asarray(w, dtype=L)[:, None]
    nrow = u.shape[0]
    C = np.zeros((nrow, len(clusters), 4), dtype=np.clongdouble)
    budget = np.zeros((nrow, len(clusters)))
    for k, cl in enumerate(clusters):
        K = len(cl["ll"])
        if K == 0:
            continue
        ll, mm, nn = (np.asarray(cl[n], dtype=L)[None, :] for n in ("ll", "mm", "nn"))
        G = 2 * pi * (u * ll + v * mm + w * nn)
        phi = 2 * pi * f * (np.abs(u * ll) + np.abs(v * mm) + np.abs(w * nn))
        ph = np.exp(1j * (G * f))
        with np.errstate(invalid="ignore", divide="ignore"):
            sm = G * L(fdelta2)
            fac = np.where(G != 0, np.abs(np.sin(sm) / np.where(G != 0, sm, 1)), L(1))
        ph = ph * fac
        st = np.asarray(cl.get("stype", np.zeros(K)), dtype=int)
        shape = np.ones((nrow, K), dtype=L)
        sigma = np.zeros((nrow, K), dtype=L)
        uf, vf, wf = u * f, v * f, w * f
        gauss, disk = cl.get("gauss"), cl.get("disk") or {}
        for s in range(K):
            if st[s] == 0:
                continue
            if st[s] == 1:
                eX, eY, eP, cxi, sxi, cphi, sphi, proj = (L(x) for x in gauss[s])
            else:
                eX, cxi, sxi, cphi, sphi, proj = (L(x) for x in disk[s])
                proj = L(1)   # disks and rings always project (predict.c:67-68,82-83)
            if proj != 0:
                terms_u = (uf * cxi, -vf * cphi * sxi, wf * sphi * sxi)
                terms_v = (uf * sxi, vf * cphi * cxi, -wf * sphi * cxi)
            else:
                terms_u, terms_v = (uf,), (vf,)
            up, vp = sum(terms_u)[:, 0], sum(terms_v)[:, 0]
            uvabs = (sum(np.abs(t) for t in terms_u) + sum(np.abs(t) for t in terms_v))[:, 0]
            if st[s] == 1:
                sP, cP = np.sin(L(float(eP))), np.cos(L(float(eP)))
                ut = eX * (cP * up - sP * vp)
                vt = eY * (sP * up + cP * vp)
                x = 2 * pi * pi * (ut * ut + vt * vt)
                shape[:, s] = np.exp(-x)
                sigma[:, s] = 2 * pi * pi * (eX * eX + eY * eY) * uvabs * uvabs * np.exp(-x)
            else:
                b = np.sqrt(up * up + vp * vp) * eX * 2 * pi
                bd = b.astype(np.float64)   # scipy's Bessel functions on the long-double argument
                shape[:, s] = (special.j1 if st[s] == 2 else special.j0)(bd)
                sigma[:, s] = 2 * pi * eX * uvabs + 1
        ph = ph * shape
        flux = [np.asarray(cl[n], dtype=L) for n in ("sI", "sQ", "sU", "sV")]
        lam = np.zeros(K, dtype=L)
        if spectral:
            si = [np.asarray(cl.get(n, np.zeros(K)), dtype=L) for n in ("spec_idx", "spec_idx1",
                                                                         "spec_idx2")]
            f0 = np.asarray(cl.get("f0", np.full(K, 150e6)), dtype=L)
            fr = np.log(f / f0)
            tf = si[0] * fr + si[1] * fr * fr + si[2] * fr * fr * fr
            tfa = np.abs(si[0] * fr) + np.abs(si[1] * fr * fr) + np.abs(si[2] * fr * fr * fr)
            on = si[0] != 0
            for j, n in enumerate(("sI0", "sQ0", "sU0", "sV0")):
                s0 = np.asarray(cl.get(n, cl[n[:2]]), dtype=L)
                with np.errstate(divide="ignore"):
                    sf = np.where(s0 > 0, np.exp(np.log(np.abs(s0)) + tf),
                                  np.where(s0 == 0, L(0), -np.exp(np.log(np.abs(s0)) + tf)))
                    lj = np.where(s0 != 0, np.abs(np.log(np.abs(s0))), L(0))
                flux[j] = np.where(on, sf, flux[j])
                lam = np.maximum(lam, np.where(on, lj + tfa, L(0)))
        I, Q, U, V = flux
        C[:, k, 0] = ph @ (I + Q)
        C[:, k, 1] = ph @ (U + 1j * V)
        C[:, k, 2] = ph @ (U - 1j * V)
        C[:, k, 3] = ph @ (I - Q)
        fa = (np.abs(I) + np.abs(Q) + np.abs(U) + np.abs(V))[None, :]
        ws = fa * (np.abs(shape) * (1 + phi) + 1 + sigma + lam[None, :])
        budget[:, k] = np.sum(ws, axis=1).astype(np.float64)
    return C, budget


def sky_edge_case(name, seed=5):
    """(u, v, w, clusters, freqs, fdelta) of one edge of the sky prediction, on the rows of
    small_problem(N=6, tilesz=4) (60 rows), every source type of the restatement present:
      long      |uv| f up to 1e5 lambda, sources 10-30 deg from the centre: |phase| 1e5 .. 1e6 rad
      centre    one source exactly at the phase centre, rows 0-3 with u = v = w = 0 (the G == 0 branch)
      widefd    a 40 MHz smearing width: the sinc far from 1 (and through its zeros)
      tinyfd    a 1 Hz smearing width
      gauss     Gaussians of extent 0, 1e-12 rad and of 1 rad (vanishing to underflow), both projections
      bessel    disks and rings sized so that rows sit on zeros of j1 and j0
      spectral  negative and zero Stokes fluxes, channels at f0 / 2, f0, 2 f0"""
    b = small_problem(N=6, M=2, tilesz=4, seed=seed)
    pr = b.pr
    u, v, w = pr.u.copy(), pr.v.copy(), pr.w.copy()
    rng = np.random.default_rng(seed + 1)
    freqs = np.array([140e6, 150e6, 163e6])
    fdelta = 195.3e3
    K = 8

    def cluster(ll, mm, sI, stype=None, **kw):
        ll, mm = np.asarray(ll, dtype=np.float64), np.asarray(mm, dtype=np.float64)
        n = len(ll)
        sI = np.asarray(sI, dtype=np.float64)
        cl = dict(ll=ll, mm=mm, nn=np.sqrt(1.0 - ll * ll - mm * mm) - 1.0, sI=sI,
                  sQ=0.3 * sI * rng.uniform(-1, 1, n), sU=0.2 * sI * rng.uniform(-1, 1, n),
                  sV=0.05 * sI * rng.uniform(-1, 1, n),
                  stype=np.zeros(n, dtype=np.uint8) if stype is None else np.asarray(stype, np.uint8))
        cl.update(kw)
        return cl

    def around(lo_deg, hi_deg, n):
        r = np.deg2rad(rng.uniform(lo_deg, hi_deg, n))
        a = rng.uniform(0, 2 * np.pi, n)
        return np.sin(r) * np.cos(a), np.sin(r) * np.sin(a)

    def gauss_tab(eX, eY, proj):
        g = np.zeros((len(eX), 8))
        xi, ph = rng.uniform(0, 2 * np.pi, len(eX)), rng.uniform(0, 0.4, len(eX))
        g[:, 0], g[:, 1], g[:, 2] = eX, eY, rng.uniform(0, np.pi, len(eX))
        g[:, 3], g[:, 4], g[:, 5], g[:, 6], g[:, 7] = np.cos(xi), np.sin(xi), np.cos(ph), np.sin(ph), proj
        return g

    if name == "long":
        s = 1e5 / (np.max(np.hypot(u, v)) * freqs[-1])
        u, v, w = u * s, v * s, w * s
        l, m = around(10, 30, K)
        st = np.array([0, 0, 0, 1, 0, 1, 0, 0], dtype=np.uint8)
        g = gauss_tab(np.full(K, 1e-7), np.full(K, 2e-7), np.arange(K) % 2)
        cls = [cluster(l[:5], m[:5], rng.lognormal(0, 1, 5), st[:5], gauss=g[:5]),
               cluster(l[5:], m[5:], rng.lognormal(0, 1, 3), st[5:], gauss=g[5:])]
    elif name == "centre":
        u[:4] = v[:4] = w[:4] = 0.0
        l, m = around(0.5, 4, K)
        l[0] = m[0] = 0.0
        st = np.array([0, 1, 0, 1, 0, 0, 0, 0], dtype=np.uint8)
        g = gauss_tab(np.full(K, 3e-4), np.full(K, 1e-4), np.arange(K) % 2)
        cls = [cluster(l[:4], m[:4], rng.lognormal(0, 1, 4), st[:4], gauss=g[:4]),
               cluster(l[4:], m[4:], rng.lognormal(0, 1, 4), st[4:], gauss=g[4:])]
    elif name in ("widefd", "tinyfd"):
        fdelta = 40e6 if name == "widefd" else 1.0
        l, m = around(1, 8, K)
        cls = [cluster(l[:4], m[:4], rng.lognormal(0, 1, 4)), cluster(l[4:], m[4:], rng.lognormal(0, 1, 4))]
    elif name == "gauss":
        l, m = around(0.5, 4, K)
        eX = np.array([0.0, 1e-12, 1.0, 1.0, 2e-4, 1e-12, 0.7, 3e-4])
        eY = np.array([0.0, 3e-12, 1.0, 0.5, 1e-4, 1e-12, 1.2, 0.0])
        g = gauss_tab(eX, eY, np.arange(K) % 2)
        cls = [cluster(l[:4], m[:4], rng.lognormal(0, 1, 4), np.ones(4), gauss=g[:4]),
               cluster(l[4:], m[4:], rng.lognormal(0, 1, 4), np.ones(4), gauss=g[4:])]
    elif name == "bessel":
        from scipy import special
        l, m = around(0.5, 4, K)
        st = np.array([2, 2, 2, 3, 3, 3, 2, 3], dtype=np.uint8)
        zeros = {2: special.jn_zeros(1, 3), 3: special.jn_zeros(0, 3)}
        disk = {}
        rows = rng.choice(np.arange(4, len(u)), K, replace=False)
        for s in range(K):
            xi, ph = rng.uniform(0, 2 * np.pi), rng.uniform(0, 0.4)
            cxi, sxi, cph, sph = np.cos(xi), np.sin(xi), np.cos(ph), np.sin(ph)
            r, f = rows[s], freqs[0]
            up = u[r] * f * cxi - v[r] * f * cph * sxi + w[r] * f * sph * sxi
            vp = u[r] * f * sxi + v[r] * f * cph * cxi - w[r] * f * sph * cxi
            eX = zeros[int(st[s])][s % 3] / (2.0 * np.pi * np.hypot(up, vp))
            disk[s] = (eX, cxi, sxi, cph, sph, 1)
        cls = [cluster(l[:4], m[:4], rng.lognormal(0, 1, 4), st[:4], disk={s: disk[s] for s in range(4)}),
               cluster(l[4:], m[4:], rng.lognormal(0, 1, 4), st[4:],
                       disk={s - 4: disk[s] for s in range(4, K)})]
    elif name == "spectral":
        freqs = np.array([75e6, 150e6, 300e6])
        l, m = around(0.5, 4, K)
        sI0 = np.array([1.5, -2.0, 0.0, 0.8, -0.3, 2.2, 1.0, 0.6])
        sQ0 = np.array([0.0, 0.4, -0.1, 0.0, 0.2, -0.5, 0.0, 0.1])
        sU0 = np.array([-0.2, 0.0, 0.3, 0.1, 0.0, 0.0, -0.4, 0.0])
        sV0 = np.array([0.05, -0.01, 0.0, 0.0, 0.02, 0.0, 0.0, -0.03])
        spec = dict(sI0=sI0, sQ0=sQ0, sU0=sU0, sV0=sV0,
                    f0=np.array([150e6, 150e6, 75e6, 300e6, 150e6, 150e6, 140e6, 150e6]),
                    spec_idx=np.array([-0.7, 0.9, -0.7, 0.0, 1.3, -2.1, 0.0, -0.8]),
                    spec_idx1=np.array([0.05, -0.2, 0.0, 0.3, 0.1, 0.0, 0.4, -0.1]),
                    spec_idx2=np.array([-0.01, 0.03, 0.2, 0.0, 0.0, -0.05, 0.0, 0.02]))
        cls = []
        for a, z in ((0, 4), (4, 8)):
            cl = cluster(l[a:z], m[a:z], 0.9 * sI0[a:z] + 0.05)
            cl.update({kk: vv[a:z] for kk, vv in spec.items()})
            cls.append(cl)
    else:
        raise ValueError(name)
    return u, v, w, cls, freqs, fdelta


SKY_EDGE_CASES = ["long", "centre", "widefd", "tinyfd", "gauss", "bessel", "spectral"]


def lsum(a):
    """sum in long double (scalar references of the device reductions)"""
    return float(np.sum(np.asarray(a, dtype=np.longdouble)))


def relerr(a, b):
    """max |a - b| / max |b|.  b is the reference: where it is a stored sample of a large reference
    answer (oracle/refreplay.py leaves the elements outside the sample NaN) only the sample counts"""
    a = np.asarray(a)
    b = np.asarray(b)
    keep = ~np.isnan(b)
    if not keep.all():
        assert keep.any(), "no reference value to compare with"
        a, b = np.broadcast_to(a, b.shape)[keep], b[keep]
    return float(np.max(np.abs(a - b)) / (np.max(np.abs(b)) + 1e-300))


def mult_hessian_ref(g, s, y, rho, npairs, next_):
    """the two-loop recursion of the reference (mult_hessian, lbfgs.c:33-111) restated literally:
    the same `idx` order of the ring buffer (oldest ... newest pair), the same gamma from the newest
    pair; dot products summed in long double.  s, y [Mmem, m], rho [Mmem]; `npairs` valid pairs,
    `next_` the slot written next.  returns (H g, magnitude companion): the companion is the same
    recursion on absolute values, the scale of the rounding error of any summation order"""
    g = np.asarray(g, dtype=np.float64)
    s = np.asarray(s, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64)
    rho = np.asarray(rho, dtype=np.float64)
    M = npairs
    idx = np.zeros(M, dtype=int)
    if M > 0:
        ii = next_ - 1 if next_ > 0 else M - 1
        for ci in range(M - ii - 1):
            idx[ci] = ii + ci + 1
        for ci in range(M - ii - 1, M):
            idx[ci] = ci - M + ii + 1
    dot = lambda a, b: lsum(a * np.asarray(b, dtype=np.longdouble))
    pk, pa = g.copy(), np.abs(g)
    alphai, alpha_a = np.zeros(M), np.zeros(M)
    for ci in range(M):
        j = idx[M - ci - 1]
        alphai[M - ci - 1] = rho[j] * dot(s[j], pk)
        alpha_a[M - ci - 1] = abs(rho[j]) * dot(np.abs(s[j]), pa)
        pk = pk - alphai[M - ci - 1] * y[j]
        pa = pa + alpha_a[M - ci - 1] * np.abs(y[j])
    if M > 0:
        j = idx[M - 1]
        gamma = dot(s[j], y[j]) / dot(y[j], y[j])
        pk = pk * gamma
        pa = pa * (dot(np.abs(s[j]), np.abs(y[j])) / dot(y[j], y[j]))
    for ci in range(M):
        j = idx[ci]
        beta = rho[j] * dot(y[j], pk)
        beta_a = abs(rho[j]) * dot(np.abs(y[j]), pa)
        pk = pk + (alphai[ci] - beta) * s[j]
        pa = pa + (alpha_a[ci] + beta_a) * np.abs(s[j])
    return pk, pa


def lbfgs_pairs(m, Mmem, seed, cond=1e3, noise=1e-3, negative=None):
    """an LBFGS history of Mmem pairs of length m as a curvature model produces them: y = B s + noise
    with B SPD of condition ~cond (diagonal, a log-spaced spectrum in random order), rho = 1 / (y . s).  `negative`: the slot of one pair with y . s < 0
    (y flipped).  returns (g, s [Mmem, m], y [Mmem, m], rho [Mmem])"""
    rng = np.random.default_rng(seed)
    lam = np.exp(np.linspace(0.0, np.log(cond), m))[rng.permutation(m)]
    s = rng.normal(0, 1, (Mmem, m)) * rng.uniform(0.1, 2.0, (Mmem, 1))
    y = s * lam + noise * rng.normal(0, 1, (Mmem, m)) * np.sqrt(lam)
    if negative is not None:
        y[negative] = -y[negative]
    rho = 1.0 / np.einsum("ij,ij->i", y, s)
    g = rng.normal(0, 1, m)
    return g, s, y, rho


#: LBFGS runs traced iteration by iteration (tests/test_gpu_lbfgs.py) and checked against the compiled
#: reference (tests/test_oracle_vs_ref.py): (id, problem, lbfgs_m, max_lbfgs, robust).  Every run starts
#: from pp0 + 0.1 N(0, 1) (lbfgs_start) so that the search directions matter; max_lbfgs >= 2 lbfgs_m + 2
#: wraps the history at least twice.  Seeds are those whose line-search decisions all lie far above
#: rounding level (orc_lbfgs_traced's margin; the Gaussian product evaluates its costs from the quartic
#: of the line model, the restatement directly).  robust-m80 runs 66 iterations with 80 pairs: past
#: the 64 pairs k_lbfgs_direction once held.
LBFGS_TRACE_CASES = [
    ("gauss-plain-m1", dict(N=8, M=2, tilesz=8, seed=1), 1, 6, False),
    ("gauss-hybrid-m3", dict(N=8, M=3, tilesz=8, nchunk=[1, 2, 3], seed=1), 3, 10, False),
    ("gauss-plain-m7", dict(N=8, M=3, tilesz=8, kmean=1.0, seed=2), 7, 18, False),
    ("robust-plain-m3", dict(N=8, M=2, tilesz=8, outliers=0.02, seed=1), 3, 10, True),
    ("robust-hybrid-m7", dict(N=8, M=3, tilesz=8, nchunk=[2, 1, 3], outliers=0.02, seed=2), 7, 16,
     True),
    ("robust-m80", dict(N=20, M=8, tilesz=3, kmean=1.0, seed=4), 80, 66, True),
]
LBFGS_TRACE_NU = 4.0


def lbfgs_start(pr, seed):
    """the perturbed starting Jones of an LBFGS_TRACE_CASES run on the problem of that seed"""
    rng = np.random.default_rng(seed + 100)
    return pr.pp0 + 0.1 * rng.normal(0, 1, pr.pp0.shape)


# ---- the minibatch band passes (k_stream_band, k_grad_tma_band) ------------------------------------------
U64 = 2.0 ** -53   # unit roundoff of float64

#: (N, M, timeslots, channels, nchunk of the clusters, capacity maxnc) of the band cases
BAND_CASES = {
    "n2c1": (2, 1, 1, 1, [1], 1),
    "n2c3": (2, 1, 1, 3, [1], 3),
    "n9": (9, 3, 5, 2, [1, 2, 1], 2),
    "n33h3": (33, 7, 9, 5, [1, 3, 1, 1, 3, 1, 1], 5),
    "n33h4": (33, 7, 9, 5, [1, 4, 1, 1, 4, 1, 1], 5),
    "n62": (62, 64, 11, 4, [2 if k % 8 == 3 else (3 if k == 60 else 1) for k in range(64)], 4),
    "n9c33": (9, 2, 2, 33, [1, 1], 40),
    "n9all": (9, 3, 5, 2, [1, 2, 1], 2),
}


def maps_agree(tilesz, Nbase, nchunk):
    """whether the cost's row map (chunk_index over the rows) and the gradient's timeslot map
    (timeslot / ceil(tilesz / nchunk)) put every row in the same chunk"""
    R = Nbase * tilesz
    rows = np.arange(R)
    return all(np.array_equal(synth.chunk_index(rows, R, n), (rows // Nbase) // (-(-tilesz // n)))
               for n in nchunk)


def band_case(name, seed=41):
    """one band of a minibatch: a problem of BAND_CASES[name] observed at nc frequencies with the same
    Jones, data with noise and outliers and NON-ZERO on flagged rows; random flag-1 and uv-cut
    (flag 2) rows, one station and one timeslot fully flagged where others remain ("n9all": every
    row flagged).  Jones points: A near the truth (small residuals), B far from it (large).
    returns a dict: the problem fields, coh [nc][row][M][4] complex, x [nc][row][8], A, B, maxnc"""
    N, M, T, nc, nchunk, maxnc = BAND_CASES[name]
    rng = np.random.default_rng(seed + 7 * N + T)
    pr = synth.make_problem(N=N, M=M, tilesz=T, seed=seed + N, kmean=1.0, nchunk=nchunk,
                            flag_frac=0.0, uvcut_frac=0.0, with_data=False)
    R, Nb = pr.Nbase1, pr.Nbase
    fl = np.zeros(R, dtype=np.uint8)
    u = rng.uniform(0, 1, R)
    fl[u < 0.06] = 1
    fl[(u >= 0.06) & (u < 0.1)] = 2
    if N > 2:
        s = N // 2
        fl[(pr.sta1 == s) | (pr.sta2 == s)] = 1
    if T > 1:
        fl[:Nb] = 2
    if name == "n9all":
        fl[:] = 1
    pr.flag = fl
    freqs = 140e6 + 4e6 * np.arange(nc)
    cohs, xs = [], []
    for f in freqs:
        coh = synth.coherencies(pr.u, pr.v, pr.w, pr.clusters, f, pr.fdelta)
        x = synth.apply_jones(coh, pr.jones_true, pr.sta1, pr.sta2, N, pr.nchunk)
        sig = 1e-3 * np.median(np.abs(x))
        x = x + rng.normal(0, sig, x.shape)
        bad = rng.uniform(0, 1, x.shape) < 0.01
        x[bad] += rng.normal(0, 50 * sig, int(bad.sum()))
        cohs.append(coh.reshape(R, M, 4))
        xs.append(x.reshape(R, 8))
    m = 8 * N * pr.Mt
    A = pr.jones_true + 1e-4 * rng.normal(0, 1, m)
    B = pr.jones_true + 0.3 * rng.normal(0, 1, m)
    return dict(pr=pr, name=name, N=N, Nbase=Nb, tilesz=T, M=M, Mt=pr.Mt, nc=nc, nchunk=pr.nchunk,
                sta1=pr.sta1, sta2=pr.sta2, flag=fl, freqs=freqs, coh=np.array(cohs), x=np.array(xs),
                A=A, B=B, maxnc=maxnc, m=m)


def band_consensus(case, seed=5):
    """consensus terms (y, z, rho) of a band case"""
    rng = np.random.default_rng(seed)
    m = case["m"]
    return (0.1 * rng.normal(0, 1, m), case["pr"].jones_true + 0.05 * rng.normal(0, 1, m),
            rng.uniform(1.0, 10.0, case["Mt"]))


#: deliberate faults band_ref can apply to itself (tests/test_cpu_refs.py: sensitivity of the cases)
BAND_FAULTS = ("cost_timeslot_map", "grad_row_map", "drop_flagged_cost", "channel0_coherencies",
               "drop_last_timeslot_block", "drop_last_baseline_group", "grad_sign")


def _mm2(A, B):
    """products of stacks of 2x2 matrices, written out (broadcast over the leading axes)"""
    out = np.empty(np.broadcast_shapes(A.shape, B.shape), dtype=np.result_type(A, B))
    for i in range(2):
        for j in range(2):
            out[..., i, j] = A[..., i, 0] * B[..., 0, j] + A[..., i, 1] * B[..., 1, j]
    return out


def _scatter2(idx, V, n):
    """sum of the 2x2 matrices V [rows, 2, 2] into n slots by idx [rows]"""
    out = np.zeros((n, 2, 2), dtype=V.dtype)
    for i in range(2):
        for j in range(2):
            v = V[:, i, j]
            if np.iscomplexobj(v):
                out[:, i, j] = (np.bincount(idx, v.real, n) + 1j * np.bincount(idx, v.imag, n))
            else:
                out[:, i, j] = np.bincount(idx, v, n)
    return out


def band_ref(case, p, nu, y=None, z=None, rho=None, fault=None):
    """plain per-row float64 restatement of one band's minibatch passes
    (robust_cost_func_multifreq / robust_grad_func_multifreq, robust_batchmode_lbfgs.c:1096-1440):
      model     V = sum_k Jp C_k Jq^H, chunk of the row by the row map (chunk_index), zero on every
                flagged row (flag 1 and uv-cut 2)
      residual  e = x - V [nc][row][8]
      cost      sum log(1.0 + e e (1/nu)) over every channel, row and real component (func_robust_th)
      gradient  minus the sum over channels of the full-batch Student's-t gradient: 2 sum psi(e) dV/dtheta,
                psi(e) = e / (nu + e^2), over the unflagged rows, chunk by the timeslot map
                (timeslot / ceil(tilesz / nchunk), :1186-1196)
      consensus cost + sum_ci y.(p - z) + rho_ci/2 |p - z|^2, gradient - y - rho_ci (p - z)
    with the a-priori error budgets of any evaluation of the same sums in float64:
      res_bound  (M + 10) u (|x| + sum_k |Jp||C_k||Jq|^T) per element
      cost_bound rounding of each term, the residual error through 2e/(nu + e^2), the summation
      grad_bound per component: the rounding of 2 sum |psi(e)||dV/dtheta| plus the residual error
                 through psi'(e)
    The reference sum is accumulated in long double (lsum).  `fault` (one of BAND_FAULTS) makes the
    restatement deliberately wrong.  returns dict(cost, res, grad, res_bound, cost_bound, grad_bound)"""
    N, Nb, T, M, nc = case["N"], case["Nbase"], case["tilesz"], case["M"], case["nc"]
    R = Nb * T
    u = U64
    sta1, sta2 = case["sta1"], case["sta2"]
    flagged = case["flag"] != 0
    rows = np.arange(R)
    tslot = rows // Nb
    # rows a faulty kernel would never visit (TB = 2 timeslots per block, 32 baselines per group)
    skip = np.zeros(R, dtype=bool)
    if fault == "drop_last_timeslot_block":
        skip = tslot >= ((T - 1) // 2) * 2
    elif fault == "drop_last_baseline_group":
        skip = (rows % Nb) >= ((Nb - 1) // 32) * 32
    coh = np.moveaxis(case["coh"].reshape(nc, R, M, 2, 2), 2, 0)
    if fault == "channel0_coherencies":
        coh = np.broadcast_to(coh[:, :1], coh.shape)
    coh = np.ascontiguousarray(coh)   # [M][nc][row][2][2]
    xc = case["x"].reshape(nc, R, 4, 2)
    xc = (xc[..., 0] + 1j * xc[..., 1]).reshape(nc, R, 2, 2)
    P = np.asarray(p, dtype=np.float64).reshape(-1, N, 4, 2)
    J = (P[..., 0] + 1j * P[..., 1]).reshape(-1, N, 2, 2)
    aJ = np.abs(J)
    H = lambda X: np.conj(np.swapaxes(X, -1, -2))
    Tt = lambda X: np.swapaxes(X, -1, -2)
    c0 = np.concatenate([[0], np.cumsum(case["nchunk"])[:-1]]).astype(int)
    rmaps, tmaps = [], []
    for k in range(M):
        nch = case["nchunk"][k]
        rmaps.append(synth.chunk_index(rows, R, nch))
        tmaps.append(tslot // (-(-T // nch)))
    V = np.zeros((nc, R, 2, 2), dtype=np.complex128)
    Va = np.zeros((nc, R, 2, 2))
    for k in range(M):
        cm = c0[k] + (tmaps[k] if fault == "cost_timeslot_map" else rmaps[k])
        Jp, Jq = J[cm, sta1], J[cm, sta2]
        V += _mm2(_mm2(Jp, coh[k]), H(Jq))
        Va += _mm2(_mm2(aJ[cm, sta1], np.abs(coh[k])), Tt(aJ[cm, sta2]))
    V[:, flagged] = 0.0
    Va[:, flagged] = 0.0
    e = xc - V
    e[:, skip] = 0.0
    scale = np.abs(xc) + Va
    res = _api_layout(e.reshape(-1, 2, 2))
    res_bound = (M + 10) * u * np.repeat(scale.reshape(-1), 2)

    e8 = res.reshape(nc, R, 8)
    de8 = res_bound.reshape(nc, R, 8)
    terms = np.log(1.0 + e8 * e8 * (1.0 / nu))
    keep = ~skip
    if fault == "drop_flagged_cost":
        keep = keep & ~flagged
    terms = terms[:, keep]
    cost = lsum(terms)
    nterm = terms.size
    cost_bound = (lsum(2 * u * (3.0 + np.abs(terms))) + nterm * u * lsum(np.abs(terms))
                  + lsum((2 * np.abs(e8) / (nu + e8 * e8) * de8)[:, keep]))

    # gradient: per-row weights psi(e) and their error from the residual's, unflagged rows only
    use = ~flagged & ~skip
    psi = e8 / (nu + e8 * e8)
    dpsi = np.abs((nu - e8 * e8) / (nu + e8 * e8) ** 2) * de8
    W = (psi[..., 0::2] + 1j * psi[..., 1::2]).reshape(nc, R, 2, 2)
    Wa = (np.abs(psi[..., 0::2]) + np.abs(psi[..., 1::2])).reshape(nc, R, 2, 2)
    Wd = (dpsi[..., 0::2] + dpsi[..., 1::2]).reshape(nc, R, 2, 2)
    W[:, ~use] = 0.0
    Wa[:, ~use] = 0.0
    Wd[:, ~use] = 0.0
    Mt = J.shape[0]
    G = np.zeros((Mt * N, 2, 2), dtype=np.complex128)
    Ga = np.zeros((Mt * N, 2, 2))
    Gd = np.zeros((Mt * N, 2, 2))
    for k in range(M):
        gm = c0[k] + (rmaps[k] if fault == "grad_row_map" else tmaps[k])
        C = coh[k]
        Ca = np.abs(C)
        Jp, Jq, ap, aq = J[gm, sta1], J[gm, sta2], aJ[gm, sta1], aJ[gm, sta2]
        ip, iq = gm * N + sta1, gm * N + sta2
        # d/dJp of Re tr(W^H Jp C Jq^H): W Jq C^H;  d/dJq: W^H Jp C  (real and imaginary parts)
        n = Mt * N
        G += _scatter2(ip, _mm2(_mm2(W, Jq), H(C)).sum(axis=0), n)
        G += _scatter2(iq, _mm2(_mm2(H(W), Jp), C).sum(axis=0), n)
        Ga += _scatter2(ip, _mm2(_mm2(Wa, aq), Tt(Ca)).sum(axis=0), n)
        Ga += _scatter2(iq, _mm2(_mm2(Tt(Wa), ap), Ca).sum(axis=0), n)
        Gd += _scatter2(ip, _mm2(_mm2(Wd, aq), Tt(Ca)).sum(axis=0), n)
        Gd += _scatter2(iq, _mm2(_mm2(Tt(Wd), ap), Ca).sum(axis=0), n)
    grad = 2.0 * _api_layout(G.reshape(-1, 2, 2))
    if fault == "grad_sign":
        grad = -grad
    nsum = 8 * nc * max(N - 1, 1) * T + 16
    grad_bound = np.repeat((2.0 * (nsum * u * Ga + Gd)).reshape(-1), 2)

    if y is not None:
        d = np.asarray(p) - z
        rr = np.repeat(np.asarray(rho, dtype=np.float64), 8 * N)
        cons = y * d + 0.5 * rr * d * d
        cost = cost + lsum(cons)
        cost_bound += (len(d) + 4) * u * lsum(np.abs(y * d) + 0.5 * rr * d * d)
        gc = -y - rr * d
        grad_bound = grad_bound + 2 * u * (np.abs(grad) + np.abs(y) + rr * np.abs(d))
        grad = grad + gc
    return dict(cost=cost, res=res, grad=grad, res_bound=res_bound, cost_bound=cost_bound,
                grad_bound=grad_bound)


# ---- the LM cluster passes (k_cluster_pass_lin, k_cluster_pass_split, k_cluster_pass, k_cluster_rowmap)
#: c of the element-wise bound c u (|beta v| + |Jp||C||Jq|^T) of one model added to or subtracted from
#: a vector: two 2x2 complex products and the add, a few roundings each
CP_C = 10.0

#: (N, timeslots, nchunk of the clusters) of the cluster-pass cases (tests/test_gpu_cluster_pass.py)
CP_CASES = {
    "n7h": (7, 5, [1, 2, 3]),
    "n2": (2, 3, [1, 2]),
    "n23": (23, 5, [1, 2, 3]),
    "n24": (24, 5, [1, 2, 3]),
    "n9e": (9, 3, [1, 4]),
    "n9r": (9, 64, [1, 2]),
    "n62": (62, 120, [1]),
    "n512": (512, 2, [1]),
    "n639": (639, 2, [1]),
    "n640": (640, 2, [1]),
}

#: deliberate faults cluster_pass_ref can apply to itself (tests/test_cpu_refs.py)
CP_FAULTS = ("model_on_flagged", "beta_on_model", "gamma_one_minus_beta", "chunk_shift",
             "jq_not_hermitian", "jte_without_q", "drop_last_group", "drop_last_slice",
             "weights_once")


def cluster_case(name, seed=61):
    """one resident problem of CP_CASES[name]: random-phase coherencies, data = model at the true
    Jones plus noise, NON-ZERO on flagged rows; random flag-1 and uv-cut (flag 2) rows, one station
    (N > 2) and one timeslot (T > 1) fully flagged.  Jones: P near the truth, P_old farther from it;
    wt positive sqrt-weights, y a second input vector, out_init a non-zero vector (API layout)."""
    N, T, nchunk = CP_CASES[name]
    rng = np.random.default_rng(seed + 3 * N + T)
    M = len(nchunk)
    pr = synth.make_problem(N=N, M=M, tilesz=T, seed=seed + N, nchunk=nchunk, flag_frac=0.0,
                            uvcut_frac=0.0, with_data=False)
    R, Nb = pr.Nbase1, pr.Nbase
    fl = np.zeros(R, dtype=np.uint8)
    uu = rng.uniform(0, 1, R)
    fl[uu < 0.06] = 1
    fl[(uu >= 0.06) & (uu < 0.1)] = 2
    if N > 2:
        s = N // 2
        fl[(pr.sta1 == s) | (pr.sta2 == s)] = 1
    if T > 1:
        t = T // 2
        fl[t * Nb:(t + 1) * Nb] = 2
    pr.flag = fl
    amp = rng.lognormal(0.0, 0.5, (R, M, 4))
    coh = amp * np.exp(2j * np.pi * rng.uniform(0, 1, (R, M, 4)))
    pr.coh = coh.reshape(-1)
    x = synth.apply_jones(pr.coh, pr.jones_true, pr.sta1, pr.sta2, N, pr.nchunk)
    x = x + 0.01 * np.median(np.abs(x)) * rng.normal(0, 1, x.shape)
    pr.x = x
    m = 8 * N * pr.Mt
    return dict(pr=pr, name=name, N=N, Nbase=Nb, tilesz=T, M=M, nchunk=list(pr.nchunk),
                sta1=pr.sta1, sta2=pr.sta2, flag=fl, coh=coh, x=x,
                y=rng.normal(0, 1, x.shape) * np.median(np.abs(x)),
                wt=rng.uniform(0.2, 1.3, x.shape), out_init=rng.normal(0, 1, x.shape),
                P=pr.jones_true + 1e-3 * rng.normal(0, 1, m),
                P_old=pr.jones_true + 0.1 * rng.normal(0, 1, m))


def chunk_offset(case, k, ck):
    """offset of the Jones block of (cluster k, chunk ck) in the parameter vector"""
    return 8 * case["N"] * (int(sum(case["nchunk"][:k])) + ck)


def chunk_tiles(case, k, ck):
    """timeslots [t0, t1) of chunk ck of cluster k (the LM fits' ranges, lmfit.c:893-905)"""
    T = case["tilesz"]
    tc = -(-T // case["nchunk"][k])
    t0 = min(ck * tc, T)
    return t0, min(t0 + tc, T)


def _cplx(v):
    """API layout [8 R] -> [R, 2, 2] complex"""
    a = np.asarray(v, dtype=np.float64).reshape(-1, 4, 2)
    return (a[..., 0] + 1j * a[..., 1]).reshape(-1, 2, 2)


def _split(z):
    """[R, 2, 2] complex -> [R, 8] real (re, im per component)"""
    return _api_layout(z).reshape(-1, 8)


def _model(J, C, p, q, fault=None):
    """Jp C Jq^H and its magnitude companion |Jp||C||Jq|^T, per row"""
    Jp, Jq = J[p], J[q]
    Jh = Jq if fault == "jq_not_hermitian" else np.conj(np.swapaxes(Jq, -1, -2))
    m = _mm2(_mm2(Jp, C), Jh)
    A = _mm2(_mm2(np.abs(Jp), np.abs(C)), np.swapaxes(np.abs(Jq), -1, -2))
    return m, A


def cluster_pass_ref(case, k, ck, mode, x, pblk, write_out=True, with_jte=False, form_hidden=False,
                     beta=1.0, pblk_old=None, wt=None, out_init=None, inplace=False, fault=None):
    """plain per-row float64 restatement of one LM cluster pass (ClusterPassArgs, kernels_stream.cu)
    of cluster k, chunk ck over its timeslots [t0, t1), input vector x (API layout, full interval):
      model  m = Jp C Jq^H at pblk, zero on flag-1 and uv-cut rows; m_old the same at pblk_old
      v      x, or with form_hidden the hidden data beta x + m_old formed per row
      mode 0 INIT   d = beta v + m -> out, e = d - m
           1 TRIAL  e = v - m -> out
           2 ADD    out = beta v + m
           3 SUB    out = v - m, with pblk_old (not form_hidden) the recovered old residual added:
                    + (1-beta)/beta (v - m_old)
           4 GIVEN  e = v -> out
      cost   ||e||^2, or ||wt.e||^2 (modes 0, 1, 4), over every row of the chunk
      J^T e  station sums over the chunk's unflagged rows of E Jq C^H (station p) and E^H Jp C
             (station q), E = e or wt^2.e, in the parameter layout
    Rows outside the chunk, and every row without write_out, keep the output vector's content (x
    itself when inplace).  The a-priori bounds of any float64 evaluation:
      out_bound   CP_C u (|beta v| + |Jp||C||Jq|^T), plus CP_C u (|beta x| + |m_old|-companion) where
                  the second model forms v, plus (1-beta)/beta CP_C u (|v| + companion) to recover
      cost_bound  per-term rounding, the residual error through 2|e|, the summation
      jte_bound   n u sum |E||J||C| plus the residual error through |J||C|, per component
    Sums in long double.  `fault` (one of CP_FAULTS) makes the restatement deliberately wrong.
    returns dict(out, out_bound, cost, cost_bound, jte, jte_bound, rows=(r0, r1))"""
    N, Nb, T = case["N"], case["Nbase"], case["tilesz"]
    R = Nb * T
    u = U64
    t0, t1 = chunk_tiles(case, k, ck)
    if fault == "chunk_shift":
        t0, t1 = min(t0 + 1, T), min(t1 + 1, T)
    r0, r1 = t0 * Nb, t1 * Nb
    rows = np.arange(r0, r1)
    keep = np.ones(r1 - r0, dtype=bool)   # rows a faulty kernel would still visit
    if fault == "drop_last_group":
        keep &= (rows % Nb) < ((Nb - 1) // 256) * 256
    elif fault == "drop_last_slice":
        keep &= rows < max(r0, r1 - Nb)
    p, q = case["sta1"][r0:r1], case["sta2"][r0:r1]
    fl = case["flag"][r0:r1] != 0
    C = case["coh"].reshape(R, case["M"], 2, 2)[r0:r1, k]
    v = _cplx(x)[r0:r1]
    vw = np.abs(v)
    m, A = _model(_jones(pblk, N), C, p, q, fault)
    old = pblk_old is not None and (form_hidden or mode == 3)
    if old:
        mo, Ao = _model(_jones(pblk_old, N), C, p, q, fault)
    if fault != "model_on_flagged":
        m[fl] = 0.0
        A[fl] = 0.0
        if old:
            mo[fl] = 0.0
            Ao[fl] = 0.0
    cu = CP_C * u
    dv = np.zeros(v.shape)
    if form_hidden:
        v = (v + beta * mo) if fault == "beta_on_model" else (beta * v + mo)
        dv = cu * (np.abs(beta) * vw + Ao)
    add = lambda a, b: (a + beta * b) if fault == "beta_on_model" else (beta * a + b)
    e = None
    if mode in (0, 2):
        o = add(v, m)
        do = cu * (np.abs(beta) * np.abs(v) + A) + np.abs(beta) * dv
        if mode == 0:
            e = o - m
    elif mode == 4:
        e = o = v
        do = dv
    else:
        e = v - m
        o = e
        do = cu * (np.abs(v) + A) + dv
        if mode == 3 and pblk_old is not None and not form_hidden:
            g = (1.0 - beta) if fault == "gamma_one_minus_beta" else (1.0 - beta) / beta
            o = e + g * (v - mo)
            do = do + abs((1.0 - beta) / beta) * cu * (np.abs(v) + Ao)
    de = do if e is not None else None
    base = np.array(x if inplace else (np.zeros(8 * R) if out_init is None else out_init),
                    dtype=np.float64)
    out = base.copy().reshape(R, 8)
    out_bound = np.zeros((R, 8))
    if write_out:
        sel = rows[keep]
        out[sel] = _split(o)[keep]
        out_bound[sel] = np.repeat(do.reshape(-1, 4)[keep], 2, axis=1)
    res = dict(out=out.reshape(-1), out_bound=out_bound.reshape(-1), cost=0.0, cost_bound=0.0,
               jte=np.zeros(8 * N), jte_bound=np.zeros(8 * N), rows=(r0, r1))
    if mode not in (0, 1, 4):
        return res
    w = np.ones((r1 - r0, 8)) if wt is None else np.asarray(wt, dtype=np.float64).reshape(R, 8)[r0:r1]
    e8 = _split(e)
    de8 = np.repeat(de.reshape(-1, 4), 2, axis=1)
    terms = ((w * e8) ** 2)[keep]
    res["cost"] = lsum(terms)
    res["cost_bound"] = (lsum(3 * u * terms) + lsum((2 * w * w * np.abs(e8) * de8 + (w * de8) ** 2)[keep])
                         + terms.size * u * lsum(terms))
    if with_jte:
        use = keep & ~fl
        w2 = w if fault == "weights_once" else w * w
        E8 = np.where(use[:, None], w2 * e8, 0.0)
        Ea8 = np.abs(E8)
        Ed8 = np.where(use[:, None], w * w * de8, 0.0)
        to2 = lambda a: (a[:, 0::2] + 1j * a[:, 1::2]).reshape(-1, 2, 2)
        E = to2(E8)
        Ea = (Ea8[:, 0::2] + Ea8[:, 1::2]).reshape(-1, 2, 2)
        Ed = (Ed8[:, 0::2] + Ed8[:, 1::2]).reshape(-1, 2, 2)
        J = _jones(pblk, N)
        aJ = np.abs(J)
        H = lambda X: np.conj(np.swapaxes(X, -1, -2))
        Tt = lambda X: np.swapaxes(X, -1, -2)
        Ca = np.abs(C)
        nt = t1 - t0
        G = _scatter2(p, _mm2(_mm2(E, J[q]), H(C)), N)
        Ga = _scatter2(p, _mm2(_mm2(Ea, aJ[q]), Tt(Ca)), N)
        Gd = _scatter2(p, _mm2(_mm2(Ed, aJ[q]), Tt(Ca)), N)
        if fault != "jte_without_q":
            G += _scatter2(q, _mm2(_mm2(H(E), J[p]), C), N)
        Ga += _scatter2(q, _mm2(_mm2(Tt(Ea), aJ[p]), Ca), N)
        Gd += _scatter2(q, _mm2(_mm2(Tt(Ed), aJ[p]), Ca), N)
        nsum = 8 * max(N - 1, 1) * max(nt, 1) + 16
        res["jte"] = _api_layout(G)
        res["jte_bound"] = np.repeat((nsum * u * Ga + Gd).reshape(-1), 2)
    return res


def cluster_rowmap_ref(case, k, sign, beta, pp, r, dh, fault=None):
    """plain per-row float64 restatement of db_cluster_hidden (k_cluster_rowmap) for cluster k at the
    full Jones vector pp, the chunk of a row by the row map (synth.chunk_index, as line_model_ref):
      sign > 0  hidden data  beta r + m
      sign < 0  residual     dh - m (+ (1-beta) r when beta != 1)
    m zero on flag-1 and uv-cut rows.  returns (out, bound) over every row, bound
    CP_C u (|beta r| + |dh| + |(1-beta) r| + |Jp||C||Jq|^T) of the terms that enter"""
    N, R = case["N"], case["Nbase"] * case["tilesz"]
    rows = np.arange(R)
    nch = case["nchunk"][k]
    px = synth.chunk_index(rows, R, nch)
    J = _jones(np.asarray(pp)[chunk_offset(case, k, 0):chunk_offset(case, k, nch)], N * nch)
    idx = px * N
    C = case["coh"].reshape(R, case["M"], 2, 2)[:, k]
    m, A = _model(J, C, idx + case["sta1"], idx + case["sta2"], fault)
    if fault != "model_on_flagged":
        fl = case["flag"] != 0
        m[fl] = 0.0
        A[fl] = 0.0
    rv, dv = _cplx(r), _cplx(dh)
    if sign > 0:
        o = (rv + beta * m) if fault == "beta_on_model" else (beta * rv + m)
        b = CP_C * U64 * (abs(beta) * np.abs(rv) + A)
    else:
        o = dv - m
        b = CP_C * U64 * (np.abs(dv) + A)
        if beta != 1.0:
            o = o + (1.0 - beta) * rv
            b = b + CP_C * U64 * abs(1.0 - beta) * np.abs(rv)
    return _api_layout(o), np.repeat(b.reshape(-1), 2)


#: the passes each cluster-pass case runs: (name, arguments); old: the visit's entry Jones P_old as
#: pblk_old, wt: the case's weights.  init/trial with and without output, J^T e and weights; the trial
#: that forms the hidden data with J^T e (k_cluster_pass_lin<true> reloads the old Jones per row) and
#: without it (the last trial, which writes the residual); ADD with beta; SUB plain, recovering at beta
#: 1/2, 1/8, 1/64 and forming the hidden data in place; the given-residual pass of the OS-LM
CP_RUNS = [
    ("init", dict(mode=0, write_out=True, with_jte=True)),
    ("init_beta", dict(mode=0, write_out=True, with_jte=True, beta=0.125)),
    ("init_quiet", dict(mode=0, write_out=False)),
    ("init_beta_out", dict(mode=0, write_out=True, beta=0.125)),
    ("trial", dict(mode=1, write_out=True, with_jte=True)),
    ("trial_quiet", dict(mode=1, write_out=False)),
    ("trial_wt", dict(mode=1, write_out=True, with_jte=True, wt=True)),
    ("trial_wt_cost", dict(mode=1, write_out=False, wt=True)),
    ("trial_form", dict(mode=1, write_out=False, with_jte=True, form_hidden=True, old=True)),
    ("trial_form_last", dict(mode=1, write_out=True, form_hidden=True, old=True)),
    ("add", dict(mode=2, write_out=True, beta=0.125)),
    ("add_quiet", dict(mode=2, write_out=False)),
    ("sub", dict(mode=3, write_out=True)),
    ("sub_rec2", dict(mode=3, write_out=True, beta=0.5, old=True)),
    ("sub_rec8", dict(mode=3, write_out=True, beta=0.125, old=True)),
    ("sub_rec64", dict(mode=3, write_out=True, beta=1.0 / 64, old=True)),
    ("sub_form_inplace", dict(mode=3, write_out=True, form_hidden=True, old=True, inplace=True)),
    ("given", dict(mode=4, write_out=True, with_jte=True, wt=True)),
]


def cp_lin_fits(N, Nbase):
    """whether the linear-mapped pass takes the array (kernels_stream.cu: cluster_pass_lin_fits): 8N
    station sums next to a 5-stage ring in 200 KB of shared memory, at most 1024 baseline groups"""
    return 5 * 8 * 256 * 16 + 8 * ((8 * N + 1) & ~1) + 40 <= 200 * 1024 and (Nbase + 255) // 256 <= 1024


def cp_run_applies(case, name, kw):
    """form_hidden runs only where the linear-mapped kernel takes the array; the given-residual pass
    at n24 and n640"""
    if kw.get("form_hidden") and not cp_lin_fits(case["N"], case["Nbase"]):
        return False
    return kw["mode"] != 4 or case["name"] in ("n24", "n640")


def cp_ref_args(case, k, ck, kw):
    """the arguments of cluster_pass_ref (and of DeviceProblem.cluster_pass) for run kw on (k, ck)"""
    N = case["N"]
    off = chunk_offset(case, k, ck)
    return dict(mode=kw["mode"], x=case["x"], pblk=case["P"][off:off + 8 * N],
                write_out=kw.get("write_out", True), with_jte=kw.get("with_jte", False),
                form_hidden=kw.get("form_hidden", False), beta=kw.get("beta", 1.0),
                pblk_old=case["P_old"][off:off + 8 * N] if kw.get("old") else None,
                wt=case["wt"] if kw.get("wt") else None, out_init=case["out_init"],
                inplace=kw.get("inplace", False))


def cp_expected_kernel(case, k, ck, kw):
    """the kernel db_launch_cluster_pass picks for run kw (kernels_stream.cu)"""
    t0, t1 = chunk_tiles(case, k, ck)
    if t1 <= t0:
        return "none"
    fits = cp_lin_fits(case["N"], case["Nbase"])
    if not kw.get("with_jte") or kw["mode"] in (2, 3):
        return "lin" if (fits and not kw.get("wt")) else "tile"
    if kw["mode"] == 4 or kw.get("wt") or not fits:
        return "split"
    return "lin_grad"


# ---- the full-interval passes (k_stream_all<0>, k_grad_tma_split) ---------------------------------------
#: (N, M, timeslots, nchunk of the clusters) of the full-interval cases (tests/test_gpu_interval_passes.py)
INTERVAL_CASES = {
    "n2": (2, 1, 1, [1]),
    "n9": (9, 3, 5, [1, 2, 1]),
    "n33h3": (33, 7, 9, [1, 3, 1, 1, 3, 1, 1]),
    "n33h4": (33, 7, 9, [1, 4, 1, 1, 4, 1, 1]),
    "n40m1": (40, 1, 3, [1]),
    "n40m2": (40, 2, 3, [1, 1]),
    "n40m4": (40, 4, 3, [1, 1, 1, 1]),
    "n62": (62, 64, 11, [2 if k % 8 == 3 else (3 if k == 60 else 1) for k in range(64)]),
    "n62t120": (62, 8, 120, [1, 1, 1, 1, 1, 3, 1, 1]),
    "n512": (512, 32, 5, [2 if k == 20 else 1 for k in range(32)]),
    "n520": (520, 4, 2, [1, 1, 1, 1]),
    "all-flagged": (9, 3, 5, [1, 2, 1]),
}

#: deliberate faults interval_ref can apply to itself (tests/test_cpu_refs.py: sensitivity of the cases)
INTERVAL_FAULTS = ("grad_over_flagged", "grad_row_map", "robust_weight_complex",
                   "drop_last_timeslot_block", "drop_last_q_tile", "drop_last_p_of_tile",
                   "stale_ring_stage", "drop_third_warp", "grad_sign")


def interval_case(name, seed=71):
    """one resident interval of INTERVAL_CASES[name]: random-phase coherencies whose cluster
    amplitudes span three decades (cluster 0 the brightest), data = model at the true Jones plus noise
    and 1 % outliers, NON-ZERO on flagged rows; random flag-1 and uv-cut (flag 2) rows, one station
    (N > 2) and one timeslot (T > 1) fully flagged ("all-flagged": every row).  Jones points: A near
    the truth (small residuals), B far from it, half: A with the first half of its values zeroed.
    Coherencies are [row][M][4] complex, the data in API layout."""
    N, M, T, nchunk = INTERVAL_CASES[name]
    rng = np.random.default_rng(seed + 5 * N + M + T)
    pr = synth.make_problem(N=N, M=M, tilesz=T, seed=seed + N, nchunk=nchunk, flag_frac=0.0,
                            uvcut_frac=0.0, with_data=False)
    R, Nb = pr.Nbase1, pr.Nbase
    fl = np.zeros(R, dtype=np.uint8)
    uu = rng.uniform(0, 1, R)
    fl[uu < 0.06] = 1
    fl[(uu >= 0.06) & (uu < 0.1)] = 2
    if N > 2:
        s = N // 2
        fl[(pr.sta1 == s) | (pr.sta2 == s)] = 1
    if T > 1:
        t = T // 2
        fl[t * Nb:(t + 1) * Nb] = 2
    if name == "all-flagged":
        fl[:] = 1
    pr.flag = fl
    amp = 10.0 ** -rng.uniform(0.0, 3.0, M)
    amp[0] = 1.0
    coh = np.empty((R, M, 4), dtype=np.complex128)
    for k in range(M):
        coh[:, k] = (amp[k] * rng.lognormal(0.0, 0.5, (R, 4))) * np.exp(2j * np.pi
                                                                        * rng.uniform(0, 1, (R, 4)))
    pr.coh = coh.reshape(-1)
    x = synth.apply_jones(pr.coh, pr.jones_true, pr.sta1, pr.sta2, N, pr.nchunk)
    sig = 1e-3 * np.median(np.abs(x))
    x += rng.normal(0, sig, x.shape)
    bad = rng.uniform(0, 1, x.shape) < 0.01
    x[bad] += rng.normal(0, 50 * sig, int(bad.sum()))
    pr.x = x
    m = 8 * N * pr.Mt
    A = pr.jones_true + 1e-4 * rng.normal(0, 1, m)
    half = A.copy()
    half[:m // 2] = 0.0
    return dict(pr=pr, name=name, N=N, Nbase=Nb, tilesz=T, M=M, Mt=pr.Mt, nchunk=list(pr.nchunk),
                sta1=pr.sta1, sta2=pr.sta2, flag=fl, coh=coh, x=x, m=m, amp=amp,
                points=dict(A=A, B=pr.jones_true + 0.3 * rng.normal(0, 1, m), half=half))


def _ld_scatter(idx, vals, n, cache, key, off=0):
    """sums of the rows of vals [rows, 8] into n slots by off + idx, accumulated in long double; the
    sort of idx is kept in cache[key] (one station map serves every cluster of one chunk count)"""
    if key not in cache:
        order = np.argsort(idx, kind="stable")
        si = idx[order]
        starts = np.flatnonzero(np.r_[True, si[1:] != si[:-1]])
        cache[key] = (order, starts, si[starts])
    order, starts, slots = cache[key]
    out = np.zeros((n, vals.shape[1]), dtype=np.longdouble)
    if len(order):
        out[off + slots] = np.add.reduceat(vals[order], starts, axis=0, dtype=np.longdouble)
    return out


def interval_ref(case, p, nus=(None,), fault=None):
    """plain per-row restatement of the full-interval passes, dirac_b200_predict (k_stream_all<0>) and
    dirac_b200_grad (k_grad_tma_split), i.e. of the reference's minimize_viz_full_pth, cost_func /
    robust_cost_func and grad_func / robust_grad_func (robust_lbfgs.c:424-560,155-316,674-735):
      model     V = sum_k Jp C_k Jq^H, the chunk of a row by the row map (chunk_index, lmfit.c:655),
                zero on every flagged row (flag 1 and uv-cut 2)
      residual  e = x - V, every row (x itself on flagged rows)
      cost      nu None: sum e^2 over every row and real component (flagged rows count with their
                data); nu: sum log(1 + e e (1/nu)) (func_robust_th)
      gradient  over the unflagged rows only, the chunk by the timeslot map (timeslot /
                ceil(tilesz / nchunk), robust_lbfgs.c:197-207,465-475), with the reference's signs:
                nu None  +2 sum Re(conj(e) dV/dtheta)      (-2 Re((f - x)^H df), :554)
                nu       -2 sum psi(e) dV/dtheta, psi(e) = e / (nu + e^2) per real component (:299)
    with the a-priori error budgets of any float64 evaluation of the same sums:
      res_bound  (M + 10) u (|x| + sum_k |Jp||C_k||Jq|^T) per element (also bounds the model's error)
      cost_bound rounding of each term, the residual error through d(term)/de, the summation
      grad_bound per component: 2 (n u sum |psi(e)||dV/dtheta| + sum |psi'(e)| res_bound |dV/dtheta|),
                 n = 8 (N - 1) T + 16
    One cluster at a time; the sums are accumulated in long double.  `nus`: the gradients and costs to
    take (None: Gaussian), all from the one model.  `fault` (one of INTERVAL_FAULTS) makes the
    restatement deliberately wrong.  returns dict(model, res, res_bound, passes={nu: dict(cost,
    cost_bound, grad, grad_bound)})"""
    N, Nb, T, M = case["N"], case["Nbase"], case["tilesz"], case["M"]
    R = Nb * T
    u = U64
    sta1, sta2 = case["sta1"], case["sta2"]
    flagged = case["flag"] != 0
    rows = np.arange(R)
    tslot = rows // Nb
    coh = case["coh"].reshape(R, M, 2, 2)
    xc = _cplx(case["x"])
    J = _jones(p, N * case["Mt"]).reshape(-1, N, 2, 2)
    aJ = np.abs(J)
    H = lambda X: np.conj(np.swapaxes(X, -1, -2))
    Tt = lambda X: np.swapaxes(X, -1, -2)
    c0 = np.concatenate([[0], np.cumsum(case["nchunk"])[:-1]]).astype(int)
    rmap = lambda nch: synth.chunk_index(rows, R, nch)
    tmap = lambda nch: tslot // (-(-T // nch))
    # rows a faulty kernel would never visit: the last time block of the predict (2 timeslots) and of
    # the gradient (4)
    skip_m = np.zeros(R, dtype=bool)
    skip_g = np.zeros(R, dtype=bool)
    if fault == "drop_last_timeslot_block":
        skip_m = tslot >= ((T - 1) // 2) * 2
        skip_g = tslot >= ((T - 1) // 4) * 4

    # a cluster whose Jones are all zero adds exactly nothing to the model and has a zero gradient
    live = [J[c0[k]:c0[k] + case["nchunk"][k]].any() for k in range(M)]
    V = np.zeros((R, 2, 2), dtype=np.clongdouble)
    Va = np.zeros((R, 2, 2))
    for k in range(M):
        if (fault == "drop_third_warp" and k % 3 == 2) or not live[k]:
            continue
        cm = c0[k] + rmap(case["nchunk"][k])
        C = np.ascontiguousarray(coh[:, k])
        V += _mm2(_mm2(J[cm, sta1], C), H(J[cm, sta2]))
        Va += _mm2(_mm2(aJ[cm, sta1], np.abs(C)), Tt(aJ[cm, sta2]))
    V = V.astype(np.complex128)
    V[flagged] = 0.0
    Va[flagged] = 0.0
    e = xc - V
    e[skip_m] = 0.0
    res = _api_layout(e)
    res_bound = (M + 10) * u * np.repeat((np.abs(xc) + Va).reshape(-1), 2)
    out = dict(model=_api_layout(V), res=res, res_bound=res_bound, passes={})

    e8 = res.reshape(R, 8)
    de8 = res_bound.reshape(R, 8)
    keep = ~skip_m
    use = ~skip_g if fault == "grad_over_flagged" else (~flagged & ~skip_g)
    psis = {}
    for nu in nus:
        if nu is None:
            terms = (e8 * e8)[keep]
            cost_bound = (lsum(2 * u * terms) + lsum((2 * np.abs(e8) * de8 + de8 * de8)[keep])
                          + terms.size * u * lsum(terms))
            psi, dpsi = e8, de8
        else:
            terms = np.log(1.0 + e8 * e8 * (1.0 / nu))[keep]
            cost_bound = (lsum(2 * u * (3.0 + terms)) + terms.size * u * lsum(terms)
                          + lsum((2 * np.abs(e8) / (nu + e8 * e8) * de8)[keep]))
            if fault == "robust_weight_complex":
                a2 = np.repeat(e8[:, 0::2] ** 2 + e8[:, 1::2] ** 2, 2, axis=1)
                psi = e8 / (nu + a2)
            else:
                psi = e8 / (nu + e8 * e8)
            dpsi = np.abs((nu - e8 * e8) / (nu + e8 * e8) ** 2) * de8
        psi = np.where(use[:, None], psi, 0.0)
        dpsi = np.where(use[:, None], dpsi, 0.0)
        W = (psi[:, 0::2] + 1j * psi[:, 1::2]).reshape(R, 2, 2)
        Wa = (np.abs(psi[:, 0::2]) + np.abs(psi[:, 1::2])).reshape(R, 2, 2)
        Wd = (dpsi[:, 0::2] + dpsi[:, 1::2]).reshape(R, 2, 2)
        psis[nu] = (W, Wa, Wd)
        out["passes"][nu] = dict(cost=lsum(terms), cost_bound=cost_bound)

    nslot = case["Mt"] * N
    nsum = 8 * max(N - 1, 1) * T + 16
    G = {nu: np.zeros((nslot, 8), dtype=np.longdouble) for nu in nus}
    Gb = {nu: np.zeros((nslot, 2, 2)) for nu in nus}
    # which rows reach each end's sums: the faults that drop a kernel tile or a tile's last p
    reach_p = np.ones(R, dtype=bool)
    reach_q = np.ones(R, dtype=bool)
    if fault == "drop_last_q_tile":
        reach_p = reach_q = (sta2 // 32) != (N - 1) // 32
    elif fault == "drop_last_p_of_tile":
        reach_p = (sta1 % 8) != 7
    cache = {}
    for k in range(M):
        if not live[k]:
            continue
        nch = case["nchunk"][k]
        mk = "row" if fault == "grad_row_map" else "time"
        lm = rmap(nch) if mk == "row" else tmap(nch)
        gm = c0[k] + lm
        kc = k - 2 if (fault == "stale_ring_stage" and k >= 2) else k
        C = np.ascontiguousarray(coh[:, kc])
        Ca = np.abs(C)
        ip, iq = gm * N + sta1, gm * N + sta2
        JqC = _mm2(J[gm, sta2], H(C))        # d/dJp of Re tr(W^H Jp C Jq^H): W Jq C^H
        JpC = _mm2(J[gm, sta1], C)           # d/dJq: W^H Jp C
        aJqC = _mm2(aJ[gm, sta2], Tt(Ca))
        aJpC = _mm2(aJ[gm, sta1], Ca)
        for nu in nus:
            W, Wa, Wd = psis[nu]
            vp = _split(_mm2(W, JqC)) * reach_p[:, None]
            vq = _split(_mm2(H(W), JpC)) * reach_q[:, None]
            G[nu] += _ld_scatter(lm * N + sta1, vp, nslot, cache, ("p", mk, nch), c0[k] * N)
            G[nu] += _ld_scatter(lm * N + sta2, vq, nslot, cache, ("q", mk, nch), c0[k] * N)
            Wb = nsum * u * Wa + Wd
            Gb[nu] += _scatter2(ip, _mm2(Wb, aJqC), nslot)
            Gb[nu] += _scatter2(iq, _mm2(Tt(Wb), aJpC), nslot)
    for nu in nus:
        sign = 2.0 if nu is None else -2.0
        if fault == "grad_sign":
            sign = -sign
        out["passes"][nu]["grad"] = (sign * G[nu]).astype(np.float64).reshape(-1)
        out["passes"][nu]["grad_bound"] = np.repeat((2.0 * Gb[nu]).reshape(-1), 2)
    return out
