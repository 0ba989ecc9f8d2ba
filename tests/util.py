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
