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
