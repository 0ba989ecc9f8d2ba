"""GPU: the minibatch band passes directly.  k_stream_band (kernels_band.cu: the Student's-t cost of
every channel of a band in one launch, or its residual) and k_grad_tma_band (grad_tma_split_body<...,
BAND=true>, kernels_stream.cu: the gradient with the reference's minibatch sign) through the functions
the minibatch fits call (BandFn of minibatch.cu, hook dirac_b200_band_eval), against util.band_ref,
the plain per-row float64 restatement that tests/test_cpu_refs.py pins to the compiled reference.

Cases (util.BAND_CASES; N stations, M clusters, T timeslots, nc channels):
  n2c1, n2c3   N 2, M 1, T 1, nc 1 / 3: one baseline, warps 1 and 2 of k_stream_band without clusters
  n9           N 9, M 3, T 5, nc 2: partial baseline group, remainder timeslot blocks of both kernels,
               nchunk [1, 2, 1] (row and timeslot chunk maps disagree)
  n33h3, n33h4 N 33, M 7, T 9, nc 5: second q block of gradient tiles, staging ring refill and parity
               flip, nchunk 3 (maps agree) and 4 (maps disagree, chunk 3 has no gradient)
  n62          N 62, M 64, T 11, nc 4: the profiled shape reduced in time, 60 baseline groups with 3
               lanes in the last, 22 clusters per warp, hybrid clusters
  n9c33        N 9, M 2, T 2, nc 33 in a band state of capacity 40
  n9all        every row flagged: the cost is the data-only sum, the gradient exactly 0
Every case has random flag-1 and uv-cut rows with non-zero data, one fully flagged station and one
fully flagged timeslot where rows remain besides them (not at N 2, T 1: one row).  Each runs at nu 2
and 30, with and without the consensus terms, on the sequence A, B, A, A with half its Jones zeroed,
A (A near the truth: small residuals, B far from it).  The file reads nothing of the reference."""
import numpy as np
import pytest

from sagecal_b200.dirac_api import SkyModel, make_barr
from util import BAND_CASES, band_case, band_consensus, band_ref

pytestmark = pytest.mark.gpu

_cases = {}
_refs = {}


def _case(name):
    if name not in _cases:
        c = band_case(name)
        pr = c["pr"]
        c["barr"] = make_barr(pr.sta1, pr.sta2, pr.flag)
        c["sky"] = SkyModel(pr.clusters, pr.N)
        _cases[name] = c
    return _cases[name]


def _ref(name, which, p, nu, cons):
    key = (name, which, nu, cons is not None)
    if key not in _refs:
        _refs[key] = band_ref(_case(name), p, nu, *(cons or ()))
    return _refs[key]


def _eval(api, c, P, nu, cons, Nf=None, maxnc=None):
    Y, Z, rho = cons if cons is not None else (None, None, None)
    pr = c["pr"]
    return api.band_eval(pr.N, pr.Nbase, pr.tilesz, c["barr"], c["sky"], c["coh"], c["x"],
                         c["nc"] if Nf is None else Nf, P, nu,
                         maxnc=c["maxnc"] if maxnc is None else maxnc, Y=Y, Z=Z, rho=rho)


def _ratio(err, bound):
    return float(np.max(np.where(err == 0, 0.0, err / np.maximum(bound, 1e-300))))


@pytest.mark.parametrize("consensus", [False, True], ids=["plain", "consensus"])
@pytest.mark.parametrize("nu", [2.0, 30.0])
@pytest.mark.parametrize("name", list(BAND_CASES))
def test_band_passes_match_restatement(api, name, nu, consensus):
    c = _case(name)
    cons = band_consensus(c) if consensus else None
    A, B = c["A"], c["B"]
    half = A.copy()
    half[:c["m"] // 2] = 0.0
    pts = {"A": A, "B": B, "half": half}
    seq = ["A", "B", "A", "half", "A"]
    P = np.array([pts[s] for s in seq])
    k13, k14 = api.kernel_count(13), api.kernel_count(14)
    out = _eval(api, c, P, nu, cons)
    assert out is not None
    npts = len(seq)
    # one k_stream_band launch per cost, a residual launch of it and a k_grad_tma_band launch per
    # gradient
    assert api.kernel_count(13) - k13 == 2 * npts
    assert api.kernel_count(14) - k14 == npts
    # the grid reduction of the cost is deterministic: the same Jones give the same bits
    assert out["cost"][0] == out["cost"][2] == out["cost"][4]
    worst = dict(res=0.0, cost=0.0, grad=0.0)
    for i, s in enumerate(seq):
        r = _ref(name, s, pts[s], nu, cons)
        worst["cost"] = max(worst["cost"], abs(out["cost"][i] - r["cost"]) / r["cost_bound"])
        assert abs(out["cost"][i] - r["cost"]) <= r["cost_bound"], (s, out["cost"][i], r["cost"])
        # the gradients are summed by atomicAdd: bounded, not bit-identical
        err = np.abs(out["grad"][i] - r["grad"])
        worst["grad"] = max(worst["grad"], _ratio(err, r["grad_bound"]))
        assert (err <= r["grad_bound"]).all(), (s, _ratio(err, r["grad_bound"]))
    r = _ref(name, "A", A, nu, cons)
    err = np.abs(out["res"] - r["res"])
    worst["res"] = _ratio(err, r["res_bound"])
    assert (err <= r["res_bound"]).all(), worst["res"]
    if name == "n9all":
        # no unflagged row: the data-only cost, no model gradient at all
        g0 = np.zeros(c["m"]) if cons is None else -cons[0] - np.repeat(cons[2], 8 * c["N"]) * (
            A - cons[1])
        assert np.array_equal(out["grad"][0], 0.0 + g0)
        assert np.array_equal(out["res"], c["x"].reshape(-1))
    print("band %s nu %g %s: largest error / bound: residual %.3g, cost %.3g, gradient %.3g"
          % (name, nu, "consensus" if consensus else "plain", worst["res"], worst["cost"],
             worst["grad"]))


@pytest.mark.parametrize("consensus", [False, True], ids=["visibilities", "consensus"])
@pytest.mark.parametrize("name", ["n9", "n33h4", "n9c33"])
def test_band_cost_is_the_fits_res0(api, name, consensus):
    """the hook's first cost times 1.0 / n (the operation the fit applies) is res_0 of
    bfgsfit_minibatch_visibilities / _consensus with no iterations, bit for bit, n = 8 R Nf"""
    c = _case(name)
    pr = c["pr"]
    cons = band_consensus(c) if consensus else None
    nu = 5.0
    out = _eval(api, c, c["B"][None], nu, cons, maxnc=c["nc"])
    n = 8 * pr.Nbase1 * c["nc"]
    pt = api.persist_init(1, c["m"], n, 5)
    Y, Z, rho = cons if cons is not None else (None, None, None)
    r0, _ = api.bfgsfit_minibatch(pr.u, pr.v, pr.w, c["x"].reshape(-1).copy(), pr.N, pr.Nbase,
                                  pr.tilesz, c["barr"], c["sky"], c["coh"].reshape(-1).copy(),
                                  c["B"].copy(), c["freqs"], pt, max_lbfgs=0, lbfgs_m=5,
                                  robust_nu=nu, Y=Y, Z=Z, rho=rho)
    api.persist_clear(pt)
    assert r0 == out["cost"][0] * (1.0 / n), (r0, out["cost"][0] * (1.0 / n))


def test_band_eval_refusals(api):
    """Nf > maxnc, npts < 1 and Nf < 0 are refused before any device work"""
    c = _case("n9")
    before = (api.launch_count(), api.kernel_count(13), api.kernel_count(14))
    assert _eval(api, c, c["A"][None], 2.0, None, maxnc=c["nc"] - 1) is None
    assert _eval(api, c, np.zeros((0, c["m"])), 2.0, None) is None
    assert _eval(api, c, c["A"][None], 2.0, None, Nf=-1) is None
    assert (api.launch_count(), api.kernel_count(13), api.kernel_count(14)) == before


def test_band_without_channels_is_the_consensus_terms(api):
    """Nf = 0: no launch, the cost and gradient of the consensus terms alone"""
    c = _case("n9")
    cons = band_consensus(c)
    k13 = api.kernel_count(13)
    out = _eval(api, c, c["B"][None], 2.0, cons, Nf=0)
    assert api.kernel_count(13) == k13
    y, z, rho = cons
    d = c["B"] - z
    rr = np.repeat(rho, 8 * c["N"])
    assert np.array_equal(out["grad"][0], 0.0 + (-y - rr * d))
    want = sum(np.dot(d[i:i + 8 * c["N"]], y[i:i + 8 * c["N"]]) for i in range(0, c["m"], 8 * c["N"]))
    want += 0.5 * np.dot(rr * d, d)
    assert abs(out["cost"][0] - want) <= 1e-13 * (np.abs(y * d).sum() + np.dot(rr * d, d))
