"""GPU: the full-interval passes directly.  k_stream_all<0, 2, 2, 3> (kernels_tma.cu: the model over
all clusters, the residual and the Gaussian or Student's-t cost) and k_grad_tma_split<4, 2>
(grad_tma_split_body, kernels_stream.cu: the all-cluster gradient from the stored residual) through the
hooks dirac_b200_predict, dirac_b200_cost and dirac_b200_grad of a resident problem, against
util.interval_ref, the plain per-row restatement that tests/test_cpu_refs.py pins to the compiled
reference.  These are the passes of every LBFGS stage of the full-batch fits.

Cases (util.INTERVAL_CASES; N stations, M clusters, T timeslots):
  n2             2 x 1 x 1: one baseline, 31 idle lanes, the ring prologue covers every cluster
  n9             9 x 3 x 5, nchunk [1, 2, 1]: partial last time block of both kernels, row and
                 timeslot chunk maps disagree
  n33h3, n33h4   33 x 7 x 9, nchunk 3 / 4: second q tile, M not a multiple of the 3 warps; with 4
                 chunks over 9 timeslots chunk 3 has no gradient (exactly 0)
  n40m1/m2/m4    40 x 1 / 2 / 4 x 3: k_stream_all warps without a cluster, or with two
  n62            62 x 64 x 11, hybrid clusters: the C2 geometry reduced in time
  n62t120        62 x 8 x 120: 30 gradient time blocks, the C3 tile's length
  n512           512 x 32 x 5, cluster 20 in 2 chunks: C4's clusters per GPU (16 wraps of the
                 gradient's two-stage ring), a chunk boundary inside a time block, a partial last block
  n520           520 x 4 x 2: ragged p and q tiles above 512 stations
  all-flagged    9 x 3 x 5, every row flagged: gradient exactly 0, cost the data-only sum
Every case has random flag-1 and uv-cut rows with non-zero data, one fully flagged station and one
fully flagged timeslot (not at N 2, T 1: one row); cluster amplitudes span three decades.  Jones
points: A near the truth (small residuals: cancellation), B far from it, A with half its values
zeroed.  Gaussian and Student's t at nu 2 and 30 (n512: nu 2).  The file reads nothing of the
reference."""
import time

import numpy as np
import pytest

from sagecal_b200 import lib as blib
from sagecal_b200.dirac_api import SkyModel, make_barr
from util import INTERVAL_CASES, interval_case, interval_ref

pytestmark = pytest.mark.gpu

POINTS = ("A", "B", "half")
_cases = {}


def _case(name):
    if name not in _cases:
        c = interval_case(name)
        pr = c["pr"]
        c["barr"] = make_barr(pr.sta1, pr.sta2, pr.flag)
        c["sky"] = SkyModel(pr.clusters, pr.N)
        _cases[name] = c
    return _cases[name]


def _nus(name):
    return (None, 2.0) if name == "n512" else (None, 2.0, 30.0)


def _ratio(err, bound):
    err = np.asarray(err, dtype=np.float64)
    return float(np.max(np.where(err == 0, 0.0, err / np.maximum(bound, 1e-300)), initial=0.0))


def _zero_blocks(c):
    """parameter indices whose gradient is exactly 0 whatever the Jones: every component of the fully
    flagged station, in every chunk block, and every chunk block with no timeslot under the timeslot
    map (nchunk 4 over 9 timeslots: chunk 3)"""
    N, T = c["N"], c["tilesz"]
    idx = []
    blk = 0
    for nch in c["nchunk"]:
        tpc = -(-T // nch)
        for ck in range(nch):
            base = 8 * N * (blk + ck)
            if ck * tpc >= T:
                idx.extend(range(base, base + 8 * N))
            elif N > 2:
                s = N // 2
                idx.extend(range(base + 8 * s, base + 8 * s + 8))
        blk += nch
    return np.array(idx, dtype=np.int64)


@pytest.mark.parametrize("name", list(INTERVAL_CASES))
def test_interval_passes_match_restatement(api, name):
    t_start = time.perf_counter()
    c = _case(name)
    pr = c["pr"]
    x = c["x"]
    flagged = c["flag"] != 0
    zero = _zero_blocks(c)
    nus = _nus(name)
    worst = dict(model=0.0, res=0.0, cost=0.0, grad=0.0, repeat=0.0)
    t_ref = 0.0
    with blib.DeviceProblem(api, pr.N, pr.Nbase, pr.tilesz, c["barr"], c["sky"], pr.coh, x) as dp:
        for s in POINTS:
            P = c["points"][s]
            t0 = time.perf_counter()
            r = interval_ref(c, P, nus)
            t_ref += time.perf_counter() - t0
            _, model = dp.predict(P, out_mode=2)
            # flagged rows carry no model at all
            assert not model.reshape(-1, 8)[flagged].any(), s
            err = np.abs(model - r["model"])
            worst["model"] = max(worst["model"], _ratio(err, r["res_bound"]))
            assert (err <= r["res_bound"]).all(), (s, _ratio(err, r["res_bound"]))
            for nu in nus:
                q = r["passes"][nu]
                robust = nu is not None
                cost, res = dp.predict(P, out_mode=1, cost_mode=2 if robust else 1,
                                       nu=nu if robust else 0.0)
                err = np.abs(res - r["res"])
                worst["res"] = max(worst["res"], _ratio(err, r["res_bound"]))
                assert (err <= r["res_bound"]).all(), (s, nu, _ratio(err, r["res_bound"]))
                # the grid reduction of the cost is deterministic: the same Jones give the same bits
                cost2 = dp.cost(P, robust=robust, nu=nu if robust else 0.0)
                assert cost2 == cost, (s, nu, cost, cost2)
                worst["cost"] = max(worst["cost"], abs(cost - q["cost"]) / q["cost_bound"])
                assert abs(cost - q["cost"]) <= q["cost_bound"], (s, nu, cost, q["cost"])
                g = dp.grad(P, robust=robust, nu=nu if robust else 0.0)
                err = np.abs(g - q["grad"])
                worst["grad"] = max(worst["grad"], _ratio(err, q["grad_bound"]))
                bad = np.flatnonzero(err > q["grad_bound"])
                assert bad.size == 0, (s, nu, "first components off (block, station, component)",
                                       [(int(i) // (8 * c["N"]), int(i) // 8 % c["N"], int(i) % 8)
                                        for i in bad[:8]], _ratio(err, q["grad_bound"]))
                assert not g[zero].any(), (s, nu)
                # the gradient is summed by atomicAdd: a second call agrees within the budget, not
                # necessarily bit for bit
                g2 = dp.grad(P, robust=robust, nu=nu if robust else 0.0)
                err = np.abs(g2 - g)
                worst["repeat"] = max(worst["repeat"], _ratio(err, q["grad_bound"]))
                assert (err <= q["grad_bound"]).all(), (s, nu)
                if name == "all-flagged":
                    assert np.array_equal(res, x)
                    assert not g.any()
    print("interval %s: largest error / bound: model %.3g, residual %.3g, cost %.3g, gradient %.3g, "
          "repeated gradient %.3g; restatement %.1f s of %.1f s"
          % (name, worst["model"], worst["res"], worst["cost"], worst["grad"], worst["repeat"], t_ref,
             time.perf_counter() - t_start))
