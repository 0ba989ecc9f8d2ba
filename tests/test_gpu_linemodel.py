"""The LBFGS line model (E0, E1, E2 of k_stream_all<1>), its quartic (k_line_poly),
the direct line costs (k_line_eval) and the line residual (k_line_residual) against a plain numpy
restatement, in both launch shapes of k_stream_all<1>.

k_stream_all<1> runs one warp per item with a 4-stage ring once the grid has at least 64 items
(32 baselines x 1 timeslot) per SM, and three warps per item with a cross-warp combine below that.
The solver's line search differentiates its costs numerically, so a wrong E1 or E2 could still let
a whole LBFGS run find some step: these tests read the line model directly."""
import math

import numpy as np
import pytest

from sagecal_b200 import lib as blib
from util import line_model_ref, lsum, relerr, small_problem

pytestmark = pytest.mark.gpu

ALPHAS = np.array([0.0, 1e-6, 0.37, 1.0, -0.5, 3.0])
NU = 3.5
ALPHA_RES = 0.63

SMALL_SHAPE = (1, 2, 3)   # (TB, NST, WARPS) below 64 items per SM
LARGE_SHAPE = (1, 4, 1)   # at or above


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _large_tilesz(N):
    """timeslots that put a problem of N stations 25 % above the 64-items-per-SM threshold"""
    nbg = (N * (N - 1) // 2 + 31) // 32
    return int(math.ceil(1.25 * 64 * _sm_count() / nbg))


CASES = {
    # 40 stations: 780 baselines (last group 12 lanes), 11 clusters over 3 warps (ring refills)
    "small-hybrid": (dict(N=40, M=11, tilesz=12, seed=61, kmean=1.0,
                          nchunk=[1, 2, 1, 1, 4, 1, 1, 1, 3, 1, 1]), SMALL_SHAPE),
    # fewer clusters than warps: one warp has none
    "small-M2": (dict(N=33, M=2, tilesz=7, seed=62), SMALL_SHAPE),
    # 100 stations: 4950 baselines (last group 22 lanes); 6 clusters through a 4-stage ring
    "large-hybrid": (dict(N=100, M=6, tilesz=None, seed=63, nchunk=[1, 3, 1, 2, 1, 1]), LARGE_SHAPE),
    "large-M1": (dict(N=100, M=1, tilesz=None, seed=64), LARGE_SHAPE),
}


def _case(name):
    case, shape = CASES[name]
    case = dict(case)
    if case["tilesz"] is None:
        case["tilesz"] = _large_tilesz(case["N"])
    return case, shape


def make_case(case):
    """(bound problem, xk, pk) of a case dict: N, M, tilesz, seed, optional nchunk / kmean"""
    kw = {k: v for k, v in case.items() if k in ("nchunk", "kmean")}
    b = small_problem(N=case["N"], M=case["M"], tilesz=case["tilesz"], seed=case["seed"], **kw)
    rng = np.random.default_rng(case["seed"] + 1000)
    xk = b.pr.pp0 + 0.1 * rng.normal(0, 1, b.pr.pp0.shape)
    pk = 0.05 * rng.normal(0, 1, b.pr.pp0.shape)
    return b, xk, pk


def run_case(api, b, xk, pk):
    pr = b.pr
    with blib.DeviceProblem(api, pr.N, pr.Nbase, pr.tilesz, b.barr, b.sky, pr.coh, pr.x) as dp:
        return dp.line_model(xk, pk, ALPHAS, NU, ALPHA_RES)


def check_line_model(b, xk, pk, got):
    pr = b.pr
    V0, V1, V2 = line_model_ref(pr, xk, pk)
    E0, E1, E2 = pr.x - V0, V1, V2
    # e(a) = E0 - a E1 - a^2 E2 (kernels_tma.cu epilogue)
    assert relerr(got["E0"], E0) < 1e-13
    assert relerr(got["E1"], E1) < 1e-13
    assert relerr(got["E2"], E2) < 1e-13
    # flagged and uv-cut rows carry no model: the residual there is the data
    fl = np.repeat(pr.flag != 0, 8)
    assert fl.any() and (pr.flag == 2).any()
    assert np.array_equal(got["E0"][fl], pr.x[fl])
    assert not got["E1"][fl].any() and not got["E2"][fl].any()

    s00, s11, s22 = lsum(E0 * E0), lsum(E1 * E1), lsum(E2 * E2)
    s01, s02, s12 = lsum(E0 * E1), lsum(E0 * E2), lsum(E1 * E2)
    q = [s00, -2.0 * s01, s11 - 2.0 * s02, 2.0 * s12, s22]
    poly = got["poly"]
    assert abs(poly[0] - q[0]) <= 1e-12 * q[0]
    assert abs(poly[4] - q[4]) <= 1e-12 * q[4]
    # signed sums: bounded by their Cauchy-Schwarz scale
    assert abs(poly[1] - q[1]) <= 1e-12 * 2.0 * math.sqrt(s00 * s11)
    assert abs(poly[2] - q[2]) <= 1e-12 * (s11 + 2.0 * math.sqrt(s00 * s22))
    assert abs(poly[3] - q[3]) <= 1e-12 * 2.0 * math.sqrt(s11 * s22)

    for i, a in enumerate(ALPHAS):
        e = E0 - a * E1 - a * a * E2
        cg, cr = lsum(e * e), lsum(np.log1p(e * e / NU))
        assert abs(got["cost_gauss"][i] - cg) <= 1e-12 * cg, (a, got["cost_gauss"][i], cg)
        assert abs(got["cost_robust"][i] - cr) <= 1e-12 * cr, (a, got["cost_robust"][i], cr)
        # the quartic the Gaussian line search evaluates against the direct reduction
        terms = [poly[j] * a ** j for j in range(5)]
        assert abs(sum(terms) - got["cost_gauss"][i]) <= 1e-12 * sum(abs(t) for t in terms)
    a = ALPHA_RES
    assert relerr(got["res"], E0 - a * E1 - a * a * E2) < 1e-13


@pytest.mark.parametrize("name", list(CASES))
def test_line_model(api, name):
    case, shape = _case(name)
    b, xk, pk = make_case(case)
    items = (b.pr.Nbase + 31) // 32 * b.pr.tilesz
    assert (items >= 64 * _sm_count()) == (shape == LARGE_SHAPE)
    got = run_case(api, b, xk, pk)
    assert got["shape"] == shape, (name, items, got["shape"])
    check_line_model(b, xk, pk, got)

