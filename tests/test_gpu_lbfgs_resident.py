"""The LBFGS stage of a SAGE call on the residual the solvers keep resident.

* After the sweeps, every solver mode leaves the residual x - sum_k model_k of the Jones it hands
  back in the problem's residual buffer: the LBFGS stage starts from it without a predict (the
  `sweep_residual` option hands it back as the call's answer).
* After a full-batch LBFGS stage that accepted a step, that buffer holds the residual at the
  returned Jones (the line residual of the last accepted step): res_1 and x_out come from it without
  a predict.  A call without an LBFGS step predicts its final residual afresh, as before.
* On one GPU the line-model pass (k_stream_all<1>) also sums the Gaussian quartic along the line; it
  equals the separate pass over E0, E1 and E2 (k_line_poly) that sharded runs take.
A full-batch solve with LBFGS steps runs one all-cluster predict (res_0) and as many gradient passes
as before: one at the start and one per accepted step."""
import ctypes as C
import math

import numpy as np
import pytest

from sagecal_b200 import lib as blib
from test_gpu_linemodel import CASES, LARGE_SHAPE, SMALL_SHAPE, _sm_count, make_case
from util import lsum, relerr, small_problem

pytestmark = pytest.mark.gpu

PREDICT, GRAD, LINE_SETUP = 0, 1, 7   # dirac_b200_kernel_count kinds

#: the reduced C2/C3 shape (62 stations, 8 clusters, 10 timeslots); clusters 2 and 5 are hybrid,
#: and 3 chunks do not tile 10 timeslots (row-mapped hidden data, db_cluster_hidden)
REDUCED = dict(N=62, M=8, tilesz=10, seed=91, kmean=1.0, flag_frac=0.05, nchunk=[1, 1, 2, 1, 1, 3, 1, 1])
MODES = [0, 1, 2, 3, 4, 5, 6]


def residual_held(dp):
    """the residual the resident problem holds, API layout"""
    L = dp.api.lib
    L.dirac_b200_residual.restype = None
    L.dirac_b200_residual.argtypes = [C.c_void_p, blib.c_double_p]
    out = np.zeros(dp.n)
    L.dirac_b200_residual(dp.h, blib.dptr(out))
    return out


@pytest.fixture
def sweep_residual(api):
    api.set_option("sweep_residual", 1)
    yield
    api.set_option("sweep_residual", 0)


def counts(api):
    return [api.kernel_count(k) for k in (PREDICT, GRAD, LINE_SETUP)]


def solve(api, b, **kw):
    """sagefit on a fresh resident problem; returns (result, Jones, x_out, residual held after the
    call, fresh predict residual at the Jones, [predicts, gradients, line setups] of the call)"""
    pr = b.pr
    with blib.DeviceProblem(api, pr.N, pr.Nbase, pr.tilesz, b.barr, b.sky, pr.coh, pr.x) as dp:
        pp = pr.pp0.copy()
        xo = np.zeros(dp.n)
        c0 = counts(api)
        res = dp.sagefit(pp, xo, **kw)
        n = [c1 - c for c, c1 in zip(c0, counts(api))]
        held = residual_held(dp)
        _, fresh = dp.predict(pp, out_mode=1)
    return res, pp, xo, held, fresh, n


def check_residual(b, res, xo, held, fresh):
    assert relerr(xo, fresh) < 1e-12, relerr(xo, fresh)
    assert np.array_equal(xo, held)
    # res_1 = ||r|| / n of that residual
    r1 = math.sqrt(lsum(fresh * fresh)) / fresh.size
    assert abs(res[3] - r1) <= 1e-12 * r1, (res[3], r1)


@pytest.mark.parametrize("mode", MODES)
def test_sweep_residual_is_current(api, sweep_residual, mode):
    """the residual the sweeps kept, handed back with max_lbfgs = 0, is the one at the Jones they
    returned"""
    b = small_problem(**REDUCED)
    res, pp, xo, held, fresh, n = solve(api, b, max_emiter=3, max_iter=3, max_lbfgs=0, lbfgs_m=7,
                                        solver_mode=mode, randomize=1)
    print(mode, res, relerr(xo, fresh))
    assert res[3] < res[2]
    check_residual(b, res, xo, held, fresh)
    assert n == [1, 0, 0]


def test_no_lbfgs_step_predicts_the_final_residual(api):
    """without an LBFGS step the final residual is a fresh predict (the sweeps' incremental one
    carries their rounding)"""
    b = small_problem(**REDUCED)
    res, pp, xo, held, fresh, n = solve(api, b, max_emiter=2, max_iter=2, max_lbfgs=0, lbfgs_m=7,
                                        solver_mode=1)
    assert np.array_equal(xo, fresh)
    assert n == [2, 0, 0]


@pytest.mark.parametrize("mode", MODES)
def test_lbfgs_stage_residual_is_current(api, mode):
    """the benchmark's LBFGS settings: the stage starts from the sweeps' residual and leaves the one
    at its answer; one predict per call, one gradient pass at the start and one per accepted step"""
    b = small_problem(**REDUCED)
    res, pp, xo, held, fresh, n = solve(api, b, max_emiter=2, max_iter=2, max_lbfgs=10, lbfgs_m=7,
                                        solver_mode=mode)
    print(mode, res, relerr(xo, fresh), n)
    check_residual(b, res, xo, held, fresh)
    npred, ngrad, nline = n
    assert npred == 1
    assert 2 <= ngrad <= 11
    assert ngrad - 1 <= nline <= ngrad


def test_lbfgs_early_break_residual_is_current(api):
    """a stage whose line search rejects a step before max_lbfgs: the residual at the last
    accepted iterate"""
    b = small_problem(N=6, M=1, tilesz=4, seed=5)
    res, pp, xo, held, fresh, n = solve(api, b, max_emiter=1, max_iter=2, max_lbfgs=200, lbfgs_m=5,
                                        solver_mode=1)
    npred, ngrad, nline = n
    print(res, n)
    # one line search more than accepted steps: the loop ended on a rejected step
    assert ngrad - 1 < 200 and nline == ngrad
    check_residual(b, res, xo, held, fresh)
    assert npred == 1


def test_lbfgs_trace_break_residual_is_current(api):
    """the bfgsfit path (fresh predict at entry) ending on a rejected step: the residual left behind
    is the one at the returned Jones"""
    b = small_problem(N=6, M=1, tilesz=4, seed=5)
    pr = b.pr
    rng = np.random.default_rng(105)
    p0 = pr.pp0 + 0.1 * rng.normal(0, 1, pr.pp0.shape)
    with blib.DeviceProblem(api, pr.N, pr.Nbase, pr.tilesz, b.barr, b.sky, pr.coh, pr.x) as dp:
        t = dp.lbfgs_trace(p0, 200, 5)
        held = residual_held(dp)
        _, fresh = dp.predict(t["p"], out_mode=1)
    assert 0 < t["niter"] < 200 and t["gnorm"][-1] > 1e-17
    assert relerr(held, fresh) < 1e-12


def line_poly_direct(dp):
    L = dp.api.lib
    L.dirac_b200_line_poly.restype = None
    L.dirac_b200_line_poly.argtypes = [C.c_void_p, blib.c_double_p]
    poly = np.zeros(5)
    L.dirac_b200_line_poly(dp.h, blib.dptr(poly))
    return poly


POLY_CASES = dict(CASES)
# the station counts of the benchmark's workloads: 62 (C2/C3, three warps per item) and 512 (C4, one
# warp per item with a 4-stage ring)
POLY_CASES["n62"] = (dict(N=62, M=8, tilesz=10, seed=65, nchunk=[1, 1, 2, 1, 1, 3, 1, 1]), SMALL_SHAPE)
POLY_CASES["n512"] = (dict(N=512, M=2, tilesz=None, seed=66), LARGE_SHAPE)


@pytest.mark.parametrize("name", list(POLY_CASES))
def test_folded_quartic_matches_line_poly(api, name):
    case, shape = POLY_CASES[name]
    case = dict(case)
    if case["tilesz"] is None:
        nbg = (case["N"] * (case["N"] - 1) // 2 + 31) // 32
        case["tilesz"] = int(math.ceil(1.25 * 64 * _sm_count() / nbg))
    b, xk, pk = make_case(case)
    pr = b.pr
    with blib.DeviceProblem(api, pr.N, pr.Nbase, pr.tilesz, b.barr, b.sky, pr.coh, pr.x) as dp:
        got = dp.line_model(xk, pk, [0.0], 3.5, 0.5)
        direct = line_poly_direct(dp)
    assert got["shape"] == shape
    E0, E1, E2 = got["E0"], got["E1"], got["E2"]
    s00, s11, s22 = lsum(E0 * E0), lsum(E1 * E1), lsum(E2 * E2)
    # bound of each coefficient's rounding: its sum of |terms| (Cauchy-Schwarz for the signed ones)
    scale = [s00, 2.0 * math.sqrt(s00 * s11), s11 + 2.0 * math.sqrt(s00 * s22),
             2.0 * math.sqrt(s11 * s22), s22]
    poly = got["poly"]
    err = [abs(poly[j] - direct[j]) / scale[j] for j in range(5)]
    print(name, err)
    assert max(err) <= 1e-13, err
