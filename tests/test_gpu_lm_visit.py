"""The plain LM visit of a one-chunk cluster (lm.cu db_lm_chunk) never stores the hidden data
d = r + f(p_entry): every pass forms it from the residual r and the entry Jones, and the trial of the
last LM iteration writes d - f(p_trial), which becomes the residual when that trial is accepted.  A
visit that ends any other way (a rejected last trial, a stop before the last trial, a budget shared
out by `randomize`) runs the closing pass.  These tests count the passes and hold every way a visit
can end against the compiled reference."""
import ctypes as C

import numpy as np
import pytest

from util import small_problem, relerr
from test_gpu_solvers import run_both, JONES_TOL

pytestmark = pytest.mark.gpu

KIND_GRAD_PASS, KIND_PLAIN_PASS = 2, 8  # J^T e carrying passes; ADD / SUB / cost-only passes


@pytest.fixture
def cp_rows(api):
    def setter(v):
        api.set_option("cp_rows", v)
    yield setter
    api.set_option("cp_rows", 0)


def lm_stats(api, reset=False):
    """(accepted, accepted with mu/3, rejected) LM trials since the last reset"""
    out = (C.c_long * 4)()
    api.lib.dirac_b200_lm_stats(out, 1 if reset else 0)
    return list(out)[:3]


@pytest.mark.parametrize("max_iter,grad_passes", [(2, 2), (1, 1)])
def test_visit_passes(api, max_iter, grad_passes):
    """every trial accepted: per visit INIT and the trials of the first max_iter-1 iterations carry
    J^T e, the last trial is a cost-only pass that writes the residual, and no closing pass runs"""
    b = small_problem(N=12, M=3, tilesz=10, seed=301)
    pr = b.pr
    max_emiter = 2
    visits = max_emiter * pr.M
    x, pp = pr.x.copy(), pr.pp0.copy()
    lm_stats(api, reset=True)
    api.profile_enable(True)
    try:
        r = api.sagefit_visibilities(pr.u, pr.v, pr.w, x, pr.N, pr.Nbase, pr.tilesz, b.fresh_barr(),
                                     b.sky, pr.coh, pp, max_emiter=max_emiter, max_iter=max_iter,
                                     max_lbfgs=0, lbfgs_m=5, solver_mode=1, randomize=0)
        grad = api.profile_read(KIND_GRAD_PASS)[0]
        plain = api.profile_read(KIND_PLAIN_PASS)[0]
    finally:
        api.profile_enable(False)
    acc, _, rej = lm_stats(api, reset=True)
    assert r[3] < r[2]
    assert rej == 0 and acc == visits * max_iter, (acc, rej)
    assert grad == visits * grad_passes, grad
    assert plain == visits, plain


def _problem(name):
    # 30 stations: 435 baselines, a second baseline group of 179; a tenth of the rows flagged, 2 %
    # under the uv cut
    common = dict(N=30, M=3, tilesz=12, flag_frac=0.1, uvcut_frac=0.02)
    if name == "rejected":
        # Jones far from the identity start: some trials are rejected (9 in the CPU restatement,
        # none of them at rounding level)
        return small_problem(seed=312, jones_amp=2.5, **common), dict(max_iter=3)
    if name == "stopped":
        # noise-free data and the true Jones as the start: every visit stops on its entry tests
        # before it evaluates a trial (no uv cut: those rows keep their data, the model skips them)
        b = small_problem(seed=312, noise_rel=0.0, **dict(common, uvcut_frac=0.0))
        b.pr.pp0 = b.pr.jones_true.copy()
        return b, dict(max_iter=3)
    # every other sweep shares the iteration budget out by the clusters' last cost reductions
    return small_problem(seed=313, kmean=1.0, **common), dict(max_iter=3, randomize=1, max_emiter=4)


@pytest.mark.parametrize("rows", [0, 5])
@pytest.mark.parametrize("name", ["rejected", "stopped", "randomize"])
def test_visit_endings_match_reference(api, ref, cp_rows, name, rows):
    b, args = _problem(name)
    kw = dict(max_emiter=3, max_lbfgs=0, lbfgs_m=5, randomize=0, solver_mode=1)
    kw.update(args)
    cp_rows(rows)
    lm_stats(api, reset=True)
    (rr, xr, ppr), (rg, xg, ppg) = run_both(api, ref, b, **kw)
    acc, _, rej = lm_stats(api, reset=True)
    if name == "rejected":
        assert rej > 0
    if name == "stopped":
        assert acc == 0 and rej == 0
        assert np.max(np.abs(ppg - b.pr.jones_true)) < 1e-9
    assert rr[0] == rg[0]
    # (the "stopped" residual is at rounding level: res_0 ~ 1e-18, compared in absolute terms)
    assert abs(rr[2] - rg[2]) <= 1e-10 * rr[2] + 1e-16
    assert relerr(ppg, ppr) < JONES_TOL, (name, relerr(ppg, ppr))
    # the residual, measured against the data
    assert np.max(np.abs(xg - xr)) <= 1e-10 * np.max(np.abs(b.pr.x)), np.max(np.abs(xg - xr))


def test_hybrid_sky_alternates_both_visits(api, ref, cp_rows):
    """one-chunk clusters (residual handed over by the last trial) next to hybrid clusters (hidden
    data stored, closing pass) on the same residual buffer"""
    b = small_problem(N=12, M=3, tilesz=20, seed=321, nchunk=[2, 1, 5], flag_frac=0.1)
    cp_rows(4)
    (rr, xr, ppr), (rg, xg, ppg) = run_both(api, ref, b, max_emiter=3, max_iter=3, max_lbfgs=0,
                                            lbfgs_m=5, randomize=0, solver_mode=1)
    assert rr[0] == rg[0]
    assert abs(rr[2] - rg[2]) <= 1e-10 * rr[2]
    assert relerr(ppg, ppr) < JONES_TOL, relerr(ppg, ppr)
    assert np.max(np.abs(xg - xr)) <= 1e-10 * np.max(np.abs(b.pr.x)), np.max(np.abs(xg - xr))
