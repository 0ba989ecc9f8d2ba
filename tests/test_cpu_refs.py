"""CPU: the plain references the GPU tests of the line model, the RTR evaluator, the IRLS update, the
LBFGS two-loop recursion and the segmented sky staging lean on, pinned against the restatement
(oracle/liboracle.so) before a GPU is involved."""
import numpy as np
import pytest

import orcdirac
from util import (big_cluster_sky, irls_ref, lbfgs_pairs, line_model_ref, mult_hessian_ref, relerr,
                  rtr_eval_ref, rtr_weights_ref, small_problem, split_cluster)

needs_oracle = pytest.mark.skipif(not orcdirac.available(), reason="oracle/liboracle.so not built")


@needs_oracle
@pytest.mark.parametrize("nchunk", [None, [1, 3, 2]], ids=["plain", "hybrid"])
def test_line_model_reference_is_the_model_along_the_line(nchunk):
    """V0 + a V1 + a^2 V2 of the numpy line model is the full model at xk + a pk"""
    b = small_problem(N=11, M=3, tilesz=7, seed=81, kmean=1.0, nchunk=nchunk)
    pr = b.pr
    rng = np.random.default_rng(3)
    xk = pr.pp0 + 0.1 * rng.normal(0, 1, pr.pp0.shape)
    pk = 0.05 * rng.normal(0, 1, pr.pp0.shape)
    V0, V1, V2 = line_model_ref(pr, xk, pk)
    orc = orcdirac.Oracle(pr)
    for a in (0.0, 0.7, -2.5):
        assert relerr(V0 + a * V1 + a * a * V2, orc.predict_full(xk + a * pk)) < 1e-14
    assert np.abs(V2).max() > 1e-3 * np.abs(V0).max()   # the quadratic term is not negligible


def _rtr_case(flags, seed):
    """an 11-station problem with a hybrid cluster whose second chunk starts at t0 > 0"""
    b = small_problem(N=11, M=2, tilesz=7, seed=seed, nchunk=[1, 2], flag_frac=0.2, uvcut_frac=0.03)
    pr = b.pr
    if flags:   # one baseline flagged in every slot, one station with every row flagged
        pr.flag[(pr.sta1 == 2) & (pr.sta2 == 5)] = 1
        pr.flag[(pr.sta1 == 7) | (pr.sta2 == 7)] = 1
    rng = np.random.default_rng(seed)
    n8 = 8 * pr.N
    x = pr.jones_true[:n8] + 0.05 * rng.normal(0, 1, n8)
    e1, e2 = rng.normal(0, 0.1, n8), rng.normal(0, 0.1, n8)
    return b, x, e1, e2


def _assert_vec(got, want, scale, tol):
    err = np.abs(np.asarray(got) - want).reshape(-1, 8).max(axis=1)
    bound = tol * scale.reshape(-1, 8).max(axis=1)
    assert (err <= bound).all(), (err / np.maximum(bound, 1e-300)).max()


@needs_oracle
@pytest.mark.parametrize("flags", [False, True], ids=["plain", "flagged"])
def test_rtr_eval_reference_matches_oracle(flags):
    """the numpy restatement of the RTR evaluator against the oracle's per-row evaluators
    (orc_rtr_raw / _counts / _weights) on both chunks of a hybrid cluster, unit and Student's-t weights"""
    b, x, e1, _ = _rtr_case(flags, 82)
    pr = b.pr
    orc = orcdirac.Oracle(pr)
    n8 = 8 * pr.N
    for k, ck in ((0, 0), (1, 0), (1, 1)):
        t0, nt = orc.chunk_tiles(k, ck)
        y = pr.x[8 * t0 * pr.Nbase:8 * (t0 + nt) * pr.Nbase]
        xk = x + 0.01 * k
        xw = xk + 0.02 * np.random.default_rng(k).normal(0, 1, n8)
        cnt = orc.rtr_counts(t0, nt)
        for nu in (None, 2.0, 30.0):
            wt = None
            if nu is not None:
                s_orc, wt_orc = orc.rtr_weights(k, t0, nt, y, xw, nu)
                slw, wt, slw_scale = rtr_weights_ref(pr, k, t0, nt, xw, nu)
                assert abs(slw - s_orc) <= 1e-13 * slw_scale
                assert relerr(wt, np.where(wt_orc > 0, wt_orc, 0.0)) < 1e-14
            for eta in (None, e1):
                c_orc, v_orc = orc.rtr_raw(k, t0, nt, y, xk, eta=eta, wt=wt)
                r = rtr_eval_ref(pr, k, t0, nt, xk, eta=eta, wt=wt)
                assert abs(r["cost"] - c_orc) <= 1e-13 * r["cost_scale"]
                _assert_vec(r["vec"], v_orc, r["vec_scale"], 1e-13)
                assert np.array_equal(r["counts"], cnt)
        if flags:
            assert cnt[7] == 0 and cnt.min() == 0 and cnt.max() > 0


@pytest.mark.parametrize("weighted", [False, True], ids=["unit", "student-t"])
def test_rtr_eval_reference_is_the_derivative_of_the_cost(weighted):
    """calculus, no other code: d/dt cost(x + t eta) = -2 vec(x) . eta and d/dt vec(x + t eta) =
    hess(x, eta).  The cost is a quartic and vec a cubic in t: both are fitted exactly from 5 points."""
    b, x, e1, e2 = _rtr_case(True, 83)
    pr = b.pr
    k, t0, nt = 1, 4, 3
    wt = rtr_weights_ref(pr, k, t0, nt, x + 0.03, 5.0)[1] if weighted else None
    ts = np.array([-1.0, -0.5, 0.0, 0.5, 1.0])
    r0 = rtr_eval_ref(pr, k, t0, nt, x, wt=wt)
    for eta in (e1, e2):
        rs = [rtr_eval_ref(pr, k, t0, nt, x + t * eta, wt=wt) for t in ts]
        c = np.polyfit(ts, [r["cost"] for r in rs], 4)
        dcost = c[-2]
        assert abs(dcost - (-2.0 * np.dot(r0["vec"], eta))) <= 1e-12 * r0["cost_scale"]
        V = np.array([r["vec"] for r in rs])
        dvec = np.polyfit(ts, V, 4)[-2]
        h = rtr_eval_ref(pr, k, t0, nt, x, eta=eta, wt=wt)
        _assert_vec(dvec, h["vec"], h["vec_scale"], 1e-11)
        # a real error would be far above the bound
        assert np.abs(h["vec"]).max() > 1e-3 * h["vec_scale"].max()


@needs_oracle
@pytest.mark.parametrize("data,nu0", [("outliers", 2.0), ("outliers", 7.6), ("clean", 30.0)])
def test_irls_reference_matches_oracle(data, nu0):
    """util.irls_ref against orc_update_w_and_nu (pinned to the compiled reference's update_w_and_nu
    by test_oracle_vs_ref.py): the same nu and weights; with non-unit incoming weights the new ones
    are scaled by lambda / ndata"""
    rng = np.random.default_rng(17)
    e = rng.normal(0, 0.5, 8 * 3000)
    if data == "outliers":
        hit = rng.random(e.size) < 0.02
        e[hit] += rng.normal(0, 5.0, hit.sum())
    orc = orcdirac.Oracle(small_problem().pr)
    nu_o, w_o = orc.update_w_and_nu(nu0, e)
    r = irls_ref(e, np.ones_like(e), nu0)
    assert r["margin"] > 1e-9
    assert r["nu"] == nu_o
    assert r["lam"] == e.size
    assert relerr(r["w"], w_o) < 1e-15
    wt_old = rng.uniform(0.2, 1.3, e.size)
    r2 = irls_ref(e, wt_old, nu0)
    assert r2["nu"] == nu_o
    assert abs(r2["lam"] - np.abs(wt_old).sum()) <= 1e-13 * r2["lam"]
    assert relerr(r2["w"], w_o * (r2["lam"] / e.size)) < 1e-15
    # clean data sits at the top of the grid, 2 % outliers well below it
    assert (r["nu"] == 2.0 + 29 * (28.0 / 30)) == (data == "clean")


@needs_oracle
def test_sky_split_identity_on_the_oracle():
    """a cluster's coherencies are the sum of those of its sources split into three clusters of at
    most 96; an empty cluster has zero coherencies"""
    clusters = big_cluster_sky()
    big = clusters[5]                     # 200 sources
    parts = (96, 96, 8)
    rng = np.random.default_rng(1)
    R = 300
    u, v, w = (rng.normal(0, 3e4, R) / 3e8 for _ in range(3))
    whole = orcdirac.OracleSky(clusters).coherencies(u, v, w, 150e6, 2e5).reshape(R, -1, 4)
    split = orcdirac.OracleSky(split_cluster(big, parts)).coherencies(u, v, w, 150e6, 2e5)
    split = split.reshape(R, 3, 4)
    assert relerr(split.sum(axis=1), whole[:, 5]) < 1e-13
    assert not whole[:, 6].any()
    freqs = np.array([146e6, 152e6, 158e6])
    xa = orcdirac.OracleSky([big]).predict_multifreq(u, v, w, freqs, 6e5, 1, np.zeros(8 * R * 3))
    xb = orcdirac.OracleSky(split_cluster(big, parts)).predict_multifreq(u, v, w, freqs, 6e5, 1,
                                                                         np.zeros(8 * R * 3))
    assert relerr(xb, xa) < 1e-13


@needs_oracle
@pytest.mark.parametrize("M", [1, 2, 7, 65, 100])
def test_mult_hessian_reference_matches_oracle(M):
    """util.mult_hessian_ref against orc_mult_hessian (the reference's mult_hessian restated in C) in
    every state the LBFGS driver produces: the partial histories (npairs, next) = (k, k), k < M, and
    the full history at every next slot; one pair with y . s < 0 (the reference keeps it)"""
    m = 37 if M > 7 else 53
    g, s, y, rho = lbfgs_pairs(m, M, seed=M, negative=M // 2)
    assert rho[M // 2] < 0
    states = [(k, k) for k in range(M)] + [(M, j) for j in range(M)]
    for npairs, nxt in states:
        want = orcdirac.mult_hessian(g, s, y, rho, npairs, nxt)
        got, scale = mult_hessian_ref(g, s, y, rho, npairs, nxt)
        if npairs == 0:
            assert np.array_equal(got, g) and np.array_equal(want, g)
            continue
        assert (np.abs(got - want) <= 1e-14 * scale).all(), (npairs, nxt,
                                                                np.max(np.abs(got - want) / scale))
        # the pairs matter: the answer is far from the scaled gradient of a memoryless step
        assert relerr(g * (s[0] @ y[0]) / (y[0] @ y[0]), got) > 1e-3
