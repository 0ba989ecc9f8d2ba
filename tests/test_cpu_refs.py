"""CPU: the plain references the GPU tests of the line model, the RTR evaluator, the IRLS update, the
LBFGS two-loop recursion, the segmented sky staging, the minibatch band passes, the LM cluster
passes and the full-interval passes lean on, pinned
against the restatement (oracle/liboracle.so) or the compiled reference's recorded answers before a GPU
is involved."""
import numpy as np
import pytest

import orcdirac
from util import (BAND_CASES, BAND_FAULTS, CP_FAULTS, CP_RUNS, INTERVAL_FAULTS, U64, band_case,
                  band_consensus, band_ref, big_cluster_sky, chunk_offset, chunk_tiles, cluster_case,
                  cluster_pass_ref, cp_ref_args, cp_run_applies, interval_case, interval_ref,
                  cluster_rowmap_ref, irls_ref, lbfgs_pairs, line_model_ref, maps_agree,
                  mult_hessian_ref, relerr, rtr_eval_ref, rtr_weights_ref, small_problem,
                  split_cluster)

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


# ---- the minibatch band passes: util.band_ref pinned to the compiled reference ----------------------
def _band_ref_inputs(case):
    from sagecal_b200.dirac_api import SkyModel, make_barr
    pr = case["pr"]
    return make_barr(pr.sta1, pr.sta2, pr.flag), SkyModel(pr.clusters, pr.N)


def _ref_band_cost(ref, case, p, nu, cons):
    """bfgsfit_minibatch_visibilities / _consensus with max_lbfgs = 0: res_0 8 R Nf is
    robust_cost_func_multifreq at p"""
    pr = case["pr"]
    barr, sky = _band_ref_inputs(case)
    n = 8 * pr.Nbase1 * case["nc"]
    pt = ref.persist_init(1, case["m"], n, 5)
    Y, Z, rho = cons if cons is not None else (None, None, None)
    r0, _ = ref.bfgsfit_minibatch(pr.u, pr.v, pr.w, case["x"].reshape(-1).copy(), pr.N, pr.Nbase,
                                  pr.tilesz, barr, sky, case["coh"].reshape(-1).copy(), p.copy(),
                                  case["freqs"], pt, max_lbfgs=0, lbfgs_m=5, robust_nu=nu, Y=Y,
                                  Z=Z, rho=rho)
    ref.persist_clear(pt)
    return r0 * n


@pytest.mark.parametrize("consensus", [False, True], ids=["plain", "consensus"])
@pytest.mark.parametrize("nu", [2.0, 30.0])
@pytest.mark.parametrize("name", ["n2c3", "n9", "n33h4"])
def test_band_reference_matches_compiled_reference(ref, name, nu, consensus):
    """util.band_ref against the compiled reference on bands with non-zero data on flagged and uv-cut
    rows and hybrid clusters whose row and timeslot chunk maps disagree (n9, n33h4): the cost is
    robust_cost_func_multifreq (res_0 of a fit with no iterations), the gradient minus the sum over
    the channels of the single-channel Student's-t gradient (robust_grad_func, which
    test_gpu_kernels.py pins the full-batch kernel to)"""
    case = band_case(name)
    pr = case["pr"]
    cons = band_consensus(case) if consensus else None
    barr, sky = _band_ref_inputs(case)
    R, M = pr.Nbase1, case["M"]
    worst = 0.0
    for p in (case["A"], case["B"]):
        r = band_ref(case, p, nu, *(cons or ()))
        c_ref = _ref_band_cost(ref, case, p, nu, cons)
        # res_0 = f * (1/n) and back: two more roundings
        bound = r["cost_bound"] + 4 * U64 * abs(r["cost"])
        assert abs(c_ref - r["cost"]) <= bound, (c_ref, r["cost"], bound)
        worst = max(worst, abs(c_ref - r["cost"]) / bound)
        g = np.zeros(case["m"])
        for c in range(case["nc"]):
            md = ref.me_data(pr.N, pr.Nbase, pr.tilesz, barr, sky,
                             np.ascontiguousarray(case["coh"][c].reshape(-1)), robust_nu=nu)
            g -= ref.grad(p.copy(), np.ascontiguousarray(case["x"][c].reshape(-1)), md, robust=True)
        if cons is not None:
            y, z, rho = cons
            g += -y - np.repeat(rho, 8 * pr.N) * (p - z)
        err = np.abs(g - r["grad"])
        ratio = err / np.maximum(r["grad_bound"], 1e-300)
        assert (err <= r["grad_bound"]).all(), ratio.max()
        worst = max(worst, ratio.max())
        assert np.abs(r["grad"]).max() > 1e3 * r["grad_bound"].max()
    print("band_ref vs compiled reference (%s, nu %g): largest error / bound %.3g" % (name, nu, worst))


def _dcost(case, p, d, nu, h):
    """fourth-order central difference of band_ref's cost along d"""
    f = [band_ref(case, p + t * h * d, nu)["cost"] for t in (-2, -1, 1, 2)]
    return (f[0] - 8 * f[1] + 8 * f[2] - f[3]) / (12 * h)


@pytest.mark.parametrize("name", ["n33h3", "n9"])
def test_band_reference_gradient_is_minus_the_derivative_of_its_cost(name):
    """calculus, no other code: on a band whose hybrid chunks are the same under the cost's row map
    and the gradient's timeslot map (n33h3), d/dt cost(p + t d) = -grad . d along directions confined
    to each chunk block.  Where the maps disagree (n9: nchunk 2 over 5 timeslots), the reference's
    gradient is NOT the derivative of its cost, and neither is band_ref's: the rows of timeslot 2
    that the row map gives to chunk 1 count with chunk 0's Jones"""
    case = band_case(name)
    agree = maps_agree(case["tilesz"], case["Nbase"], case["nchunk"])
    assert agree == (name == "n33h3")
    N, nu = case["N"], 5.0
    rng = np.random.default_rng(3)
    p = case["B"]
    r = band_ref(case, p, nu)
    worst_off = 0.0
    for ci in range(case["Mt"]):
        d = np.zeros(case["m"])
        d[8 * N * ci:8 * N * (ci + 1)] = rng.normal(0, 1, 8 * N)
        fd = _dcost(case, p, d, nu, 1e-4)
        want = -np.dot(r["grad"], d)
        scale = np.dot(np.abs(r["grad"]) + r["grad_bound"], np.abs(d))
        off = abs(fd - want) / scale
        worst_off = max(worst_off, off)
        if agree:
            assert off < 1e-8, (ci, fd, want)
    if not agree:
        assert worst_off > 1e-3, worst_off


def test_band_cases_discriminate():
    """every deliberate fault of BAND_FAULTS, applied to band_ref, moves some quantity of some GPU case
    (test_gpu_band.py) past its bound by more than 10^3: the case set can see it"""
    names = [n for n in BAND_CASES if n != "n62"]   # the smaller cases already reach every fault
    cases = [band_case(n) for n in names]
    for fault in BAND_FAULTS:
        worst = 0.0
        for case in cases:
            for p in (case["A"], case["B"]):
                for nu in (2.0, 30.0):
                    good = band_ref(case, p, nu)
                    bad = band_ref(case, p, nu, fault=fault)
                    worst = max(worst,
                                abs(bad["cost"] - good["cost"]) / good["cost_bound"],
                                (np.abs(bad["res"] - good["res"]) / good["res_bound"]).max(),
                                (np.abs(bad["grad"] - good["grad"])
                                 / np.maximum(good["grad_bound"], 1e-300)).max())
        print("fault %s: largest error / bound %.3g" % (fault, worst))
        assert worst > 1e3, (fault, worst)


# ---- the LM cluster passes: util.cluster_pass_ref / cluster_rowmap_ref ----------------------------------
def _worst(err, bound):
    """largest err / bound (0 where both are 0)"""
    err = np.asarray(err, dtype=np.float64)
    return float(np.max(np.where(err == 0, 0.0, err / np.maximum(bound, 1e-300)), initial=0.0))


def test_cluster_pass_reference_matches_compiled_reference(ref):
    """on every (cluster, chunk) of a hybrid case whose chunks do not tile the interval evenly
    (n7h: nchunk [1, 2, 3] over 5 timeslots), with non-zero data on flag-1 and uv-cut rows, the
    restatement's model (x - the TRIAL output) is the reference's lm_func and its J^T e is lm_jac^T e
    with e = x - lm_func, within the stated bounds; its row-mapped add and subtract (sign +1 / -1,
    beta 1, r = dh = 0) are +- predict_cluster, the reference's row-mapped model of one cluster"""
    from sagecal_b200.dirac_api import SkyModel, make_barr
    case = cluster_case("n7h")
    pr = case["pr"]
    N, Nb = pr.N, pr.Nbase
    barr, sky = make_barr(pr.sta1, pr.sta2, pr.flag), SkyModel(pr.clusters, N)
    worst = dict(model=0.0, jte=0.0, rowmap=0.0)
    for k in range(case["M"]):
        for ck in range(case["nchunk"][k]):
            t0, t1 = chunk_tiles(case, k, ck)
            if t1 <= t0:
                continue
            off = chunk_offset(case, k, ck)
            pblk = case["P_old"][off:off + 8 * N].copy()
            r = cluster_pass_ref(case, k, ck, 1, case["x"], pblk, with_jte=True)
            md = ref.me_data(N, Nb, t1 - t0, barr, sky, pr.coh, clus=k, tileoff=t0)
            nn = 8 * (t1 - t0) * Nb
            sl = slice(8 * t0 * Nb, 8 * t1 * Nb)
            f = ref.lm_func(pblk, md, nn)
            J = ref.lm_jac(pblk, md, nn)
            assert not np.isnan(J).any()   # small enough to be recorded whole
            err = np.abs((case["x"][sl] - r["out"][sl]) - f)
            assert (err <= r["out_bound"][sl]).all(), (k, ck)
            worst["model"] = max(worst["model"], _worst(err, r["out_bound"][sl]))
            jte = J.T @ (case["x"][sl] - f)
            err = np.abs(jte - r["jte"])
            assert (err <= r["jte_bound"]).all(), (k, ck, _worst(err, r["jte_bound"]))
            worst["jte"] = max(worst["jte"], _worst(err, r["jte_bound"]))
            assert np.abs(r["jte"]).max() > 1e6 * r["jte_bound"].max()
    n = 8 * pr.Nbase1
    z = np.zeros(n)
    for k in range(case["M"]):
        md = ref.me_data(N, Nb, pr.tilesz, barr, sky, pr.coh, clus=k)
        f = ref.predict_cluster(case["P_old"].copy(), md, n)
        for sign in (1, -1):
            o, b = cluster_rowmap_ref(case, k, sign, 1.0, case["P_old"], z, z)
            err = np.abs(o - sign * f)
            assert (err <= b).all(), (k, sign)
            worst["rowmap"] = max(worst["rowmap"], _worst(err, b))
    print("cluster_pass_ref vs compiled reference: largest error / bound: model %.3g, J^T e %.3g, "
          "row map %.3g" % (worst["model"], worst["jte"], worst["rowmap"]))


@pytest.mark.parametrize("beta", [0.5, 0.125, 1.0 / 64])
def test_cluster_pass_reference_beta_identities(beta):
    """the sharded hidden-data weight has no counterpart in the reference: pinned by identity on the
    restatement itself.  d = INIT(beta, r, p_old) is beta r + f(p_old); the closing pass SUB(d, p,
    recover from p_old) is d - f(p) + (1-beta) r; the row-mapped add and subtract satisfy the same
    identities; with form_hidden, TRIAL and SUB on r equal TRIAL and SUB on the stored d"""
    case = cluster_case("n7h")
    N = case["N"]
    r = case["y"]
    worst = 0.0
    for k, ck in ((0, 0), (1, 1), (2, 1)):
        off = chunk_offset(case, k, ck)
        p, po = case["P"][off:off + 8 * N], case["P_old"][off:off + 8 * N]
        t0, t1 = chunk_tiles(case, k, ck)
        sl = slice(8 * t0 * case["Nbase"], 8 * t1 * case["Nbase"])
        d = cluster_pass_ref(case, k, ck, 0, r, po, beta=beta)
        f_old = r - cluster_pass_ref(case, k, ck, 1, r, po)["out"]      # f(p_old) on the chunk
        f_new = r - cluster_pass_ref(case, k, ck, 1, r, p)["out"]
        err = np.abs(d["out"][sl] - (beta * r + f_old)[sl])
        assert (err <= 2 * d["out_bound"][sl]).all()
        worst = max(worst, _worst(err, 2 * d["out_bound"][sl]))
        rec = cluster_pass_ref(case, k, ck, 3, d["out"], p, beta=beta, pblk_old=po)
        want = d["out"] - f_new + (1.0 - beta) * r
        bound = rec["out_bound"] + d["out_bound"] / beta
        err = np.abs(rec["out"][sl] - want[sl])
        assert (err <= bound[sl]).all(), _worst(err, bound[sl])
        worst = max(worst, _worst(err, bound[sl]))
        # the recovered residual is not the plain d - f(p): the (1-beta) r term is far above the bound
        assert np.abs(rec["out"][sl] - (d["out"] - f_new)[sl]).max() > 1e6 * bound[sl].max()
        # form_hidden on r is the pass on the stored hidden data (beta 1, as the visits use it)
        d1 = cluster_pass_ref(case, k, ck, 0, r, po)["out"]
        for mode in (1, 3):
            a = cluster_pass_ref(case, k, ck, mode, r, p, form_hidden=True, pblk_old=po)
            b = cluster_pass_ref(case, k, ck, mode, d1, p)
            err = np.abs(a["out"][sl] - b["out"][sl])
            assert (err <= a["out_bound"][sl] + b["out_bound"][sl]).all()
    pp = case["P"]
    for k in range(case["M"]):
        dh, bd = cluster_rowmap_ref(case, k, 1, beta, case["P_old"], r, np.zeros_like(r))
        m_old = cluster_rowmap_ref(case, k, 1, 1.0, case["P_old"], np.zeros_like(r), r)[0]
        assert (np.abs(dh - (beta * r + m_old)) <= bd).all()
        o, bo = cluster_rowmap_ref(case, k, -1, beta, pp, r, dh)
        m_new = cluster_rowmap_ref(case, k, 1, 1.0, pp, np.zeros_like(r), r)[0]
        err = np.abs(o - (dh - m_new + (1.0 - beta) * r))
        assert (err <= bo).all()
    print("beta %g: largest error / bound %.3g" % (beta, worst))


def _cp_runs(case):
    """(k, ck, name, run) of the cluster-pass checks of tests/test_gpu_cluster_pass.py on a case"""
    return [(k, ck, name, kw) for k in range(case["M"]) for ck in range(case["nchunk"][k])
            for name, kw in CP_RUNS if cp_run_applies(case, name, kw)]


def test_cluster_pass_cases_discriminate():
    """every deliberate fault of CP_FAULTS, applied to cluster_pass_ref, moves some quantity of some GPU
    case (test_gpu_cluster_pass.py) past its bound by more than 10^3: the cases can see it"""
    cases = [cluster_case(n) for n in ("n2", "n24", "n9e", "n9r")]
    for fault in CP_FAULTS:
        worst = 0.0
        for case in cases:
            for k, ck, name, kw in _cp_runs(case):
                a = cp_ref_args(case, k, ck, kw)
                good = cluster_pass_ref(case, k, ck, **a)
                bad = cluster_pass_ref(case, k, ck, fault=fault, **a)
                worst = max(worst, _worst(np.abs(bad["out"] - good["out"]), good["out_bound"]),
                            _worst(abs(bad["cost"] - good["cost"]), good["cost_bound"]),
                            _worst(np.abs(bad["jte"] - good["jte"]), good["jte_bound"]))
        print("fault %s: largest error / bound %.3g" % (fault, worst))
        assert worst > 1e3, (fault, worst)


# ---- the full-interval passes: util.interval_ref ----------------------------------------------------------
@pytest.mark.parametrize("nu", [None, 2.0, 30.0], ids=["gaussian", "nu2", "nu30"])
def test_interval_reference_matches_compiled_reference(ref, nu):
    """util.interval_ref against the compiled reference (minimize_viz_full_pth, cost_func /
    robust_cost_func, grad_func / robust_grad_func) and the oracle's restatement of them, on an
    interval with non-zero data on flag-1 and uv-cut rows and a hybrid cluster whose row and timeslot
    chunk maps disagree (n9: nchunk 2 over 5 timeslots), near and far from the truth"""
    from sagecal_b200.dirac_api import SkyModel, make_barr
    case = interval_case("n9")
    pr = case["pr"]
    assert not maps_agree(case["tilesz"], case["Nbase"], case["nchunk"])
    barr, sky = make_barr(pr.sta1, pr.sta2, pr.flag), SkyModel(pr.clusters, pr.N)
    md = ref.me_data(pr.N, pr.Nbase, pr.tilesz, barr, sky, pr.coh, robust_nu=2.0 if nu is None else nu)
    orc = orcdirac.Oracle(pr) if orcdirac.available() else None
    robust = nu is not None
    worst = dict(model=0.0, cost=0.0, grad=0.0)
    for s in ("A", "B"):
        p = case["points"][s]
        r = interval_ref(case, p, (nu,))
        q = r["passes"][nu]
        # the reference's cost is one more rounding away (the square of dnrm2, or the threads' sums)
        cost_bound = q["cost_bound"] + 4 * U64 * abs(q["cost"])
        want = [(ref.predict_full(p.copy(), md, 8 * pr.Nbase1), ref.cost(p.copy(), pr.x, md, robust),
                 ref.grad(p.copy(), pr.x, md, robust))]
        if orc is not None:
            want.append((orc.predict_full(p), orc.cost(p, pr.x, robust, 2.0 if nu is None else nu),
                         orc.grad(p, pr.x, robust, 2.0 if nu is None else nu)))
        for V, c, g in want:
            err = np.abs(V - r["model"])
            assert (err <= r["res_bound"]).all(), (s, _worst(err, r["res_bound"]))
            worst["model"] = max(worst["model"], _worst(err, r["res_bound"]))
            assert abs(c - q["cost"]) <= cost_bound, (s, c, q["cost"], cost_bound)
            worst["cost"] = max(worst["cost"], abs(c - q["cost"]) / cost_bound)
            err = np.abs(g - q["grad"])
            assert (err <= q["grad_bound"]).all(), (s, _worst(err, q["grad_bound"]))
            worst["grad"] = max(worst["grad"], _worst(err, q["grad_bound"]))
        # a real error would be far above the bound
        assert np.abs(q["grad"]).max() > 1e6 * q["grad_bound"].max()
    print("interval_ref vs compiled reference (nu %s): largest error / bound: model %.3g, cost %.3g, "
          "gradient %.3g" % (nu, worst["model"], worst["cost"], worst["grad"]))


@pytest.mark.parametrize("nu", [None, 5.0], ids=["gaussian", "student-t"])
def test_interval_reference_gradient_is_the_derivative_of_its_cost(nu):
    """calculus, no other code: on an interval whose hybrid chunks are the same under the model's row
    map and the gradient's timeslot map (n33h3), the fourth-order central difference of the cost along
    a direction confined to one chunk block is -grad . d for the Gaussian gradient (the reference's
    grad_func returns minus the true gradient) and +grad . d for the Student's-t one"""
    case = interval_case("n33h3")
    assert maps_agree(case["tilesz"], case["Nbase"], case["nchunk"])
    N = case["N"]
    rng = np.random.default_rng(4)
    p = case["points"]["B"]
    q = interval_ref(case, p, (nu,))["passes"][nu]
    sign = -1.0 if nu is None else 1.0
    h = 1e-4
    worst = 0.0
    for ci in range(case["Mt"]):
        d = np.zeros(case["m"])
        d[8 * N * ci:8 * N * (ci + 1)] = rng.normal(0, 1, 8 * N)
        f = [interval_ref(case, p + t * h * d, (nu,))["passes"][nu]["cost"] for t in (-2, -1, 1, 2)]
        fd = (f[0] - 8 * f[1] + 8 * f[2] - f[3]) / (12 * h)
        want = sign * np.dot(q["grad"], d)
        off = abs(fd - want) / np.dot(np.abs(q["grad"]) + q["grad_bound"], np.abs(d))
        worst = max(worst, off)
        assert off < 1e-7, (ci, fd, want)
    print("interval_ref gradient vs central differences (nu %s): largest relative deviation %.3g"
          % (nu, worst))


def test_interval_cases_discriminate():
    """every deliberate fault of INTERVAL_FAULTS, applied to interval_ref, moves some quantity of some
    GPU case (test_gpu_interval_passes.py) past its bound by more than 10^3: the cases can see it"""
    names = ["n2", "n9", "n33h3", "n33h4", "n40m1", "n40m2", "n40m4", "all-flagged"]
    nus = (None, 2.0, 30.0)
    runs = []
    for n in names:
        case = interval_case(n)
        for s in ("A", "B"):
            p = case["points"][s]
            runs.append((case, p, interval_ref(case, p, nus)))
    for fault in INTERVAL_FAULTS:
        worst = 0.0
        for case, p, good in runs:
            bad = interval_ref(case, p, nus, fault=fault)
            worst = max(worst, _worst(np.abs(bad["res"] - good["res"]), good["res_bound"]),
                        _worst(np.abs(bad["model"] - good["model"]), good["res_bound"]))
            for nu in nus:
                g, b = good["passes"][nu], bad["passes"][nu]
                worst = max(worst, _worst(abs(b["cost"] - g["cost"]), g["cost_bound"]),
                            _worst(np.abs(b["grad"] - g["grad"]), g["grad_bound"]))
        print("fault %s: largest error / bound %.3g" % (fault, worst))
        assert worst > 1e3, (fault, worst)
