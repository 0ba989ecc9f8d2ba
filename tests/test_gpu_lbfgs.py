"""The LBFGS iteration of lbfgs.cu / kernels_lbfgs.cu kernel by kernel and iteration by iteration:

* k_lbfgs_direction (the two-loop recursion in one 8-CTA cluster, hook dirac_b200_lbfgs_direction)
  against util.mult_hessian_ref, the reference's mult_hessian restated literally, in every history
  state the driver produces;
* k_lbfgs_step / k_lbfgs_update / k_lbfgs_nrm2 (hooks dirac_b200_lbfgs_step_update / _nrm2) against
  the arithmetic they stand for;
* whole LBFGS runs traced per iteration (dirac_b200_lbfgs_trace) against the restatement's trace
  (orc_lbfgs_traced): the same iterations, the same cost evaluations, the same history slots.

The end-to-end solver tests hold the Jones to 1e-5 after a few iterations: a wrong ring-buffer
rotation or a gamma from the wrong pair still gives a descent direction, and the line search still
finds some step.  These tests read the recursion and the iteration directly."""
import numpy as np
import pytest

import orcdirac
from bench import workload_shape
from sagecal_b200 import lib as blib
from util import (LBFGS_TRACE_CASES, LBFGS_TRACE_NU, lbfgs_pairs, lbfgs_start, lsum,
                  mult_hessian_ref, relerr, small_problem)

pytestmark = pytest.mark.gpu


def _bench_m(name, clusters_per_gpu=None):
    w = workload_shape(name)
    return 8 * w["N"] * (clusters_per_gpu or w["M"])


M_C2 = _bench_m("C2")                       # C2 and C3: 62 stations, 64 clusters
M_C4 = _bench_m("C4", clusters_per_gpu=32)  # C4 on 8 GPUs: 512 stations, 32 clusters per GPU
#: 1, 3: most of the 8 CTAs own an empty slice; 8, 9, 511, 4097: ragged slices
M_VALUES = [1, 3, 8, 9, 511, 4097, M_C2, M_C4]
assert M_C2 == 31744 and M_C4 == 131072

DIR_TOL = 1e-14     # of the magnitude companion; measured <= 5.6e-16 (m 4097, M 65)


def _states(M):
    """(npairs, next) as the driver produces them: partial histories, then the full one at every
    next slot"""
    return [(k, k) for k in range(M)] + [(M, j) for j in range(M)]


def _check_direction(api, g, s, y, rho, npairs, nxt):
    pk = api.lbfgs_direction(g, s, y, rho, npairs, nxt)
    assert pk is not None
    if npairs == 0:
        assert np.array_equal(pk, -g)
        return 0.0, pk
    want, scale = mult_hessian_ref(g, s, y, rho, npairs, nxt)
    err = float(np.max(np.abs(-pk - want) / scale))
    assert err <= DIR_TOL, (npairs, nxt, err)
    return err, pk


@pytest.mark.parametrize("m", M_VALUES)
def test_direction_benchmark_memory(api, m):
    """M = 7 (the benchmark's lbfgs_m) at every m; one stored pair has y . s < 0 (the reference keeps
    it in the recursion, so the kernel must too)"""
    M = 7
    g, s, y, rho = lbfgs_pairs(m, M, seed=m % 1000 + 1, negative=2 if m > 1 else None)
    worst = 0.0
    for npairs, nxt in _states(M):
        err, pk = _check_direction(api, g, s, y, rho, npairs, nxt)
        worst = max(worst, err)
        # deterministic: the same launch gives the same bits
        assert np.array_equal(api.lbfgs_direction(g, s, y, rho, npairs, nxt), pk)
    print("m=%d M=%d: max error %.3g of the companion" % (m, M, worst))


@pytest.mark.parametrize("m,M", [(9, 64), (511, 64), (511, 65), (4097, 65), (511, 100), (9, 7000)])
def test_direction_large_memory(api, m, M):
    """memory sizes at and past the 64 pairs k_lbfgs_direction once held in static shared memory;
    7000 pairs (56 KB of alpha_i) need the opt-in shared-memory size"""
    g, s, y, rho = lbfgs_pairs(m, M, seed=M + m, negative=M // 3)
    states = _states(M) if M <= 100 else [(M, 0), (M, 1), (M, M // 2), (M, M - 1), (M - 1, M - 1)]
    worst = 0.0
    for npairs, nxt in states:
        worst = max(worst, _check_direction(api, g, s, y, rho, npairs, nxt)[0])
    print("m=%d M=%d: max error %.3g of the companion" % (m, M, worst))


@pytest.mark.parametrize("m,M", [(9, 7), (4097, 7), (M_C2, 7), (511, 65)])
def test_direction_rotation_is_exact(api, m, M):
    """the pairs stored r slots further round the ring, with `next` moved by r, are the same history:
    the kernel does the same operations in the same order, so pk is bit-identical.  A slot-mapping
    error shows as a difference"""
    g, s, y, rho = lbfgs_pairs(m, M, seed=5, negative=1)
    for nxt in sorted({0, 1, M // 2, M - 1}):
        base = api.lbfgs_direction(g, s, y, rho, M, nxt)
        for r in sorted({1, 2, M - 1}):
            perm = (np.arange(M) + r) % M          # pair j now lives in slot (j + r) % M
            s2, y2, rho2 = np.empty_like(s), np.empty_like(y), np.empty_like(rho)
            s2[perm], y2[perm], rho2[perm] = s, y, rho
            got = api.lbfgs_direction(g, s2, y2, rho2, M, (nxt + r) % M)
            assert np.array_equal(got, base), (nxt, r)


def test_direction_refuses_what_it_cannot_hold(api):
    """the hook validates on the host and launches nothing it cannot hold"""
    g, s, y, rho = lbfgs_pairs(3, 4, seed=9)
    assert api.lbfgs_direction(g, s, y, rho, 5, 0) is None       # npairs > Mmem
    assert api.lbfgs_direction(g, s, y, rho, 4, 4) is None       # next >= Mmem
    big = 40000                                                  # 320 KB of alpha_i
    g1 = np.ones(1)
    s1 = np.ones((big, 1))
    assert api.lbfgs_direction(g1, s1, s1, np.ones(big), big, 0) is None


@pytest.mark.parametrize("m", M_VALUES)
def test_step_and_update(api, m):
    rng = np.random.default_rng(m)
    xk, pk = rng.normal(0, 1, m), rng.normal(0, 0.3, m)
    g0, g1 = rng.normal(0, 2, m), rng.normal(0, 1, m)
    Mmem, ci = 7, 4
    rho_in = rng.normal(0, 1, Mmem)
    alpha = 0.37
    r = api.lbfgs_step_update(alpha, xk, pk, g0, g1, rho_in, ci)
    # xk1 = xk + alpha pk to 1 ulp (one fma), beside the long double reference's own rounding of
    # alpha pk (64-bit mantissa) where x and alpha pk nearly cancel; sk and yk are the exact double
    # differences
    ap = np.longdouble(alpha) * pk.astype(np.longdouble)
    want = xk.astype(np.longdouble) + ap
    bound = np.spacing(np.abs(want.astype(np.float64))) + 2.0 ** -62 * np.abs(ap).astype(np.float64)
    assert (np.abs(r["xk1"] - want).astype(np.float64) <= bound).all()
    assert np.array_equal(r["sk"], r["xk1"] - xk)
    assert np.array_equal(r["yk"], g1 - g0)
    assert np.array_equal(r["xk"], r["xk1"])
    ys = lsum(r["yk"].astype(np.longdouble) * r["sk"])
    ys_scale = lsum(np.abs(r["yk"].astype(np.longdouble) * r["sk"]))
    assert abs(1.0 / r["rho"][ci] - ys) <= 1e-14 * ys_scale
    others = np.arange(Mmem) != ci
    assert np.array_equal(r["rho"][others], rho_in[others])
    gg = lsum(g1.astype(np.longdouble) * g1)
    assert abs(r["gg"] - gg) <= 1e-14 * gg
    assert abs(api.lbfgs_nrm2(g1) - gg) <= 1e-14 * gg


# -------------------------------------------------------------------------------------------------
# whole runs, iteration by iteration

TRACE_MARGIN = 1e3   # smallest line-search decision margin, in units of the costs' rounding noise
#: relative error bounds (alphak, ||g|| per iteration, iterates), measured on an H100:
#: Gaussian: alphak bit-identical, ||g|| <= 2.9e-8, iterates <= 6.7e-10.  The gradient after a step is
#: taken from the line residual E0 - a E1 - a^2 E2, which at the accepted a (up to 10) cancels to the
#: residual of nearly clean data: its rounding is a few 1e-10 of the iterate, not eps.
#: Student's t (outliers keep the residual large): alphak <= 3e-14, ||g|| <= 7.7e-11, iterates <= 1.4e-12.
#: robust-m80: 66 iterations amplify that rounding smoothly (the restatement and the compiled
#: reference differ by 3.1e-6 there too): ||g|| <= 2.8e-4, iterates <= 2.6e-6; its decisions, and so
#: every cost evaluation and slot, still agree exactly.
TRACE_TOL = {False: dict(alphak=1e-12, gnorm=1e-7, iterates=2e-9),
             True: dict(alphak=1e-12, gnorm=1e-9, iterates=1e-11),
             "robust-m80": dict(alphak=1e-12, gnorm=1e-3, iterates=1e-5)}


def run_trace(api, name):
    """(product trace, oracle trace) of one LBFGS_TRACE_CASES run"""
    _, prob, lbfgs_m, itmax, robust = next(c for c in LBFGS_TRACE_CASES if c[0] == name)
    b = small_problem(**prob)
    pr = b.pr
    p0 = lbfgs_start(pr, prob["seed"])
    want = orcdirac.Oracle(pr).lbfgs_trace(pr.x, p0, itmax, lbfgs_m, robust, LBFGS_TRACE_NU)
    with blib.DeviceProblem(api, pr.N, pr.Nbase, pr.tilesz, b.barr, b.sky, pr.coh, pr.x) as dp:
        got = dp.lbfgs_trace(p0, itmax, lbfgs_m, robust, LBFGS_TRACE_NU)
    return got, want, itmax, lbfgs_m, robust


def trace_errors(got, want):
    return dict(alphak=relerr(got["alphak"], want["alphak"]),
                gnorm=float(np.max(np.abs(got["gnorm"] - want["gnorm"]) / want["gnorm"])),
                iterates=max(relerr(a, b) for a, b in zip(got["iterates"], want["iterates"])))


@pytest.mark.parametrize("name", [c[0] for c in LBFGS_TRACE_CASES])
def test_trace_matches_restatement(api, name):
    got, want, itmax, lbfgs_m, robust = run_trace(api, name)
    err = trace_errors(got, want) if got["niter"] == want["niter"] else None
    print(name, got["niter"], want["niter"], "margin %.3g" % want["margin"], err)
    assert want["margin"] > TRACE_MARGIN, want["margin"]
    # the control flow: every iteration, every cost evaluation of its line search, every slot
    assert got["niter"] == want["niter"] == itmax
    assert np.array_equal(got["ncost"], want["ncost"])
    assert np.array_equal(got["slot"], want["slot"])
    assert np.array_equal(want["slot"], np.arange(itmax) % lbfgs_m)
    for k, tol in TRACE_TOL.get(name, TRACE_TOL[robust]).items():
        assert err[k] <= tol, (k, err[k])
    assert np.array_equal(got["p"], got["iterates"][-1])


def test_trace_refuses_what_it_cannot_hold(api):
    b = small_problem(N=8, M=2, tilesz=4, seed=3)
    pr = b.pr
    with blib.DeviceProblem(api, pr.N, pr.Nbase, pr.tilesz, b.barr, b.sky, pr.coh, pr.x) as dp:
        assert dp.lbfgs_trace(pr.pp0, 2, 1 << 20) is None


#: measured on an H100: Jones 1.6e-9 and 1.7e-9 in two runs, res_1 1.8e-10
SAGE_TOL = 1e-8


def test_sagefit_lbfgs_stage(api):
    """one sagefit with the benchmark's LBFGS settings (max_lbfgs 10, lbfgs_m 7): the history wraps in
    the LBFGS stage that ends the call.  Held tightly where the LM stage took no decision at rounding
    level in either library and the LBFGS stage's decisions are far above it"""
    b = small_problem(N=10, M=3, tilesz=8, seed=72, kmean=1.0)
    pr = b.pr
    kw = dict(max_emiter=2, max_iter=2, max_lbfgs=10, lbfgs_m=7, solver_mode=1)
    orc = orcdirac.Oracle(pr)
    orc.L.orc_noise_decisions(1)
    xo, ppo = pr.x.copy(), pr.pp0.copy()
    ro = orc.sagefit(xo, ppo, **kw)
    assert orc.L.orc_noise_decisions(0) == 0
    assert orc.L.orc_lbfgs_last_margin() > TRACE_MARGIN
    api.noise_decisions(reset=True)
    with blib.DeviceProblem(api, pr.N, pr.Nbase, pr.tilesz, b.barr, b.sky, pr.coh, pr.x) as dp:
        ppg = pr.pp0.copy()
        rg = dp.sagefit(ppg, **kw)
    assert api.noise_decisions() == 0
    assert rg[0] == ro[0]
    err = relerr(ppg, ppo)
    print("sagefit + LBFGS stage: Jones %.3g, res_1 %.3g" % (err, abs(rg[3] - ro[3]) / ro[3]))
    assert err <= SAGE_TOL
    assert abs(rg[3] - ro[3]) <= SAGE_TOL * ro[3]
