"""The RTR evaluator kernels themselves (k_rtr_stats, k_rtr_reduce, k_rtr_eval through the production
RtrDevEval of rtr.cu, hook dirac_b200_rtr_eval) against the plain float64 per-row restatement
(util.rtr_eval_ref, pinned to the oracle and to calculus by tests/test_cpu_refs.py).

The solvers tolerate a slightly wrong cost, gradient, Hessian or weight: the trust region mostly
spends a few more tCG steps, and the end-to-end tests (test_gpu_rtr.py) compare solved Jones within
1e-5.  These tests read every evaluation directly: both Jones paths (parameter block up to 64
stations, device memory above, and forced at any N), the time-slice split including a ragged last
slice, flagged stations and baselines, unit and Student's-t weights, and evaluation sequences that
would expose a stale mailbox or a stale cached Jones vector."""
import numpy as np
import pytest

from sagecal_b200 import synth
from util import Bound, rtr_eval_ref, rtr_weights_ref

pytestmark = pytest.mark.gpu

TOL = 1e-12        # of the magnitude companion (DESIGN.md 5.3)
SLW_TOL = 1e-13


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _slicing(N, tilesz, nt):
    """(nslice, tslice) rtr.cu derives for a chunk of nt slots on this device"""
    nbb = (N * (N - 1) // 2 + 127) // 128
    ns = max(1, min((_sm_count() + nbb - 1) // nbb, tilesz))
    ns = min(ns, nt)
    ts = (nt + ns - 1) // ns
    return (nt + ts - 1) // ts, ts


# name: problem, cluster, chunk, row flags ("third": a third of the rows; "dead": one baseline in every
# slot and every row of one station), ragged (the last time slice is short)
CASES = [
    ("n2", dict(N=2, M=1, tilesz=5), 0, 0, None),
    ("n3-one-slot", dict(N=3, M=1, tilesz=1), 0, 0, None),
    ("n4", dict(N=4, M=1, tilesz=6), 0, 0, "dead"),
    ("n31-third", dict(N=31, M=1, tilesz=6), 0, 0, "third"),
    ("n32", dict(N=32, M=1, tilesz=5), 0, 0, "dead"),
    ("n33", dict(N=33, M=1, tilesz=8), 0, 0, None),
    ("n40-even", dict(N=40, M=1, tilesz=24), 0, 0, "dead"),
    ("n62-ragged", dict(N=62, M=1, tilesz=13), 0, 0, "dead"),
    ("n62-c3rtr", dict(N=62, M=1, tilesz=120), 0, 0, "third"),
    ("n62-hybrid-ragged", dict(N=62, M=2, tilesz=26, nchunk=[1, 2]), 1, 1, None),
    ("n64", dict(N=64, M=1, tilesz=4), 0, 0, "dead"),
    ("n65", dict(N=65, M=1, tilesz=3), 0, 0, "dead"),
    ("n70-hybrid", dict(N=70, M=2, tilesz=9, nchunk=[1, 2]), 1, 1, "third"),
    ("n100", dict(N=100, M=1, tilesz=3), 0, 0, None),
    ("n512", dict(N=512, M=1, tilesz=2), 0, 0, "dead"),
]
RAGGED = {"n62-ragged", "n62-c3rtr", "n62-hybrid-ragged"}


def _problem(name, prob, flags):
    seed = 900 + [c[0] for c in CASES].index(name)
    kw = dict(prob)
    if flags == "third":
        kw["flag_frac"] = 1.0 / 3.0
    pr = synth.make_problem(seed=seed, uvcut_frac=0.01, **kw)
    if flags == "dead":
        N = pr.N
        pr.flag[(pr.sta1 == 0) & (pr.sta2 == N - 1)] = 1
        pr.flag[(pr.sta1 == N // 2) | (pr.sta2 == N // 2)] = 1
    return Bound(pr), seed


def _chunk(pr, k, ck):
    nch = pr.nchunk[k]
    tc = (pr.tilesz + nch - 1) // nch
    t0 = min(ck * tc, pr.tilesz)
    return t0, min(t0 + tc, pr.tilesz) - t0


def _check_vec(got, ref, tol=TOL):
    err = np.abs(got - ref["vec"]).reshape(-1, 8).max(axis=1)
    bound = tol * ref["vec_scale"].reshape(-1, 8).max(axis=1)
    bad = err > bound
    assert not bad.any(), (np.flatnonzero(bad)[:8], (err / np.maximum(bound, 1e-300)).max())


def _sequence(x1, x2, e1, e2, alternate):
    """the evaluations of one condensation; `alternate`: a different x between the Hessian products,
    so that the cached device copy of x must be refreshed"""
    xa = x2 if alternate else x1
    a, b = 0.75, -1.5
    return [
        dict(x=x1, cost=True),                          # 0 cost only
        dict(x=x1, cost=True, vec=True),                # 1 cost and gradient
        dict(x=x1, eta=e1, vec=True),                   # 2 Hessian along e1
        dict(x=xa, cost=True, vec=True),                # 3 (another x above 64 stations)
        dict(x=x1, eta=e2, vec=True),                   # 4 Hessian along e2
        dict(x=x1, counts=True),                        # 5 counts (the evaluator's counts())
        dict(x=x2, cost=True, vec=True, counts=True),   # 6 all three from one launch
        dict(x=x1, eta=e1, vec=True),                   # 7 = 2, after counts and another x
        dict(x=x1, eta=a * e1 + b * e2, vec=True),      # 8 linearity
        dict(x=x1, cost=True, vec=True),                # 9 = 1
    ], (a, b)


def _check_sequence(pr, k, t0, nt, got, seq, ab, wt):
    R = got["results"]
    ref = {}

    def r(x, eta=None):
        key = (x.tobytes(), None if eta is None else eta.tobytes())
        if key not in ref:
            ref[key] = rtr_eval_ref(pr, k, t0, nt, x, eta=eta, wt=wt)
        return ref[key]

    for i, (ev, res) in enumerate(zip(seq, R)):
        want = r(ev["x"], ev.get("eta"))
        if ev.get("cost"):
            assert abs(res["cost"] - want["cost"]) <= TOL * want["cost_scale"], \
                (i, res["cost"], want["cost"], want["cost_scale"])
        if ev.get("vec"):
            _check_vec(res["vec"], want)
        if ev.get("counts"):
            assert np.array_equal(res["counts"], want["counts"]), i
    # bit-reproducible: no atomics in the kernels
    assert R[7]["vec"].tobytes() == R[2]["vec"].tobytes()
    assert R[9]["vec"].tobytes() == R[1]["vec"].tobytes() and R[9]["cost"] == R[1]["cost"]
    # the Hessian is symmetric and linear in eta (device values only; the companions give the scale)
    e1, e2 = seq[2]["eta"], seq[4]["eta"]
    h1, h2 = R[2]["vec"], R[4]["vec"]
    s1, s2 = r(seq[2]["x"], e1)["vec_scale"], r(seq[4]["x"], e2)["vec_scale"]
    sym_scale = np.dot(np.abs(e2), s1) + np.dot(np.abs(e1), s2)
    assert abs(np.dot(e2, h1) - np.dot(e1, h2)) <= TOL * sym_scale
    a, b = ab
    lin = dict(vec=a * h1 + b * h2, vec_scale=abs(a) * s1 + abs(b) * s2)
    _check_vec(R[8]["vec"], lin)
    return ref


# up to 64 stations both Jones paths: the parameter block and (forced) device memory
PARAMS = [c + (fd,) for c in CASES for fd in ((False, True) if c[1]["N"] <= 64 else (False,))]


@pytest.mark.parametrize("name,prob,k,ck,flags,force_device", PARAMS,
                         ids=[p[0] + ("-devmem" if p[-1] else "") for p in PARAMS])
def test_rtr_evaluator(api, name, prob, k, ck, flags, force_device):
    from sagecal_b200 import lib as blib
    b, seed = _problem(name, prob, flags)
    pr = b.pr
    N, n8 = pr.N, 8 * pr.N
    t0, nt = _chunk(pr, k, ck)
    if name == "n62-hybrid-ragged" or name == "n70-hybrid":
        assert t0 > 0
    blk = sum(pr.nchunk[:k]) + ck
    xt = pr.jones_true[blk * n8:(blk + 1) * n8]
    rng = np.random.default_rng(seed)
    x1 = xt + 1e-3 * rng.normal(0, 1, n8)            # near the solution: c0 - ... cancels
    x2 = xt + 0.1 * rng.normal(0, 1, n8)
    xw = xt + 0.05 * rng.normal(0, 1, n8)
    e1, e2 = rng.normal(0, 0.1, n8), rng.normal(0, 0.1, n8)
    seq, ab = _sequence(x1, x2, e1, e2, alternate=N > 64)
    inline = N <= 64 and not force_device
    ns_want, ts_want = _slicing(N, pr.tilesz, nt)
    if flags == "dead":
        assert rtr_eval_ref(pr, k, t0, nt, x1)["counts"][N // 2] == 0
    assert (pr.flag[t0 * pr.Nbase:(t0 + nt) * pr.Nbase] == 2).any() or nt * pr.Nbase < 200

    with blib.DeviceProblem(api, N, pr.Nbase, pr.tilesz, b.barr, b.sky, pr.coh, pr.x) as dp:
        # unit weights
        got = dp.rtr_eval(k, ck, seq, force_device=force_device)
        assert (got["nslice"], got["tslice"]) == (ns_want, ts_want)
        assert got["inline"] == inline
        if name in RAGGED:
            assert got["nslice"] > 1 and got["tslice"] > 1 and nt % got["tslice"] != 0, \
                (name, got["nslice"], got["tslice"], nt)
        assert got["slw"] == 0.0
        _check_sequence(pr, k, t0, nt, got, seq, ab, None)

        # Student's-t weights at xw != x, kept for the evaluations until unit_weights()
        for nu in (2.0, 30.0):
            slw, wt, slw_scale = rtr_weights_ref(pr, k, t0, nt, xw, nu)
            seq_u = seq + [dict(x=x1, cost=True, vec=True, unit=True),
                           dict(x=x1, eta=e1, vec=True)]
            got = dp.rtr_eval(k, ck, seq_u, xw=xw, nu=nu, keep=True, force_device=force_device)
            assert abs(got["slw"] - slw) <= SLW_TOL * slw_scale, (nu, got["slw"], slw)
            assert got["inline"] == inline
            _check_sequence(pr, k, t0, nt, got, seq, ab, wt)
            R = got["results"]
            u1, u2 = rtr_eval_ref(pr, k, t0, nt, x1), rtr_eval_ref(pr, k, t0, nt, x1, eta=e1)
            assert abs(R[10]["cost"] - u1["cost"]) <= TOL * u1["cost_scale"]
            _check_vec(R[10]["vec"], u1)
            _check_vec(R[11]["vec"], u2)

        # scalars only (the final nu of robust RTR): sum(log w - w) and the counts; tensors and c0 are
        # not rebuilt.  A later unit_weights() condenses the tensors again.
        slw, _, slw_scale = rtr_weights_ref(pr, k, t0, nt, xw, 5.0)
        got = dp.rtr_eval(k, ck, [dict(x=x1, counts=True), dict(x=x1, cost=True, vec=True, unit=True)],
                          xw=xw, nu=5.0, keep=False, force_device=force_device)
        assert abs(got["slw"] - slw) <= SLW_TOL * slw_scale
        u1 = rtr_eval_ref(pr, k, t0, nt, x1)
        assert np.array_equal(got["results"][0]["counts"], u1["counts"])
        assert abs(got["results"][1]["cost"] - u1["cost"]) <= TOL * u1["cost_scale"]
        _check_vec(got["results"][1]["vec"], u1)


def test_rtr_evaluator_slicing_covers_the_edges(api):
    """the cases above include, on this device: one slot, one slice, several even slices and a
    ragged last slice with more than one slot per slice; both Jones paths run (asserted per case)"""
    kinds = set()
    for name, prob, k, ck, _ in CASES:
        N, tilesz = prob["N"], prob["tilesz"]
        nch = (prob.get("nchunk") or [1] * prob["M"])[k]
        tc = (tilesz + nch - 1) // nch
        t0 = min(ck * tc, tilesz)
        nt = min(t0 + tc, tilesz) - t0
        ns, ts = _slicing(N, tilesz, nt)
        kinds.add("one-slot" if nt == 1 else "one-slice" if ns == 1 else
                  "ragged" if nt % ts else "even")
        if name in RAGGED:
            assert ns > 1 and ts > 1 and nt % ts, (name, ns, ts)
    assert kinds == {"one-slot", "one-slice", "even", "ragged"}, kinds
