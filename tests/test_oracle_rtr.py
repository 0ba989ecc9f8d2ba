"""CPU: pins the RTR / RSD / NSD control flow (sagecal_b200/csrc/rtr_algo.h, the code the product
runs on the host) against the compiled reference's rtr_solve_nocuda, rtr_solve_nocuda_robust and
nsd_solve_nocuda_robust, with the oracle's plain O(rows) evaluators underneath
(oracle/rtr_harness.cpp).  Runs without a GPU."""
import numpy as np
import pytest

import orcdirac
from util import small_problem, perturbed_jones, relerr

CASES = [
    dict(N=8, M=2, tilesz=10, seed=61),
    dict(N=11, M=3, tilesz=6, seed=62, kmean=2.0, outliers=0.03),
    dict(N=9, M=2, tilesz=12, seed=63, nchunk=[3, 1], outliers=0.02),
]


@pytest.fixture(scope="module", autouse=True)
def _need_oracle():
    if not orcdirac.available() or not orcdirac.os.path.exists(orcdirac.RTR_PATH):
        pytest.skip("oracle/liboracle.so / librtr_harness.so not built")


@pytest.mark.parametrize("case", range(len(CASES)))
@pytest.mark.parametrize("kind", [4, 5, 6], ids=["rtr", "rtr-robust", "nsd"])
def test_rtr_chunk_matches_reference(ref, refser, case, kind):
    ref = ref if kind == 4 else refser  # robust kinds: serialised threads (race in the nu update)
    b = small_problem(**CASES[case])
    pr = b.pr
    orc = orcdirac.Oracle(pr)
    pp = perturbed_jones(pr, seed=9, amp=0.05)
    # residual of the full model, then the hidden data of each cluster in turn (lmfit.c:866-891)
    res = pr.x - orc.predict_full(pp)
    off = 0
    for k in range(pr.M):
        hidden = res + orc.predict_cluster(k, pp)
        for ck in range(pr.nchunk[k]):
            t0, nt = orc.chunk_tiles(k, ck)
            pblk = pp[off:off + 8 * pr.N].copy()
            off += 8 * pr.N
            if nt <= 0:
                continue
            xd = hidden[8 * t0 * pr.Nbase: 8 * (t0 + nt) * pr.Nbase]
            md = ref.me_data(pr.N, pr.Nbase, nt, b.barr, b.sky, pr.coh, clus=k, tileoff=t0,
                             robust_nu=3.0)
            ita, itb = (8, 13) if kind != 6 else (18, 0)
            pw, iw, nuw = ref.rtr(pblk, xd, md, pr.N, nt * pr.Nbase, kind, ita, itb)
            pg, ig, nug = orc.rtr_chunk(k, t0, nt, pblk, xd, kind, ita, itb, nu0=3.0)
            assert relerr(pg, pw) < 1e-9, (k, ck, relerr(pg, pw))
            if kind != 6:
                assert abs(ig[0] - iw[0]) <= 1e-10 * abs(iw[0])
            assert abs(ig[1] - iw[1]) <= 1e-9 * abs(iw[1])
            if kind != 4:
                assert nug == nuw
            # the same solve with the arithmetic of the product's kernels (per-baseline tensors,
            # sagecal_b200/csrc/rtr_math.cuh) run on the CPU
            pt, it, nut = orc.rtr_chunk(k, t0, nt, pblk, xd, kind, ita, itb, nu0=3.0, tensor=True)
            assert relerr(pt, pw) < 1e-8, (k, ck, relerr(pt, pw))
            assert abs(it[1] - iw[1]) <= 1e-8 * abs(iw[1])
            if kind != 4:
                assert nut == nuw


@pytest.mark.parametrize("mode", [4, 5, 6])
def test_sagefit_rtr_modes_match_reference(ref, refser, mode):
    ref = ref if mode == 4 else refser
    b = small_problem(N=10, M=3, tilesz=10, seed=64, outliers=0.02 if mode > 4 else 0.0,
                      nchunk=[1, 2, 1])
    pr = b.pr
    orc = orcdirac.Oracle(pr)
    kw = dict(max_emiter=3, max_iter=3, max_lbfgs=4, lbfgs_m=7, solver_mode=mode, randomize=0)
    xr, ppr = pr.x.copy(), pr.pp0.copy()
    rr = ref.sagefit_visibilities(pr.u, pr.v, pr.w, xr, pr.N, pr.Nbase, pr.tilesz, b.fresh_barr(),
                                  b.sky, pr.coh, ppr, **kw)
    xo, ppo = pr.x.copy(), pr.pp0.copy()
    ro = orc.sagefit(xo, ppo, **kw)
    assert ro[0] == rr[0]
    assert abs(ro[1] - rr[1]) < 1e-9
    assert abs(ro[2] - rr[2]) <= 1e-12 * rr[2]
    assert relerr(ppo, ppr) < 1e-6, relerr(ppo, ppr)
    assert abs(ro[3] - rr[3]) <= 1e-6 * rr[3]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_rtr_admm_chunk_matches_reference(refser, case):
    """rtr_solve_nocuda_robust_admm (the J-update of the reference's consensus calibration) per
    chunk: the control flow of rtr_algo.h with consensus terms on the per-row evaluators and on the
    per-baseline tensor arithmetic of the product's kernels"""
    b = small_problem(**CASES[case])
    pr = b.pr
    orc = orcdirac.Oracle(pr)
    rng = np.random.default_rng(4 + case)
    pp = perturbed_jones(pr, seed=9, amp=0.05)
    res = pr.x - orc.predict_full(pp)
    n8 = 8 * pr.N
    off = 0
    for k in range(pr.M):
        hidden = res + orc.predict_cluster(k, pp)
        for ck in range(pr.nchunk[k]):
            t0, nt = orc.chunk_tiles(k, ck)
            pblk = pp[off:off + n8].copy()
            off += n8
            if nt <= 0:
                continue
            Y = 0.3 * rng.normal(0, 1, n8)
            BZ = pblk + 0.05 * rng.normal(0, 1, n8)
            rho = float(rng.uniform(2.0, 40.0))
            xd = hidden[8 * t0 * pr.Nbase: 8 * (t0 + nt) * pr.Nbase]
            md = refser.me_data(pr.N, pr.Nbase, nt, b.barr, b.sky, pr.coh, clus=k, tileoff=t0,
                                robust_nu=3.0)
            pw, iw, nuw = refser.rtr_admm(pblk, Y, BZ, xd, md, pr.N, nt * pr.Nbase, 7, 12, rho)
            for tensor, tol in ((False, 1e-9), (True, 1e-8)):
                pg, ig, nug = orc.rtr_chunk(k, t0, nt, pblk, xd, 5, 7, 12, nu0=3.0, tensor=tensor,
                                            Y=Y, BZ=BZ, rho=rho)
                assert relerr(pg, pw) < tol, (k, ck, tensor, relerr(pg, pw))
                assert abs(ig[0] - iw[0]) <= 1e-9 * abs(iw[0])
                assert abs(ig[1] - iw[1]) <= 10 * tol * abs(iw[1])
                assert nug == nuw


EDGE = [
    ("one-slot", dict(N=8, M=2, tilesz=1, seed=65), 4),
    ("heavy-flags", dict(N=9, M=2, tilesz=6, seed=66, flag_frac=0.4, uvcut_frac=0.05), 5),
    ("heavy-flags-nsd", dict(N=9, M=2, tilesz=6, seed=67, flag_frac=0.4), 6),
    ("zero-budget", dict(N=8, M=2, tilesz=6, seed=68), 4),   # this_itermax = 0: 5 RSD + 10 RTR iterations
]


@pytest.mark.parametrize("name,prob,kind", EDGE, ids=[e[0] for e in EDGE])
def test_rtr_chunk_edge_cases(ref, refser, name, prob, kind):
    b = small_problem(**prob)
    pr = b.pr
    orc = orcdirac.Oracle(pr)
    lib = ref if kind == 4 else refser
    pp = perturbed_jones(pr, seed=2, amp=0.1)
    res = pr.x - orc.predict_full(pp)
    n8 = 8 * pr.N
    ita, itb = ((5, 10) if name == "zero-budget" else (7, 12)) if kind != 6 else (17, 0)
    for k in range(pr.M):
        hidden = res + orc.predict_cluster(k, pp)
        pblk = pp[k * n8:(k + 1) * n8].copy()
        md = lib.me_data(pr.N, pr.Nbase, pr.tilesz, b.barr, b.sky, pr.coh, clus=k, robust_nu=4.0)
        pw, iw, nuw = lib.rtr(pblk, hidden, md, pr.N, pr.Nbase1, kind, ita, itb)
        for tensor, tol in ((False, 1e-9), (True, 1e-7)):
            pg, ig, nug = orc.rtr_chunk(k, 0, pr.tilesz, pblk, hidden, kind, ita, itb, nu0=4.0,
                                        tensor=tensor)
            assert relerr(pg, pw) < tol, (name, k, tensor, relerr(pg, pw))
            assert abs(ig[1] - iw[1]) <= 100 * tol * abs(iw[1])
            if kind != 4:
                assert nug == nuw


@pytest.mark.parametrize("mode", [4, 5, 6])
def test_sagefit_rtr_modes_match_reference_at_reduced_c3(ref, refser, mode):
    """the whole SAGE call under the Riemannian solvers at the reduced C2/C3 shape of BASELINE.md 5.5
    (62 stations, 1891 baselines, 8 clusters, 10 timeslots, the benchmark's solver settings): the
    restatement with the product's control flow against the COMPILED REFERENCE, live (its RTR family is
    matrix free, so it runs in seconds here).  This is the pin behind tests/golden/full/C3rtr, C2rtr,
    C3nsd, which the restatement generated at the full 62-station shapes."""
    from sagecal_b200 import synth
    from util import Bound
    ref = ref if mode == 4 else refser
    b = Bound(synth.make_problem(N=62, M=8, tilesz=10, radius=40e3, kmean=2.0, seed=20260921 + 30 + mode,
                                 outliers=0.02 if mode > 4 else 0.0))
    pr = b.pr
    orc = orcdirac.Oracle(pr)
    kw = dict(max_emiter=3, max_iter=2, max_lbfgs=10, lbfgs_m=7, solver_mode=mode, randomize=0)
    xr, ppr = pr.x.copy(), pr.pp0.copy()
    rr = ref.sagefit_visibilities(pr.u, pr.v, pr.w, xr, pr.N, pr.Nbase, pr.tilesz, b.fresh_barr(),
                                  b.sky, pr.coh, ppr, Nt=8, **kw)
    xo, ppo = pr.x.copy(), pr.pp0.copy()
    ro = orc.sagefit(xo, ppo, **kw)
    assert ro[0] == rr[0]
    assert abs(ro[1] - rr[1]) < 1e-9
    assert abs(ro[2] - rr[2]) <= 1e-12 * rr[2]
    assert relerr(ppo, ppr) < 1e-6, relerr(ppo, ppr)
    assert abs(ro[3] - rr[3]) <= 1e-6 * rr[3]
    assert relerr(xo, xr) < 1e-6


# (data noise relative to the median visibility, distance of the start from the true Jones, bound on
# max |Jones(tensor) - Jones(per-row)|).  Measured on seeds 91-93: 6.7e-16, 1.4e-13, 5.9e-10, 5.6e-10
LOW_NOISE = [(1e-2, 1e-4, 1e-13), (1e-4, 1e-4, 1e-11), (1e-6, 1e-4, 1e-8), (0.0, 0.0, 1e-8)]


@pytest.mark.parametrize("noise,start,bound", LOW_NOISE, ids=["1e-2", "1e-4", "1e-6", "exact"])
@pytest.mark.parametrize("kind", [4, 6], ids=["rtr", "nsd"])
def test_rtr_tensor_drift_at_low_noise(kind, noise, start, bound):
    """The kernels' tensor form gives the cost as c0 - Re(...): it cancels when the model nearly fits
    the data.  The same solve on the kernels' arithmetic and on the per-row evaluators, from near the
    truth, as the data noise goes to zero: the Jones stay within `bound` of each other, and on
    noise-free data started at the truth the per-row solve does not move at all"""
    for seed in (91, 92, 93):
        b = small_problem(N=11, M=1, tilesz=8, seed=seed, noise_rel=noise)
        pr = b.pr
        orc = orcdirac.Oracle(pr)
        rng = np.random.default_rng(seed)
        p0 = pr.jones_true + start * rng.normal(0, 1, pr.jones_true.shape)
        ita, itb = (8, 13) if kind != 6 else (18, 0)
        pw, _, _ = orc.rtr_chunk(0, 0, pr.tilesz, p0, pr.x, kind, ita, itb, nu0=3.0)
        pt, _, _ = orc.rtr_chunk(0, 0, pr.tilesz, p0, pr.x, kind, ita, itb, nu0=3.0, tensor=True)
        assert np.max(np.abs(pt - pw)) < bound, (seed, np.max(np.abs(pt - pw)))
        if start == 0.0:
            assert np.max(np.abs(pw - p0)) < 1e-15
