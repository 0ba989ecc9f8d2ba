"""Per-channel refinement on the GPU (driver option -b 1, fullbatch_mode.cpp:453-499): the
single-channel residual calculate_residuals against the compiled reference (residual.c:314-674), and
dirac_b200_bfgsfit_channels, the whole channel loop of an interval on one resident problem, against
the same loop made of the reference's precalculate_coherencies, bfgsfit_visibilities and
calculate_residuals, and against this library's own three calls.

The tests that compare with the reference call it first and ask for the product library afterwards,
so that the reference's answers can be recorded on a machine without a GPU."""
import numpy as np
import pytest

from util import small_problem, relerr, perturbed_jones
from sagecal_b200 import synth
from sagecal_b200.dirac_api import SkyModel, barr_to_numpy

pytestmark = pytest.mark.gpu

NO_CCID = -99999
FREQS = np.array([146e6, 150e6, 154e6, 158e6])
JONES_TOL = 1e-5   # the bound of the bfgsfit parity test (test_gpu_solvers.py)
# two runs of the same LBFGS fit on the same device: the gradient kernels sum with atomics, so the
# iterates differ in the last bits from run to run and a few iterations amplify that (measured here:
# 7e-12 of the cost after 8 iterations)
RERUN_TOL = 1e-9


def _spectral(clusters, ids):
    for k, cl in enumerate(clusters):
        K = len(cl["ll"])
        cl["spec_idx"] = np.where(np.arange(K) % 2 == 0, -0.7, 0.0)
        cl["spec_idx1"] = np.full(K, 0.05)
        cl["spec_idx2"] = np.full(K, -0.01)
        cl["f0"] = np.full(K, 140e6)
        cl["id"] = ids[k]


def residual_problem(nchunk=None, ids=(-1, 1, 2)):
    """9 stations, 3 clusters (the first with a negative id), 6 timeslots, spectral indices, points,
    Gaussians, disks, rings and shapelets, 10 % flagged rows, one channel of data and perturbed Jones"""
    from test_gpu_kernels import _extended_sky
    b = small_problem(N=9, M=3, tilesz=6, seed=23, kmean=4.0, gaussian_frac=0.3, nchunk=nchunk,
                      flag_frac=0.1)
    pr = b.pr
    assert (pr.flag != 0).any()
    _spectral(pr.clusters, ids)
    sky = _extended_sky(pr)
    assert set(int(t) for cl in pr.clusters for t in cl["stype"]) >= {0, 1, 2, 3, 4}
    x0 = np.random.default_rng(4).normal(0, 1, 8 * pr.Nbase1)
    return b, sky, x0, perturbed_jones(pr, amp=0.2)


def residual(lib, b, sky, x0, pp, freq=FREQS[1], **kw):
    pr = b.pr
    x = x0.copy()
    assert lib.calculate_residuals(pr.u, pr.v, pr.w, pp.copy(), x, pr.N, pr.Nbase, pr.tilesz,
                                   b.fresh_barr(), sky, freq, pr.fdelta, **kw) == 0
    return x


# (nchunk, cluster ids, ccid, rho)
RES_CASES = [(None, (-1, 1, 2), NO_CCID, 1e-9), (None, (-1, 1, 2), 1, 1e-9),
             (None, (-1, 1, 2), -1, 1e-9), ([1, 4, 5], (-1, 1, 2), 2, 1e-9),
             ([2, 1, 4], (-1, 2, 2), 2, 1e-9), (None, (-1, 1, 2), 1, 0.5)]
RES_IDS = ["no-correction", "correct-by-1", "correct-by-negative-id", "hybrid-correct-by-2",
           "shared-ccid-last-wins", "large-rho"]


@pytest.mark.parametrize("nchunk,ids,ccid,rho", RES_CASES, ids=RES_IDS)
def test_calculate_residuals_against_reference(ref, request, nchunk, ids, ccid, rho):
    """hybrid chunk counts 4 and 5 do not divide the 6 timeslots: the chunk of a row comes from the
    row index (residual.c:350)"""
    b, sky, x0, pp = residual_problem(nchunk, ids)
    want = residual(ref, b, sky, x0, pp, ccid=ccid, rho=rho)
    assert relerr(want, x0) > 1e-3
    api = request.getfixturevalue("api")
    got = residual(api, b, sky, x0, pp, ccid=ccid, rho=rho)
    assert relerr(got, want) < 1e-11, relerr(got, want)
    if ccid != NO_CCID:   # the correction, and which cluster and rho it takes, are visible
        plain = residual(api, b, sky, x0, pp)
        assert relerr(got, plain) > 1e-3
        if rho > 1e-3:
            assert relerr(got, residual(api, b, sky, x0, pp, ccid=ccid, rho=1e-9)) > 1e-3
        if len(set(ids)) < len(ids):   # not the first cluster carrying the id
            first = ids.index(ccid)
            other = list(ids)
            other[first + 1:] = [77] * (len(ids) - first - 1)
            b2, sky2, _, _ = residual_problem(nchunk, tuple(other))
            assert relerr(got, residual(api, b2, sky2, x0, pp, ccid=ccid, rho=rho)) > 1e-3


@pytest.mark.parametrize("nchunk,ccid", [(None, NO_CCID), ([1, 4, 5], 2)], ids=["plain", "hybrid-corrected"])
def test_calculate_residuals_is_the_one_channel_multifreq_residual(api, nchunk, ccid):
    """one code path: the same bits as calculate_residuals_multifreq with one channel, phase_only 0"""
    b, sky, x0, pp = residual_problem(nchunk)
    pr = b.pr
    got = residual(api, b, sky, x0, pp, ccid=ccid, rho=1e-6)
    xm = x0.copy()
    assert api.calculate_residuals_multifreq(pr.u, pr.v, pr.w, pp.copy(), xm, pr.N, pr.Nbase, pr.tilesz,
                                             b.fresh_barr(), sky, FREQS[1:2], pr.fdelta, ccid=ccid,
                                             rho=1e-6, phase_only=0) == 0
    assert np.array_equal(got, xm)
    assert relerr(got, x0) > 1e-3


# ---- the channel loop ---------------------------------------------------------------------------------

def channel_problem(nchunk=None, outliers=0.0, freqs=FREQS, seed=41):
    """9 stations, 3 clusters (the first with a negative id), 8 timeslots, points and Gaussians with
    spectral indices; per channel the data of the true Jones on the channel's coherencies plus noise.
    The fit starts from unit Jones."""
    b = small_problem(N=9, M=3, tilesz=8, seed=seed, kmean=1.0, gaussian_frac=0.3, nchunk=nchunk,
                      flag_frac=0.05)
    pr = b.pr
    _spectral(pr.clusters, (-1, 1, 2))
    sky = SkyModel(pr.clusters, pr.N)
    rng = np.random.default_rng(seed + 1)
    xo = np.zeros((len(freqs), 8 * pr.Nbase1))
    for ci, f in enumerate(freqs):
        coh = synth.coherencies(pr.u, pr.v, pr.w, pr.clusters, f, pr.fdelta)
        x = synth.apply_jones(coh, pr.jones_true, pr.sta1, pr.sta2, pr.N, pr.nchunk)
        sigma = 1e-2 * np.median(np.abs(x))
        noise = rng.normal(0, sigma, x.shape)
        if outliers > 0:
            bad = rng.uniform(0, 1, x.shape) < outliers
            noise[bad] += 20.0 * sigma * rng.choice([-1.0, 1.0], size=int(bad.sum()))
        x = x + noise
        x.reshape(pr.Nbase1, 8)[pr.flag == 1] = 0.0
        xo[ci] = x
    return b, sky, xo


def loop_of_three(lib, b, sky, xo, freqs, p0, uvmin=0.0, uvmax=1e9, max_lbfgs=8, lbfgs_m=5,
                  solver_mode=1, mean_nu=2.0, ccid=NO_CCID, rho=1e-9):
    """fullbatch_mode.cpp:464-497 literally, through the three reference-named calls of `lib`.
    returns dict(xo, res_00, res_01, pfreq, p, flag)"""
    pr = b.pr
    barr = b.fresh_barr()
    xo = xo.copy()
    n = len(freqs)
    r0, r1, pfreq = np.zeros(n), np.zeros(n), np.zeros((n, len(p0)))
    for ci in range(n):
        pf = p0.copy()
        xf = xo[ci].copy()
        coh = lib.precalculate_coherencies(pr.u, pr.v, pr.w, pr.N, pr.Nbase1, barr, sky, freqs[ci],
                                           pr.fdelta, uvmin=uvmin, uvmax=uvmax)
        _, r0[ci], r1[ci] = lib.bfgsfit_visibilities(pr.u, pr.v, pr.w, xf, pr.N, pr.Nbase, pr.tilesz,
                                                     barr, sky, coh, pf, freq0=freqs[ci],
                                                     fdelta=pr.fdelta, max_lbfgs=max_lbfgs,
                                                     lbfgs_m=lbfgs_m, solver_mode=solver_mode,
                                                     mean_nu=mean_nu)
        assert lib.calculate_residuals(pr.u, pr.v, pr.w, pf, xo[ci], pr.N, pr.Nbase, pr.tilesz, barr,
                                       sky, freqs[ci], pr.fdelta, ccid=ccid, rho=rho) == 0
        pfreq[ci] = pf
    return dict(xo=xo, res_00=r0, res_01=r1, pfreq=pfreq, p=pfreq[-1].copy(),
                flag=barr_to_numpy(barr, pr.Nbase1)[2])


def resident(api, b, sky, xo, freqs, p0, keep_pfreq=True, **kw):
    pr = b.pr
    barr = b.fresh_barr()
    xo = xo.copy()
    p = p0.copy()
    rv, r0, r1, pfreq = api.bfgsfit_channels(pr.u, pr.v, pr.w, xo.reshape(-1), pr.N, pr.Nbase,
                                             pr.tilesz, barr, sky, freqs, pr.fdelta, p,
                                             keep_pfreq=keep_pfreq, **kw)
    assert rv == 0
    return dict(xo=xo, res_00=r0, res_01=r1, pfreq=pfreq, p=p, flag=barr_to_numpy(barr, pr.Nbase1)[2])


def assert_same_loop(got, want, xo, tol_jones, tol_res0, tol_res1, tol_x):
    assert np.array_equal(got["flag"], want["flag"])
    assert np.max(np.abs(got["res_00"] - want["res_00"]) / want["res_00"]) <= tol_res0
    assert np.max(np.abs(got["res_01"] - want["res_01"]) / want["res_01"]) <= tol_res1
    for ci in range(len(xo)):
        assert relerr(got["pfreq"][ci], want["pfreq"][ci]) <= tol_jones, ci
        scale = max(1.0, np.max(np.abs(xo[ci])) / np.max(np.abs(want["xo"][ci])))
        assert relerr(got["xo"][ci], want["xo"][ci]) <= tol_x * scale, ci
    assert relerr(got["p"], want["p"]) <= tol_jones
    assert np.array_equal(got["p"], got["pfreq"][-1])


LOOP_CASES = [(1, 2.0, None), (1, 2.0, [1, 3, 2]), (2, 4.0, None), (2, 4.0, [2, 1, 3])]
LOOP_IDS = ["gauss", "gauss-hybrid", "robust", "robust-hybrid"]


@pytest.mark.parametrize("mode,nu,nchunk", LOOP_CASES, ids=LOOP_IDS)
def test_resident_loop_against_reference(ref, request, mode, nu, nchunk):
    """4 channels, corrected by cluster 1: residuals, costs, every channel's Jones, the returned p"""
    b, sky, xo = channel_problem(nchunk, outliers=0.02 if mode == 2 else 0.0)
    p0 = b.pr.pp0
    kw = dict(solver_mode=mode, mean_nu=nu, ccid=1, rho=1e-9)
    want = loop_of_three(ref, b, sky, xo, FREQS, p0, **kw)
    assert (want["res_01"] < want["res_00"]).all()
    assert relerr(want["pfreq"][0], want["pfreq"][-1]) > 1e-4   # the channels' solutions differ
    api = request.getfixturevalue("api")
    got = resident(api, b, sky, xo, FREQS, p0, max_lbfgs=8, lbfgs_m=5, **kw)
    assert_same_loop(got, want, xo, JONES_TOL, 1e-10, 1e-5, 1e-5)


@pytest.mark.parametrize("mode,nu,nchunk", [LOOP_CASES[1], LOOP_CASES[3]],
                         ids=[LOOP_IDS[1], LOOP_IDS[3]])
def test_resident_loop_equals_the_three_calls(api, mode, nu, nchunk):
    """keeping the coherencies on the device changes nothing: the resident call and this library's
    precalculate_coherencies, bfgsfit_visibilities, calculate_residuals per channel agree as closely as
    two runs of one of them do (RERUN_TOL; the costs before the fit, which no atomics touch, to 1e-14);
    and the resident call uploads the sky once and moves no coherencies, where the three calls upload
    it twice per channel and move every channel's coherencies down and up again"""
    b, sky, xo = channel_problem(nchunk, outliers=0.02 if mode == 2 else 0.0)
    pr = b.pr
    kw = dict(solver_mode=mode, mean_nu=nu, ccid=2, rho=1e-9, uvmin=20.0, uvmax=4e3)
    api.transfer_stats(reset=True)
    want = loop_of_three(api, b, sky, xo, FREQS, pr.pp0, **kw)
    assert api.transfer_stats(reset=True) == (2 * len(FREQS), 2 * len(FREQS) * pr.Nbase1 * pr.M * 64)
    got = resident(api, b, sky, xo, FREQS, pr.pp0, max_lbfgs=8, lbfgs_m=5, **kw)
    assert api.transfer_stats(reset=True) == (1, 0)
    assert_same_loop(got, want, xo, RERUN_TOL, 1e-14, RERUN_TOL, RERUN_TOL)


def test_uv_cut_accumulates_over_the_channels(ref, request):
    """precalculate_coherencies flags unflagged rows outside [uvmin, uvmax] wavelengths AT THE CHANNEL
    and never clears a flag (predict.c:489-495), and the driver hands one barr to every channel: the
    first channel cuts short rows that the last would keep, the last cuts long rows that the first
    kept, and every channel's fit sees the flags of the channels before it"""
    freqs = np.array([120e6, 140e6, 160e6, 180e6])
    b, sky, xo = channel_problem([1, 2, 1], freqs=freqs, seed=43)
    pr = b.pr
    uvd = np.sqrt(pr.u * pr.u + pr.v * pr.v)
    free = pr.flag == 0
    uvmin = np.quantile(uvd[free], 0.15) * freqs[0]
    uvmax = np.quantile(uvd[free], 0.85) * freqs[-1]
    cut = lambda f: free & ((uvd * f < uvmin) | (uvd * f > uvmax))
    first, last = cut(freqs[0]), cut(freqs[-1])
    assert (first & ~last).sum() >= 5 and (last & ~first).sum() >= 5
    kw = dict(uvmin=uvmin, uvmax=uvmax, solver_mode=1, ccid=NO_CCID)
    want = loop_of_three(ref, b, sky, xo, freqs, pr.pp0, **kw)
    expect = pr.flag.copy()
    for f in freqs:
        expect[cut(f)] = 2
    assert np.array_equal(want["flag"], expect)
    api = request.getfixturevalue("api")
    got = resident(api, b, sky, xo, freqs, pr.pp0, max_lbfgs=8, lbfgs_m=5, **kw)
    assert_same_loop(got, want, xo, JONES_TOL, 1e-10, 1e-5, 1e-5)
    # the accumulated flags matter to the fit: the last channel on its own cut solves differently
    alone = resident(api, b, sky, xo[-1:], freqs[-1:], pr.pp0, max_lbfgs=8, lbfgs_m=5, **kw)
    assert not np.array_equal(alone["flag"], got["flag"])
    assert relerr(alone["p"], got["p"]) > 1e-7


def test_no_iterations_one_channel_and_no_jones_out(api):
    b, sky, xo = channel_problem([1, 3, 2])
    pr = b.pr
    p0 = perturbed_jones(pr, amp=0.05)
    # max_lbfgs = 0: the residual with the start Jones
    got = resident(api, b, sky, xo, FREQS, p0, max_lbfgs=0, ccid=1)
    assert np.array_equal(got["res_01"], got["res_00"])
    assert np.array_equal(got["p"], p0)
    for ci, f in enumerate(FREQS):
        assert np.array_equal(got["xo"][ci], residual(api, b, sky, xo[ci], p0, freq=f, ccid=1))
    # one channel is the first channel of four
    full = resident(api, b, sky, xo, FREQS, p0, max_lbfgs=6, lbfgs_m=5, ccid=1)
    one = resident(api, b, sky, xo[:1], FREQS[:1], p0, max_lbfgs=6, lbfgs_m=5, ccid=1)
    assert relerr(one["xo"][0], full["xo"][0]) < RERUN_TOL
    assert relerr(one["p"], full["pfreq"][0]) < RERUN_TOL
    assert one["res_00"][0] == full["res_00"][0]
    assert abs(one["res_01"][0] - full["res_01"][0]) < RERUN_TOL * full["res_01"][0]
    assert full["res_01"][0] < full["res_00"][0]
    # without the per-channel Jones the rest is the same
    bare = resident(api, b, sky, xo, FREQS, p0, keep_pfreq=False, max_lbfgs=6, lbfgs_m=5, ccid=1)
    assert bare["pfreq"] is None
    assert np.array_equal(bare["flag"], full["flag"]) and np.array_equal(bare["res_00"], full["res_00"])
    for k in ("xo", "res_01", "p"):
        assert relerr(bare[k], full[k]) < RERUN_TOL, k
