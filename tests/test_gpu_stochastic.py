"""Stochastic calibration of a whole interval (sagecal -N <epochs> -M <minibatches> -w <bands>,
minibatch_mode.cpp:364-509, no beam): dirac_b200_stochastic_interval against the driver's loop restated
with the reference's precalculate_coherencies_multifreq, bfgsfit_minibatch_visibilities and
calculate_residuals_multifreq (flags freshly preset at every load), and against the same loop made of
this library's reference-named calls.

The tests that compare with the reference call it first and ask for the product library afterwards,
so that the reference's answers can be recorded on a machine without a GPU."""
import ctypes as C

import numpy as np
import pytest

from util import small_problem, relerr
from sagecal_b200 import synth
from sagecal_b200.dirac_api import SkyModel, make_barr

pytestmark = pytest.mark.gpu

NO_CCID = -99999
# two runs of the same LBFGS fit on the same device differ in the last bits (the gradient kernels sum
# with atomics), and a few iterations amplify that
RERUN_TOL = 1e-9
FREQS5 = np.array([142e6, 146e6, 150e6, 154e6, 158e6])
FREQS9 = np.linspace(140e6, 164e6, 9)
NMB, TMB = 2, 4              # minibatches of an interval, timeslots of a minibatch
LBFGS = dict(max_lbfgs=3, lbfgs_m=5, robust_nu=2.0)


class Interval:
    """one interval of NMB minibatches of TMB timeslots: u, v, w, preset flags and data per minibatch"""

    def __init__(self, pr, sky, freqs, ivl, seed):
        R = pr.Nbase * TMB
        rows = slice(ivl * NMB * R, (ivl + 1) * NMB * R)
        self.u = np.ascontiguousarray(pr.u[rows].reshape(NMB, R))
        self.v = np.ascontiguousarray(pr.v[rows].reshape(NMB, R))
        self.w = np.ascontiguousarray(pr.w[rows].reshape(NMB, R))
        self.sta1 = pr.sta1[rows].reshape(NMB, R)
        self.sta2 = pr.sta2[rows].reshape(NMB, R)
        self.flag = pr.flag[rows].reshape(NMB, R)
        rng = np.random.default_rng(seed)
        self.x = np.zeros((NMB, len(freqs), 8 * R))
        for mb in range(NMB):
            r = np.arange(ivl * NMB * R + mb * R, ivl * NMB * R + (mb + 1) * R)
            for ci, f in enumerate(freqs):
                coh = synth.coherencies(pr.u[r], pr.v[r], pr.w[r], pr.clusters, f, pr.fdelta)
                x = synth.apply_jones(coh, pr.jones_true, pr.sta1[r], pr.sta2[r], pr.N, pr.nchunk)
                sig = 1e-2 * np.median(np.abs(x))
                x = x + rng.normal(0, sig, x.shape)
                bad = rng.uniform(0, 1, x.shape) < 0.02
                x[bad] += rng.normal(0, 20 * sig, int(bad.sum()))
                x.reshape(R, 8)[self.flag[mb] != 0] = 0.0   # preset_flags_and_data
                self.x[mb, ci] = x
        self.R = R

    def barr(self, mb=None):
        """flags as preset_flags_and_data leaves them: one minibatch, or all of them back to back"""
        if mb is not None:
            return make_barr(self.sta1[mb], self.sta2[mb], self.flag[mb])
        return make_barr(self.sta1.reshape(-1), self.sta2.reshape(-1), self.flag.reshape(-1))


def problem(freqs):
    """9 stations, 3 clusters (hybrid chunks 1, 2, 1; the first with a negative id), 2 intervals of 2
    minibatches of 4 timeslots, 5 % flagged rows, 2 % outliers, one set of true Jones"""
    b = small_problem(N=9, M=3, tilesz=2 * NMB * TMB, seed=61, kmean=1.0, nchunk=[1, 2, 1],
                      flag_frac=0.05)
    pr = b.pr
    for k, cl in enumerate(pr.clusters):
        cl["id"] = (-1, 1, 2)[k]
    sky = SkyModel(pr.clusters, pr.N)
    assert (pr.flag != 0).any()
    return b, sky, [Interval(pr, sky, freqs, i, seed=70 + i) for i in range(2)]


def uv_cut(pr, freqs):
    """a uvmin that cuts about a fifth of the unflagged rows at the first channel"""
    uvd = np.sqrt(pr.u * pr.u + pr.v * pr.v)
    return float(np.quantile(uvd[pr.flag == 0], 0.2) * freqs[0])


def bands(nchan, nsolbw):
    """minibatch_mode.cpp:93-116"""
    per = (nchan + nsolbw - 1) // nsolbw
    out, count = [], 0
    for _ in range(nsolbw):
        n = per if count + per < nchan else nchan - count
        out.append((count, n))
        count += n
    return out


def driver_loop(lib, b, sky, ivl, freqs, nsolbw, nepochs, pts, pfreq, uvmin, ccid=NO_CCID, rho=1e-9,
                phase_only=0, **kw):
    """minibatch_mode.cpp:368-506 through the reference-named calls of `lib`; pfreq in/out.
    returns (residuals [NMB, Nchan, 8R], res_00, res_01 [nepochs, NMB, nsolbw])"""
    pr = b.pr
    nchan = len(freqs)
    deltaf = pr.fdelta * nchan
    bl = bands(nchan, nsolbw)
    r0 = np.zeros((nepochs, NMB, nsolbw))
    r1 = np.zeros((nepochs, NMB, nsolbw))
    coh_all = [None] * NMB
    R, M = ivl.R, sky.M
    for ep in range(nepochs):
        for mb in range(NMB):
            barr = ivl.barr(mb)
            if ep == 0:
                coh_all[mb] = lib.precalculate_coherencies_multifreq(
                    ivl.u[mb], ivl.v[mb], ivl.w[mb], pr.N, R, barr, sky, freqs, deltaf, uvmin=uvmin)
            for bi, (c0, nc) in enumerate(bl):
                coh = np.ascontiguousarray(coh_all[mb][c0 * R * M * 4:(c0 + nc) * R * M * 4])
                x = np.ascontiguousarray(ivl.x[mb, c0:c0 + nc]).reshape(-1)
                r0[ep, mb, bi], r1[ep, mb, bi] = lib.bfgsfit_minibatch(
                    ivl.u[mb], ivl.v[mb], ivl.w[mb], x, pr.N, pr.Nbase, TMB, barr, sky, coh, pfreq[bi],
                    freqs[c0:c0 + nc], pts[bi], fdelta=pr.fdelta * nc, nmb=mb, totalmb=NMB, **kw)
    res = ivl.x.copy()
    for mb in range(NMB):
        barr = ivl.barr(mb)
        for bi, (c0, nc) in enumerate(bl):
            xr = np.ascontiguousarray(res[mb, c0:c0 + nc])
            assert lib.calculate_residuals_multifreq(
                ivl.u[mb], ivl.v[mb], ivl.w[mb], pfreq[bi], xr.reshape(-1), pr.N, pr.Nbase, TMB, barr,
                sky, freqs[c0:c0 + nc], pr.fdelta * nc, ccid=ccid, rho=rho, phase_only=phase_only) == 0
            res[mb, c0:c0 + nc] = xr
    return res, r0, r1


def run_driver(lib, b, sky, ivls, freqs, nsolbw, nepochs, uvmin, **kw):
    """both intervals back to back, pt and pfreq carried over; one (res, r0, r1, pfreq) per interval"""
    m = b.m
    pts = [lib.persist_init(NMB, m, 8 * ivls[0].R, LBFGS["lbfgs_m"]) for _ in range(nsolbw)]
    pfreq = np.tile(b.pr.pp0, (nsolbw, 1))
    out = []
    for ivl in ivls:
        res, r0, r1 = driver_loop(lib, b, sky, ivl, freqs, nsolbw, nepochs, pts, pfreq, uvmin, **kw)
        out.append((res, r0, r1, pfreq.copy()))
    for pt in pts:
        lib.persist_clear(pt)
    return out


def run_interval(api, b, sky, ivls, freqs, nsolbw, nepochs, uvmin, ccid=NO_CCID, rho=1e-9,
                 phase_only=0, **kw):
    pr = b.pr
    pts = api.persist_init_array(nsolbw, NMB, b.m, 8 * ivls[0].R, kw.get("lbfgs_m", 5))
    pfreq = np.tile(pr.pp0, (nsolbw, 1))
    out = []
    for ivl in ivls:
        xo = ivl.x.copy()
        barr = ivl.barr()
        rv, r0, r1 = api.stochastic_interval(ivl.u, ivl.v, ivl.w, xo, pr.N, pr.Nbase, TMB, barr, sky,
                                             freqs, pr.fdelta * len(freqs), pts, pfreq, nsolbw,
                                             nepochs, uvmin=uvmin, ccid=ccid, rho=rho,
                                             phase_only=phase_only, **kw)
        assert rv == 0
        out.append((xo, r0, r1, pfreq.copy()))
    for b_ in range(nsolbw):
        api.lib.lbfgs_persist_clear(C.byref(pts[b_]))
    return out


def assert_close(got, want, tol_r0, tol_r1, tol_p, tol_x):
    for (xg, g0, g1, pg), (xw, w0, w1, pw) in zip(got, want):
        fin = np.isfinite(w0)
        assert np.array_equal(fin, np.isfinite(g0)) and np.array_equal(np.isfinite(w1), np.isfinite(g1))
        assert np.max(np.abs(g0[fin] - w0[fin]) / np.abs(w0[fin])) <= tol_r0
        assert np.max(np.abs(g1[fin] - w1[fin]) / np.abs(w1[fin])) <= tol_r1
        for bi in range(len(pw)):
            assert relerr(pg[bi], pw[bi]) <= tol_p, (bi, relerr(pg[bi], pw[bi]))
        assert np.max(np.abs(xg - xw)) <= tol_x * np.max(np.abs(xw)), np.max(np.abs(xg - xw))


CASES = [(NO_CCID, 0), (1, 0), (2, 1)]
CASE_IDS = ["plain", "correct-by-1", "hybrid-correct-by-2-phase-only"]


@pytest.mark.parametrize("ccid,phase_only", CASES, ids=CASE_IDS)
def test_interval_against_reference(ref, request, ccid, phase_only):
    """5 channels in bands of 3 and 2, 2 minibatches, 3 epochs, two intervals: every fit's costs, each
    band's Jones after each interval, the residuals with the correction"""
    b, sky, ivls = problem(FREQS5)
    uvmin = uv_cut(b.pr, FREQS5)
    kw = dict(ccid=ccid, rho=1e-9, phase_only=phase_only, **LBFGS)
    want = run_driver(ref, b, sky, ivls, FREQS5, 2, 3, uvmin, **kw)
    assert want[1][2][-1].mean() < 0.5 * want[0][1][0].mean()   # it calibrates
    assert relerr(want[1][3][0], want[1][3][1]) > 1e-4           # the bands' solutions differ
    api = request.getfixturevalue("api")
    got = run_interval(api, b, sky, ivls, FREQS5, 2, 3, uvmin, **kw)
    assert_close(got, want, 1e-9, 1e-7, 1e-6, 1e-6)


def test_uv_cut_holds_in_the_first_epoch_only(api):
    """the driver flags rows outside the uv cut in epoch 0 only; later loads re-preset the flags, so
    those rows are fitted again.  With the cut moved out of reach the first epoch changes, the later
    ones start from a different point, and the interval call follows the restated loop in both"""
    b, sky, ivls = problem(FREQS5)
    uvmin = uv_cut(b.pr, FREQS5)
    got = run_interval(api, b, sky, ivls[:1], FREQS5, 2, 2, uvmin, **LBFGS)
    nocut = run_interval(api, b, sky, ivls[:1], FREQS5, 2, 2, 0.0, **LBFGS)
    assert abs(got[0][1][0, 0, 0] - nocut[0][1][0, 0, 0]) > 1e-6 * nocut[0][1][0, 0, 0]
    want = run_driver(api, b, sky, ivls[:1], FREQS5, 2, 2, uvmin, **LBFGS)
    assert_close(got, want, RERUN_TOL, RERUN_TOL, RERUN_TOL, RERUN_TOL)


@pytest.mark.parametrize("ccid,phase_only", [CASES[1], CASES[2]], ids=CASE_IDS[1:])
def test_interval_equals_the_reference_named_loop(api, ccid, phase_only):
    """keeping the coherencies on the device changes nothing: the interval call and this library's
    own three calls agree as closely as two runs of one of them; the interval uploads the sky once
    and moves no coherencies"""
    b, sky, ivls = problem(FREQS5)
    uvmin = uv_cut(b.pr, FREQS5)
    kw = dict(ccid=ccid, rho=1e-9, phase_only=phase_only, **LBFGS)
    want = run_driver(api, b, sky, ivls, FREQS5, 2, 3, uvmin, **kw)
    api.transfer_stats(reset=True)
    got = run_interval(api, b, sky, ivls[:1], FREQS5, 2, 3, uvmin, **kw)
    assert api.transfer_stats(reset=True) == (1, 0)
    got = run_interval(api, b, sky, ivls, FREQS5, 2, 3, uvmin, **kw)
    assert_close(got, want, RERUN_TOL, RERUN_TOL, RERUN_TOL, RERUN_TOL)


def test_no_iterations_bit_identical_and_one_launch_per_cost(api):
    """max_lbfgs = 0: the residuals of the interval call are those of the reference-named loop to the
    bit.  Each fit then evaluates the cost twice and the gradient once; a band's cost is one
    k_stream_band launch whatever its channels, its gradient one more and one k_grad_tma_band"""
    b, sky, ivls = problem(FREQS5)
    uvmin = uv_cut(b.pr, FREQS5)
    kw = dict(LBFGS, max_lbfgs=0, ccid=1)
    want = run_driver(api, b, sky, ivls[:1], FREQS5, 2, 3, uvmin, **kw)
    k13, k14 = api.kernel_count(13), api.kernel_count(14)
    got = run_interval(api, b, sky, ivls[:1], FREQS5, 2, 3, uvmin, **kw)
    nfits = 3 * NMB * 2
    assert api.kernel_count(13) - k13 == 3 * nfits
    assert api.kernel_count(14) - k14 == nfits
    assert np.array_equal(got[0][0], want[0][0])
    assert np.array_equal(got[0][3], want[0][3])
    assert np.array_equal(got[0][3][0], b.pr.pp0)
    for k in (1, 2):
        assert relerr(got[0][k], want[0][k]) < 1e-13


def test_band_without_channels(ref, request):
    """9 channels in 4 bands: 3, 3, 3 and 0 channels (minibatch_mode.cpp:93-116).  The reference fits
    the empty band without touching its Jones, at costs 0 x 1/0 = NaN; the interval call does the same
    and matches the reference on the other bands"""
    b, sky, ivls = problem(FREQS9)
    uvmin = uv_cut(b.pr, FREQS9)
    kw = dict(ccid=1, **LBFGS)
    want = run_driver(ref, b, sky, ivls, FREQS9, 4, 2, uvmin, **kw)
    for res, r0, r1, pf in want:
        assert np.isnan(r0[:, :, 3]).all() and np.isnan(r1[:, :, 3]).all()
        assert np.isfinite(r0[:, :, :3]).all()
        assert np.array_equal(pf[3], b.pr.pp0)
    api = request.getfixturevalue("api")
    got = run_interval(api, b, sky, ivls, FREQS9, 4, 2, uvmin, **kw)
    assert_close(got, want, 1e-9, 1e-7, 1e-6, 1e-6)
    assert np.array_equal(got[1][3][3], b.pr.pp0)


def test_more_bands_than_channels_is_refused(api):
    """nsolbw > Nchan (the driver clamps it before sizing pfreq and pt): -1, no output touched"""
    b, sky, ivls = problem(FREQS5)
    pr = b.pr
    ivl = ivls[0]
    pts = api.persist_init_array(6, NMB, b.m, 8 * ivl.R, 5)
    pfreq = np.tile(pr.pp0, (6, 1)) + 0.25
    xo = ivl.x.copy()
    for nsolbw in (6, 0):
        rv, r0, r1 = api.stochastic_interval(ivl.u, ivl.v, ivl.w, xo, pr.N, pr.Nbase, TMB, ivl.barr(),
                                             sky, FREQS5, pr.fdelta * 5, pts, pfreq[:max(nsolbw, 1)],
                                             nsolbw, 2, **LBFGS)
        assert rv == -1
        assert not r0.any() and not r1.any()
    assert np.array_equal(xo, ivl.x)
    assert np.array_equal(pfreq, np.tile(pr.pp0, (6, 1)) + 0.25)
    for i in range(6):
        api.lib.lbfgs_persist_clear(C.byref(pts[i]))
