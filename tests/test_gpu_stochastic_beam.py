"""Stochastic calibration of a whole interval with station beams (sagecal -N -M -w -B <doBeam>, and with
-A): dirac_b200_stochastic_interval_withbeam and dirac_b200_stochastic_consensus_interval_withbeam
against the driver's loops (minibatch_mode.cpp:368-506, minibatch_consensus_mode.cpp:453-672 with their
beam branches) restated with the reference's calls, and against the same loops made of this library's
reference-named _withbeam calls.

The problem is the 9-station, 3-cluster, 2 x 4-timeslot one of test_gpu_stochastic.py with the sky and
stations of test_gpu_beam.py: sources a few degrees from the phase centre, one below the horizon,
per-station element positions, one JD per timeslot.  The element coefficient tables come from the
reference's set_elementcoeffs(_wb).

The reference's CPU precalculate_coherencies_multifreq_withbeam cannot serve as the pin
(test_gpu_beam.py::test_coherencies_multifreq_withbeam): its channels overlap and all see the first
channel's beam.  The restated loop therefore predicts channel c with the reference's single-channel
precalculate_coherencies_withbeam at freqs[c], smearing width deltaf / Nchan and, for wide-band element
beams, coefficient set c, and applies the uv cut at ph_freq0 (predict_withbeam.c:474-476,784) to the
rows of the first pass.

The tests that compare with the reference call it first and ask for the product library afterwards,
so that the reference's answers can be recorded on a machine without a GPU."""
import ctypes as C

import numpy as np
import pytest

from util import relerr
from sagecal_b200.dirac_api import BeamSetup, SkyModel, elementcoeff, dptr, make_barr
from test_gpu_beam import DOBEAM
from test_gpu_stochastic import (FREQS5, LBFGS, NMB, NO_CCID, RERUN_TOL, TMB, bands, problem, uv_cut,
                                 assert_close)
import test_gpu_stochastic_consensus as tc

pytestmark = pytest.mark.gpu

RA0, DEC0, PH_FREQ0 = 1.2, np.deg2rad(58.0), 148e6


class Beams:
    """the sky with directions, the stations' positions and elements and the coefficient tables of
    one beam mode; one BeamSetup per interval ([NMB][TMB] JD), per minibatch, and per (minibatch,
    channel) with that channel's coefficient set"""

    def __init__(self, ref, b, mode, tile, freqs, seed=31):
        pr = b.pr
        rng = np.random.default_rng(seed)
        for cl in pr.clusters:   # sources a few degrees around the phase centre
            K = len(cl["ll"])
            cl["ra"] = RA0 + np.deg2rad(rng.uniform(-4, 4, K))
            cl["dec"] = DEC0 + np.deg2rad(rng.uniform(-4, 4, K))
        pr.clusters[-1]["dec"][0] = np.deg2rad(-60.0)   # one source below the horizon: zero gain
        self.sky = SkyModel(pr.clusters, pr.N)
        self.lon = np.deg2rad(6.87 + rng.uniform(-0.5, 0.5, pr.N))
        self.lat = np.deg2rad(52.9 + rng.uniform(-0.3, 0.3, pr.N))
        self.elems = []
        for n in range(pr.N):
            if tile:   # 16 dipoles of a 4 x 4 tile, then 20-24 tile centroids
                g = (np.arange(4) - 1.5) * 1.25
                dip = np.array([[x, y, 0.0] for x in g for y in g])
                cen = np.c_[rng.uniform(-15, 15, (20 + n % 5, 2)), rng.normal(0, 0.05, 20 + n % 5)]
                self.elems.append(np.vstack([dip, cen]))
            else:
                K = 40 + 3 * n
                self.elems.append(np.c_[rng.uniform(-40, 40, (K, 2)), rng.normal(0, 0.1, K)])
        self.mode, self.tile, self.freqs = mode, tile, np.asarray(freqs, dtype=np.float64)
        self.ec = None
        if "element" in mode or "full" in mode:
            self.ec = elementcoeff()
            if mode.endswith("_wb"):
                ref.lib.set_elementcoeffs_wb(1 if tile else 0, dptr(self.freqs), len(self.freqs),
                                             C.byref(self.ec))
            else:
                ref.lib.set_elementcoeffs(1 if tile else 0, C.c_double(float(np.mean(freqs))),
                                          C.byref(self.ec))

    def times(self, ivl, mb=None):
        t0 = 2456789.3 + ivl * NMB * TMB * 10.0 / 86400.0
        t = t0 + np.arange(NMB * TMB) * 10.0 / 86400.0
        return t if mb is None else t[mb * TMB:(mb + 1) * TMB]

    def setup(self, t, ec=None, doBeam=None):
        return BeamSetup(2 if self.tile else 1, RA0 + 0.01, DEC0 - 0.01, RA0, DEC0, PH_FREQ0, self.lon,
                         self.lat, t, self.elems, self.ec if ec is None else ec,
                         DOBEAM[self.mode] if doBeam is None else doBeam)

    def channel_coeff(self, c):
        """coefficient set c of a wide-band table as a one-frequency table"""
        if self.ec is None or not self.mode.endswith("_wb"):
            return None
        ec = elementcoeff(self.ec.M, self.ec.Nmodes, 1, self.ec.beta, None, None, self.ec.preamble)
        off = 16 * self.ec.Nmodes * c
        ec.pattern_phi = self.ec.pattern_phi + off
        ec.pattern_theta = self.ec.pattern_theta + off
        return ec


def beam_cut(u, v, flag, uvmin, uvmax):
    """predict_withbeam.c:474-476 with freq0 = ph_freq0 (:784): unflagged rows outside the cut get 2"""
    uvd = np.sqrt(u * u + v * v) * PH_FREQ0
    out = np.array(flag, dtype=np.uint8)
    out[(out == 0) & ((uvd < uvmin) | (uvd > uvmax))] = 2
    return out


class RefCalls:
    """the driver's beam branches through the reference: coherencies per channel (see the module
    docstring), calculate_residuals_multifreq_withbeam"""

    def __init__(self, ref, beams):
        self.lib, self.bm = ref, beams

    def coherencies(self, pr, ivl, ivi, mb, freqs, deltaf, uvmin, uvmax=1e9):
        R = ivl.R
        coh = []
        for c, f in enumerate(freqs):
            ec = self.bm.channel_coeff(c)
            beam = self.bm.setup(self.bm.times(ivi, mb), ec=ec)
            coh.append(self.lib.precalculate_coherencies_withbeam(
                ivl.u[mb], ivl.v[mb], ivl.w[mb], pr.N, R, ivl.barr(mb), self.bm.sky, f,
                deltaf / len(freqs), beam, uvmin=0.0, uvmax=1e300))
        flag = beam_cut(ivl.u[mb], ivl.v[mb], ivl.flag[mb], uvmin, uvmax)
        return np.concatenate(coh), make_barr(ivl.sta1[mb], ivl.sta2[mb], flag)

    def residuals(self, pr, ivl, ivi, mb, p, xr, freqs, fdelta, **kw):
        beam = self.bm.setup(self.bm.times(ivi, mb))
        return self.lib.calculate_residuals_multifreq_withbeam(
            ivl.u[mb], ivl.v[mb], ivl.w[mb], p, xr, pr.N, pr.Nbase, TMB, ivl.barr(mb), self.bm.sky,
            freqs, fdelta, beam, **kw)


class OwnCalls(RefCalls):
    """the same through this library's reference-named _withbeam calls"""

    def coherencies(self, pr, ivl, ivi, mb, freqs, deltaf, uvmin, uvmax=1e9):
        barr = ivl.barr(mb)
        coh = self.lib.precalculate_coherencies_multifreq(
            ivl.u[mb], ivl.v[mb], ivl.w[mb], pr.N, ivl.R, barr, self.bm.sky, freqs, deltaf,
            self.bm.setup(self.bm.times(ivi, mb)), uvmin=uvmin, uvmax=uvmax)
        return coh, barr


def driver_loop(calls, b, ivl, ivi, freqs, nsolbw, nepochs, pts, pfreq, uvmin, uvmax=1e9, ccid=NO_CCID,
                rho=1e-9, phase_only=0, consensus=None, **kw):
    """minibatch_mode.cpp:368-506 with beams, or with consensus = (step, B, Bi, rhok, Z, nadmm)
    minibatch_consensus_mode.cpp:453-672 with beams; flags preset again at every load.  pfreq (and Z)
    in/out.  returns (residuals, res_00, res_01[, res_0, res_1, fband])"""
    pr, sky, lib = b.pr, calls.bm.sky, calls.lib
    nchan = len(freqs)
    bl = bands(nchan, nsolbw)
    nadmm = consensus[5] if consensus else 1
    shape = (nadmm, nepochs, NMB, nsolbw)
    r0, r1 = np.zeros(shape), np.zeros(shape)
    Y = np.zeros((nsolbw, b.m))
    res_0 = res_1 = 0.0
    fband = None
    coh_all = [None] * NMB
    R, M = ivl.R, sky.M
    for ad in range(nadmm):
        for ep in range(nepochs):
            for mb in range(NMB):
                barr = ivl.barr(mb)
                if ep == 0 and ad == 0:
                    coh_all[mb], barr = calls.coherencies(pr, ivl, ivi, mb, freqs, pr.fdelta * nchan,
                                                          uvmin, uvmax)
                for bi, (c0, nc) in enumerate(bl):
                    coh = np.ascontiguousarray(coh_all[mb][c0 * R * M * 4:(c0 + nc) * R * M * 4])
                    x = np.ascontiguousarray(ivl.x[mb, c0:c0 + nc]).reshape(-1)
                    cons = {}
                    if consensus:
                        cons = dict(Y=Y[bi], Z=tc.bz(consensus[4], consensus[1][bi]),
                                    rho=np.ascontiguousarray(consensus[3][bi]))
                    r0[ad, ep, mb, bi], r1[ad, ep, mb, bi] = lib.bfgsfit_minibatch(
                        ivl.u[mb], ivl.v[mb], ivl.w[mb], x, pr.N, pr.Nbase, TMB, barr, sky, coh,
                        pfreq[bi], freqs[c0:c0 + nc], pts[bi], fdelta=pr.fdelta * nc, nmb=mb,
                        totalmb=NMB, **cons, **kw)
                if consensus:
                    step, B, Bi, rhok, Z, _ = consensus
                    res_0, res_1, fband, _ = step(r0[ad, ep, mb], r1[ad, ep, mb], pfreq, B, Bi, rhok,
                                                  res_0, res_1, Y, Z)
    res = ivl.x.copy()
    for mb in range(NMB):
        for bi, (c0, nc) in enumerate(bl):
            xr = np.ascontiguousarray(res[mb, c0:c0 + nc])
            assert calls.residuals(pr, ivl, ivi, mb, pfreq[bi], xr.reshape(-1), freqs[c0:c0 + nc],
                                   pr.fdelta * nc, ccid=ccid, rho=rho, phase_only=phase_only) == 0
            res[mb, c0:c0 + nc] = xr
    if consensus:
        return res, r0, r1, res_0, res_1, fband
    return res, r0[0], r1[0]


def run_driver(calls, b, ivls, freqs, nsolbw, nepochs, uvmin, **kw):
    lib = calls.lib
    pts = [lib.persist_init(NMB, b.m, 8 * ivls[0].R, LBFGS["lbfgs_m"]) for _ in range(nsolbw)]
    pfreq = np.tile(b.pr.pp0, (nsolbw, 1))
    out = []
    for ivi, ivl in enumerate(ivls):
        res, r0, r1 = driver_loop(calls, b, ivl, ivi, freqs, nsolbw, nepochs, pts, pfreq, uvmin, **kw)
        out.append((res, r0, r1, pfreq.copy()))
    for pt in pts:
        lib.persist_clear(pt)
    return out


def run_interval(api, b, beams, ivls, freqs, nsolbw, nepochs, uvmin, doBeam=None, plain=False, **kw):
    """two intervals back to back through the _withbeam call (plain: the call without beams)"""
    pr = b.pr
    pts = api.persist_init_array(nsolbw, NMB, b.m, 8 * ivls[0].R, kw.get("lbfgs_m", 5))
    pfreq = np.tile(pr.pp0, (nsolbw, 1))
    out = []
    for ivi, ivl in enumerate(ivls):
        xo = ivl.x.copy()
        beam = None if plain else beams.setup(beams.times(ivi), doBeam=doBeam)
        rv, r0, r1 = api.stochastic_interval(ivl.u, ivl.v, ivl.w, xo, pr.N, pr.Nbase, TMB, ivl.barr(),
                                             beams.sky, freqs, pr.fdelta * len(freqs), pts, pfreq,
                                             nsolbw, nepochs, uvmin=uvmin, beam=beam, **kw)
        assert rv == 0
        out.append((xo, r0, r1, pfreq.copy()))
    for i in range(nsolbw):
        api.lib.lbfgs_persist_clear(C.byref(pts[i]))
    return out


def setup(ref, mode, tile, freqs=FREQS5):
    b, _, ivls = problem(freqs)
    beams = Beams(ref, b, mode, tile, freqs)
    return b, beams, ivls, uv_cut(b.pr, freqs)


CASES = [("array", False, NO_CCID, 0), ("full", True, 1, 0), ("element_wb", False, 2, 1),
         ("full_wb", True, NO_CCID, 0)]
CASE_IDS = ["array-single", "full-tile-correct-by-1", "element_wb-single-correct-by-2-phase-only",
            "full_wb-tile"]


@pytest.mark.parametrize("mode,tile,ccid,phase_only", CASES, ids=CASE_IDS)
def test_interval_against_reference(ref, request, mode, tile, ccid, phase_only):
    """5 channels in bands of 3 and 2, 3 epochs, two intervals: every fit's costs, each band's Jones
    after each interval and the residuals with the correction; the beam changes the answer"""
    b, beams, ivls, uvmin = setup(ref, mode, tile)
    kw = dict(ccid=ccid, rho=1e-9, phase_only=phase_only, **LBFGS)
    want = run_driver(RefCalls(ref, beams), b, ivls, FREQS5, 2, 3, uvmin, **kw)
    assert relerr(want[1][3][0], want[1][3][1]) > 1e-4           # the bands' solutions differ
    api = request.getfixturevalue("api")
    got = run_interval(api, b, beams, ivls, FREQS5, 2, 3, uvmin, **kw)
    assert_close(got, want, 1e-9, 1e-7, 1e-6, 1e-6)
    plain = run_interval(api, b, beams, ivls, FREQS5, 2, 3, uvmin, plain=True, **kw)
    assert relerr(plain[1][0], got[1][0]) > 1e-3
    assert relerr(plain[1][3], got[1][3]) > 1e-4


def run_consensus(api, b, beams, ivls, freqs, nsolbw, B, Bi, rhok, uvmin, **kw):
    pr = b.pr
    pts = api.persist_init_array(nsolbw, NMB, b.m, 8 * ivls[0].R, kw.get("lbfgs_m", 5))
    pfreq = np.tile(pr.pp0, (nsolbw, 1))
    Z = np.zeros((beams.sky.Mt, B.shape[1], 8 * pr.N))
    out = []
    for ivi, ivl in enumerate(ivls):
        xo = ivl.x.copy()
        rv, r0, r1, q0, q1, fb = api.stochastic_consensus_interval(
            ivl.u, ivl.v, ivl.w, xo, pr.N, pr.Nbase, TMB, ivl.barr(), beams.sky, freqs,
            pr.fdelta * len(freqs), pts, pfreq, nsolbw, tc.NEPOCHS, tc.NADMM, B, Bi, rhok, Z,
            uvmin=uvmin, beam=beams.setup(beams.times(ivi)), **kw)
        assert rv == 0
        out.append((xo, r0, r1, pfreq.copy(), Z.copy(), q0, q1, fb.copy()))
    for i in range(nsolbw):
        api.lib.lbfgs_persist_clear(C.byref(pts[i]))
    return out


def run_consensus_driver(calls, step, b, ivls, freqs, nsolbw, B, Bi, rhok, uvmin, **kw):
    lib = calls.lib
    pts = [lib.persist_init(NMB, b.m, 8 * ivls[0].R, LBFGS["lbfgs_m"]) for _ in range(nsolbw)]
    pfreq = np.tile(b.pr.pp0, (nsolbw, 1))
    Z = np.zeros((calls.bm.sky.Mt, B.shape[1], 8 * b.pr.N))
    out = []
    for ivi, ivl in enumerate(ivls):
        res, r0, r1, q0, q1, fb = driver_loop(calls, b, ivl, ivi, freqs, nsolbw, tc.NEPOCHS, pts,
                                              pfreq, uvmin,
                                              consensus=(step, B, Bi, rhok, Z, tc.NADMM), **kw)
        out.append((res, r0, r1, pfreq.copy(), Z.copy(), q0, q1, np.array(fb)))
    for pt in pts:
        lib.persist_clear(pt)
    return out


@pytest.mark.parametrize("mode,tile,ccid", [("full", False, 1), ("array_wb", True, NO_CCID)],
                         ids=["full-single-correct-by-1", "array_wb-tile"])
def test_consensus_interval_against_reference(ref, request, mode, tile, ccid):
    """the consensus interval with beams, Npoly 2, 3 ADMM iterations of 2 epochs, two intervals: every
    fit's costs, each band's Jones, Z, fband, res_0 / res_1 and the residuals"""
    b, beams, ivls, uvmin = setup(ref, mode, tile)
    kw = dict(ccid=ccid, rho=1e-9, **LBFGS)
    B, Bi, rhok = tc.consensus_setup(ref, FREQS5, 2, beams.sky.Mt, 2)
    want = run_consensus_driver(RefCalls(ref, beams), tc.ref_step(ref, b.pr.N), b, ivls, FREQS5, 2, B,
                                Bi, rhok, uvmin, **kw)
    api = request.getfixturevalue("api")
    got = run_consensus(api, b, beams, ivls, FREQS5, 2, B, Bi, rhok, uvmin, **kw)
    tc.assert_close(got, want, 1e-9, 1e-7, 1e-6, 1e-6)


# The data are simulated without beams, so a beam model fits them poorly, and over 3 LBFGS
# iterations x 3 epochs x 2 intervals the last-bit differences of the atomic gradient sums grow more
# than on the beam-less problem of test_gpu_stochastic.py: 2.7e-9 in the array-single case on an H100
# (test_no_iterations_bit_identical_and_launch_counts shows the two paths compute the same thing)
@pytest.mark.parametrize("mode,tile,tol", [("full_wb", True, RERUN_TOL), ("array", False, 1e-8)],
                         ids=["full_wb-tile", "array-single"])
def test_interval_equals_the_reference_named_loop(ref, request, mode, tile, tol):
    """keeping the coherencies and the beam tables on the device changes nothing: the interval call
    and this library's own _withbeam calls agree as closely as two runs of one of them; the interval
    uploads the sky once and moves no coherencies, the loop uploads it at every call"""
    b, beams, ivls, uvmin = setup(ref, mode, tile)
    api = request.getfixturevalue("api")
    kw = dict(ccid=1, rho=1e-9, **LBFGS)
    api.transfer_stats(reset=True)
    want = run_driver(OwnCalls(api, beams), b, ivls, FREQS5, 2, 3, uvmin, **kw)
    # per interval: NMB x 5 channel predictions and NMB x 2 band residuals; the fits move coherencies
    nup, nbytes = api.transfer_stats(reset=True)
    assert nup == 2 * NMB * (5 + 2) and nbytes > 0
    got = run_interval(api, b, beams, ivls, FREQS5, 2, 3, uvmin, **kw)
    assert api.transfer_stats(reset=True) == (2, 0)
    assert_close(got, want, tol, tol, tol, tol)


def test_no_iterations_bit_identical_and_launch_counts(ref, request):
    """max_lbfgs = 0: the interval call's residuals are those of this library's _withbeam loop to the
    bit.  Beam tables: one launch per (minibatch, channel) in the first pass and one per (minibatch,
    non-empty band) in the residual pass; coherencies: one launch per (minibatch, channel); cost and
    gradient launches per fit as without beams"""
    b, beams, ivls, uvmin = setup(ref, "full_wb", True)
    api = request.getfixturevalue("api")
    kw = dict(LBFGS, max_lbfgs=0, ccid=1)
    want = run_driver(OwnCalls(api, beams), b, ivls[:1], FREQS5, 2, 3, uvmin, **kw)
    k = {i: api.kernel_count(i) for i in (13, 14, 15, 16)}
    got = run_interval(api, b, beams, ivls[:1], FREQS5, 2, 3, uvmin, **kw)
    d = {i: api.kernel_count(i) - k[i] for i in k}
    nfits = 3 * NMB * 2
    assert d[15] == NMB * 5 + NMB * 2
    assert d[16] == NMB * 5
    assert d[13] == 3 * nfits and d[14] == nfits
    assert np.array_equal(got[0][0], want[0][0])
    assert np.array_equal(got[0][3], want[0][3])
    for i in (1, 2):
        assert relerr(got[0][i], want[0][i]) < 1e-13


def test_nine_channels_with_an_empty_band_launch_counts(ref, request):
    """9 channels in 4 bands (3, 3, 3, 0): the residual pass builds tables for the three bands with
    channels only"""
    freqs = np.linspace(140e6, 164e6, 9)
    b, beams, ivls, uvmin = setup(ref, "element_wb", False, freqs=freqs)
    api = request.getfixturevalue("api")
    k15 = api.kernel_count(15)
    got = run_interval(api, b, beams, ivls[:1], freqs, 4, 1, uvmin, **dict(LBFGS, max_lbfgs=0))
    assert api.kernel_count(15) - k15 == NMB * 9 + NMB * 3
    assert np.isnan(got[0][1][:, :, 3]).all()


def test_uv_cut_at_ph_freq0_in_the_first_pass_only(ref, request):
    """the beam's cut is taken at ph_freq0, both ways, in the first epoch only: a uvmax that cuts
    rows at ph_freq0 changes the first epoch's costs, and the interval follows this library's
    _withbeam loop, which cuts in the same way, for uvmin and uvmax; the later epochs re-preset the
    flags"""
    b, beams, ivls, uvmin = setup(ref, "array", True)
    api = request.getfixturevalue("api")
    pr = b.pr
    uvd = np.sqrt(pr.u ** 2 + pr.v ** 2)[pr.flag == 0] * PH_FREQ0
    uvmax = float(np.quantile(uvd, 0.8))
    # the cut at ph_freq0 differs from one at the first or last channel
    lo = np.sqrt(pr.u ** 2 + pr.v ** 2)[pr.flag == 0]
    assert np.sum(lo * PH_FREQ0 < uvmin) != np.sum(lo * FREQS5[0] < uvmin)
    ref_ = run_interval(api, b, beams, ivls[:1], FREQS5, 2, 2, 0.0, **LBFGS)
    for lo_, hi_ in ((uvmin, 1e9), (0.0, uvmax)):
        got = run_interval(api, b, beams, ivls[:1], FREQS5, 2, 2, lo_, uvmax=hi_, **LBFGS)
        assert abs(got[0][1][0, 0, 0] - ref_[0][1][0, 0, 0]) > 1e-6 * ref_[0][1][0, 0, 0]
        want = run_driver(OwnCalls(api, beams), b, ivls[:1], FREQS5, 2, 2, lo_, uvmax=hi_, **LBFGS)
        assert_close(got, want, RERUN_TOL, RERUN_TOL, RERUN_TOL, RERUN_TOL)


def test_dobeam_none_is_the_plain_call(ref, request):
    """doBeam = 0 through the _withbeam call is the call without beams, to the bit at max_lbfgs = 0"""
    b, beams, ivls, uvmin = setup(ref, "full", False)
    api = request.getfixturevalue("api")
    kw = dict(LBFGS, max_lbfgs=0, ccid=1)
    k15 = api.kernel_count(15)
    got = run_interval(api, b, beams, ivls, FREQS5, 2, 2, uvmin, doBeam=0, **kw)
    assert api.kernel_count(15) == k15
    want = run_interval(api, b, beams, ivls, FREQS5, 2, 2, uvmin, plain=True, **kw)
    for g, w in zip(got, want):
        for i in range(4):
            assert np.array_equal(g[i], w[i])


class _Stripped:
    """a BeamSetup with some of its tail replaced"""

    def __init__(self, beam, **repl):
        self.b, self.repl, self.tilesz = beam, repl, beam.tilesz

    def head(self):
        h = list(self.b.head())
        if "bf_type" in self.repl:
            h[0] = self.repl["bf_type"]
        return tuple(h)

    def tail(self):
        Nelem, xx, yy, zz, ec, doBeam = self.b.tail()
        t = dict(Nelem=Nelem, xx=xx, yy=yy, zz=zz, ec=ec, doBeam=doBeam)
        t.update({k: v for k, v in self.repl.items() if k != "bf_type"})
        return t["Nelem"], t["xx"], t["yy"], t["zz"], t["ec"], t["doBeam"]


def test_refusals(ref, request, capfd):
    """bad beam arguments: -1 with a message, before any device work, xo, pfreq, the costs and Z
    untouched, for both calls"""
    b, beams, ivls, uvmin = setup(ref, "full_wb", True)
    narrow = Beams(ref, b, "element", True, FREQS5)
    short = elementcoeff()
    ref.lib.set_elementcoeffs_wb(1, dptr(FREQS5[:3]), 3, C.byref(short))
    api = request.getfixturevalue("api")
    pr, ivl = b.pr, ivls[0]
    full = beams.setup(beams.times(0))
    cases = [
        (_Stripped(full, doBeam=7), "doBeam = 7 is not a beam mode"),
        (_Stripped(full, doBeam=-1), "doBeam = -1 is not a beam mode"),
        (_Stripped(full, bf_type=3), "needs bf_type STAT_SINGLE or STAT_TILE"),
        (_Stripped(full, doBeam=1, bf_type=0), "needs bf_type STAT_SINGLE or STAT_TILE"),
        (_Stripped(full, Nelem=None), "needs Nelem and the element positions"),
        (_Stripped(full, doBeam=4, xx=None), "needs Nelem and the element positions"),
        (_Stripped(full, ec=None), "needs coefficient tables"),
        (_Stripped(narrow.setup(beams.times(0)), ec=None), "needs coefficient tables"),
        (_Stripped(full, ec=C.byref(short)), "needs one coefficient set per channel"),
    ]
    pts = api.persist_init_array(2, NMB, b.m, 8 * ivl.R, 5)
    B, Bi, rhok = np.ones((2, 2)), np.ones((beams.sky.Mt, 2, 2)), np.ones((2, beams.sky.Mt))
    for beam, msg in cases:
        for consensus in (False, True):
            xo = ivl.x.copy()
            pfreq = np.tile(pr.pp0, (2, 1)) + 0.25
            Z = np.full((beams.sky.Mt, 2, 8 * pr.N), 3.0)
            if consensus:
                rv, r0, r1, q0, q1, fb = api.stochastic_consensus_interval(
                    ivl.u, ivl.v, ivl.w, xo, pr.N, pr.Nbase, TMB, ivl.barr(), beams.sky, FREQS5,
                    pr.fdelta * 5, pts, pfreq, 2, 2, 2, B, Bi, rhok, Z, beam=beam, **LBFGS)
                assert q0 == 0.0 and q1 == 0.0 and not fb.any()
            else:
                rv, r0, r1 = api.stochastic_interval(ivl.u, ivl.v, ivl.w, xo, pr.N, pr.Nbase, TMB,
                                                     ivl.barr(), beams.sky, FREQS5, pr.fdelta * 5, pts,
                                                     pfreq, 2, 2, beam=beam, **LBFGS)
            assert rv == -1, msg
            assert msg in capfd.readouterr().err, msg
            assert not r0.any() and not r1.any()
            assert np.array_equal(xo, ivl.x)
            assert np.array_equal(pfreq, np.tile(pr.pp0, (2, 1)) + 0.25)
            assert (Z == 3.0).all()
    for i in range(2):
        api.lib.lbfgs_persist_clear(C.byref(pts[i]))
