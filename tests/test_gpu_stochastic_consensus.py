"""Stochastic calibration with spectral consensus over the bands (sagecal -N <epochs> -M <minibatches>
-w <bands> -A <nadmm>, minibatch_consensus_mode.cpp:450-672, no beam):
dirac_b200_stochastic_consensus_interval against the driver's loop restated with the reference's
precalculate_coherencies_multifreq, bfgsfit_minibatch_consensus, calculate_residuals_multifreq and
update_global_z_multi, and against the same loop made of this library's reference-named calls and
dirac_b200_consensus_bands_update.  Two intervals run back to back with the LBFGS state, the bands'
Jones and Z carried over, at 3 ADMM iterations of 2 epochs, PolyType 2 (Bernstein, the driver's
default).

The tests that compare with the reference call it first and ask for the product library afterwards,
so that the reference's answers can be recorded on a machine without a GPU."""
import ctypes as C

import numpy as np
import pytest

from util import relerr
from test_gpu_stochastic import (FREQS5, FREQS9, LBFGS, NMB, NO_CCID, RERUN_TOL, TMB, bands,
                                 problem, uv_cut)

pytestmark = pytest.mark.gpu

NADMM, NEPOCHS = 3, 2
ADMM_RHO = 5.0            # the driver's -r default
POLYTYPE = 2
RES_RATIO, CLM_DBL_MAX = 1.5, 1e12
vp = C.c_void_p


def _p(a):
    return a.ctypes.data_as(vp)


def band_freqs(freqs, nsolbw):
    """each band's mean frequency (:350-357).  The mean over a band without channels is 0/0 in the
    driver, which makes the whole basis NaN; such a band is put at the last channel's frequency here"""
    return np.array([freqs[c0:c0 + nc].mean() if nc else freqs[-1] for c0, nc in bands(len(freqs),
                                                                                      nsolbw)])


def consensus_setup(ref, freqs, nsolbw, Mt, Npoly, rho=ADMM_RHO):
    """B by setup_polynomials (type 1 when Npoly is 1, :359), rhok = rho everywhere (setweights), Bi by
    find_prod_inverse_full, all from the reference"""
    ffreq = band_freqs(freqs, nsolbw)
    B = np.zeros((nsolbw, Npoly))
    ref.lib.setup_polynomials.argtypes = [vp, C.c_int, C.c_int, vp, C.c_double, C.c_int]
    ref.lib.setup_polynomials(_p(B), Npoly, nsolbw, _p(ffreq), float(np.mean(freqs)),
                              1 if Npoly == 1 else POLYTYPE)
    rhok = np.full((nsolbw, Mt), rho)
    Bi = np.zeros((Mt, Npoly, Npoly))
    ref.lib.find_prod_inverse_full.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, vp, C.c_int]
    ref.lib.find_prod_inverse_full(_p(B), _p(Bi), Npoly, nsolbw, Mt, _p(rhok), 4)
    return B, Bi, rhok


def bz(Z, Bb):
    """B_b Z in the driver's order (:526-531); Z [Mt, Npoly, 8N] -> [Mt * 8N]"""
    z = np.zeros(Z.shape[0] * Z.shape[2])
    for p in range(Z.shape[1]):
        z += Bb[p] * Z[:, p, :].reshape(-1)
    return z


def ref_step(ref, N):
    """the ADMM step (:540-601) in numpy around the reference's update_global_z_multi; also returns
    every band's distance to the 1.5 res_1 threshold"""
    def step(r00, r01, J, B, Bi, rhok, res_0, res_1, Y, Z):
        nsolbw, Npoly = B.shape
        Mt = Bi.shape[0]
        resband = np.zeros(nsolbw)
        with np.errstate(invalid="ignore"):     # a band without channels: its costs are not finite
            for b in range(nsolbw):
                res_0 += r00[b]
                res_1 += r01[b]
                resband[b] = r01[b] if (r00[b] > 0.0 and r01[b] > 0.0) else CLM_DBL_MAX
            res_0 /= nsolbw
            res_1 /= nsolbw
            fband = (resband > RES_RATIO * res_1).astype(np.int32)
        rho_i = np.repeat(rhok, 8 * N, axis=1)
        for b in range(nsolbw):
            if not fband[b]:
                Y[b] += rho_i[b] * J[b]
        z = B[0][:, None] * Y[0][None, :]
        for b in range(1, nsolbw):
            if not fband[b]:
                z += B[b][:, None] * Y[b][None, :]
        z = np.ascontiguousarray(z)
        ref.lib.update_global_z_multi.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp, vp, C.c_int]
        ref.lib.update_global_z_multi(_p(Z), N, Mt, Npoly, _p(z), _p(np.ascontiguousarray(Bi)), 4)
        for b in range(nsolbw):
            if not fband[b]:
                Y[b] -= rho_i[b] * bz(Z, B[b])
        return res_0, res_1, fband, np.abs(resband - RES_RATIO * res_1)
    return step


def api_step(api, N):
    def step(r00, r01, J, B, Bi, rhok, res_0, res_1, Y, Z):
        rv, res_0, res_1, fband = api.consensus_bands_update(N, r00, r01, J, B, Bi, rhok, res_0, res_1,
                                                             Y, Z)
        assert rv == 0
        return res_0, res_1, fband, None
    return step


def driver_loop(lib, step, b, sky, ivl, freqs, nsolbw, pts, pfreq, Z, B, Bi, rhok, uvmin, nadmm,
                nepochs, use_global=0, ccid=NO_CCID, rho=1e-9, phase_only=0, **kw):
    """minibatch_consensus_mode.cpp:453-672 through the reference-named calls of `lib` and the ADMM
    step `step`; pfreq and Z in/out.  returns (residuals, res_00, res_01, res_0, res_1, fband, primal
    [nadmm, nepochs, NMB, nsolbw], threshold distances)"""
    pr = b.pr
    nchan = len(freqs)
    deltaf = pr.fdelta * nchan
    bl = bands(nchan, nsolbw)
    shape = (nadmm, nepochs, NMB, nsolbw)
    r0, r1, primal = np.zeros(shape), np.zeros(shape), np.zeros(shape)
    Y = np.zeros((nsolbw, b.m))
    res_0 = res_1 = 0.0
    fband, margins = None, []
    coh_all = [None] * NMB
    R, M = ivl.R, sky.M
    for ad in range(nadmm):
        for ep in range(nepochs):
            for mb in range(NMB):
                barr = ivl.barr(mb)
                if ep == 0 and ad == 0:
                    coh_all[mb] = lib.precalculate_coherencies_multifreq(
                        ivl.u[mb], ivl.v[mb], ivl.w[mb], pr.N, R, barr, sky, freqs, deltaf, uvmin=uvmin)
                for bi, (c0, nc) in enumerate(bl):
                    z = bz(Z, B[bi])
                    coh = np.ascontiguousarray(coh_all[mb][c0 * R * M * 4:(c0 + nc) * R * M * 4])
                    x = np.ascontiguousarray(ivl.x[mb, c0:c0 + nc]).reshape(-1)
                    r0[ad, ep, mb, bi], r1[ad, ep, mb, bi] = lib.bfgsfit_minibatch(
                        ivl.u[mb], ivl.v[mb], ivl.w[mb], x, pr.N, pr.Nbase, TMB, barr, sky, coh,
                        pfreq[bi], freqs[c0:c0 + nc], pts[bi], fdelta=pr.fdelta * nc, nmb=mb,
                        totalmb=NMB, Y=Y[bi], Z=z, rho=np.ascontiguousarray(rhok[bi]), **kw)
                    primal[ad, ep, mb, bi] = np.linalg.norm(pfreq[bi] - z)
                res_0, res_1, fband, mg = step(r0[ad, ep, mb], r1[ad, ep, mb], pfreq, B, Bi, rhok,
                                               res_0, res_1, Y, Z)
                margins.append(mg)
    if use_global:
        for bi in range(nsolbw):
            pfreq[bi] = bz(Z, B[bi])
    res = ivl.x.copy()
    for mb in range(NMB):
        barr = ivl.barr(mb)
        for bi, (c0, nc) in enumerate(bl):
            if nc == 0:
                continue
            xr = np.ascontiguousarray(res[mb, c0:c0 + nc])
            assert lib.calculate_residuals_multifreq(
                ivl.u[mb], ivl.v[mb], ivl.w[mb], pfreq[bi], xr.reshape(-1), pr.N, pr.Nbase, TMB, barr,
                sky, freqs[c0:c0 + nc], pr.fdelta * nc, ccid=ccid, rho=rho, phase_only=phase_only) == 0
            res[mb, c0:c0 + nc] = xr
    return res, r0, r1, res_0, res_1, fband, primal, margins


def run_driver(lib, step, b, sky, ivls, freqs, nsolbw, B, Bi, rhok, uvmin, nadmm=NADMM,
               nepochs=NEPOCHS, **kw):
    """both intervals back to back, pt, pfreq and Z carried over; one tuple per interval:
    (res, r00, r01, pfreq, Z, res_0, res_1, fband, primal, margins)"""
    pts = [lib.persist_init(NMB, b.m, 8 * ivls[0].R, LBFGS["lbfgs_m"]) for _ in range(nsolbw)]
    pfreq = np.tile(b.pr.pp0, (nsolbw, 1))
    Z = np.zeros((sky.Mt, B.shape[1], 8 * b.pr.N))
    out = []
    for ivl in ivls:
        res, r0, r1, q0, q1, fb, primal, mg = driver_loop(lib, step, b, sky, ivl, freqs, nsolbw, pts,
                                                          pfreq, Z, B, Bi, rhok, uvmin, nadmm, nepochs,
                                                          **kw)
        out.append((res, r0, r1, pfreq.copy(), Z.copy(), q0, q1, np.array(fb), primal, mg))
    for pt in pts:
        lib.persist_clear(pt)
    return out


def run_interval(api, b, sky, ivls, freqs, nsolbw, B, Bi, rhok, uvmin, nadmm=NADMM, nepochs=NEPOCHS,
                 use_global=0, **kw):
    pr = b.pr
    pts = api.persist_init_array(nsolbw, NMB, b.m, 8 * ivls[0].R, kw.get("lbfgs_m", 5))
    pfreq = np.tile(pr.pp0, (nsolbw, 1))
    Z = np.zeros((sky.Mt, B.shape[1], 8 * pr.N))
    out = []
    for ivl in ivls:
        xo = ivl.x.copy()
        rv, r0, r1, q0, q1, fb = api.stochastic_consensus_interval(
            ivl.u, ivl.v, ivl.w, xo, pr.N, pr.Nbase, TMB, ivl.barr(), sky, freqs,
            pr.fdelta * len(freqs), pts, pfreq, nsolbw, nepochs, nadmm, B, Bi, rhok, Z,
            use_global=use_global, uvmin=uvmin, **kw)
        assert rv == 0
        out.append((xo, r0, r1, pfreq.copy(), Z.copy(), q0, q1, fb.copy()))
    for b_ in range(nsolbw):
        api.lib.lbfgs_persist_clear(C.byref(pts[b_]))
    return out


def _costs_close(g, w, tol):
    fin = np.isfinite(w)
    assert np.array_equal(fin, np.isfinite(g))
    assert np.array_equal(g[~fin], w[~fin], equal_nan=True)
    if fin.any():
        assert np.max(np.abs(g[fin] - w[fin]) / np.abs(w[fin])) <= tol


def assert_close(got, want, tol_r0, tol_r1, tol_p, tol_x):
    for g, w in zip(got, want):
        xg, g0, g1, pg, Zg, q0g, q1g, fbg = g
        xw, w0, w1, pw, Zw, q0w, q1w, fbw = w[:8]
        _costs_close(g0, w0, tol_r0)
        _costs_close(g1, w1, tol_r1)
        _costs_close(np.array([q0g]), np.array([q0w]), tol_r0)
        _costs_close(np.array([q1g]), np.array([q1w]), tol_r1)
        assert np.array_equal(fbg, fbw), (fbg, fbw)
        for bi in range(len(pw)):
            assert relerr(pg[bi], pw[bi]) <= tol_p, (bi, relerr(pg[bi], pw[bi]))
        assert relerr(Zg, Zw) <= tol_p, relerr(Zg, Zw)
        assert np.max(np.abs(xg - xw)) <= tol_x * np.max(np.abs(xw)), np.max(np.abs(xg - xw))


def _assert_no_band_at_the_threshold(want):
    for iv in want:
        for mg in iv[9]:
            assert np.all(mg > 1e-6), mg


CASES = [(NO_CCID, 0), (1, 0)]
CASE_IDS = ["plain", "correct-by-1"]


@pytest.mark.parametrize("ccid,phase_only", CASES, ids=CASE_IDS)
def test_interval_against_reference(ref, request, ccid, phase_only):
    """5 channels in bands of 3 and 2, Npoly 2: every fit's costs, each band's Jones, Z, fband,
    res_0 / res_1 and the residuals after each of two intervals"""
    b, sky, ivls = problem(FREQS5)
    uvmin = uv_cut(b.pr, FREQS5)
    kw = dict(ccid=ccid, rho=1e-9, phase_only=phase_only, **LBFGS)
    B, Bi, rhok = consensus_setup(ref, FREQS5, 2, sky.Mt, 2)
    want = run_driver(ref, ref_step(ref, b.pr.N), b, sky, ivls, FREQS5, 2, B, Bi, rhok, uvmin, **kw)
    primal = want[0][8]
    assert primal[-1].mean() < primal[0].mean()                 # the bands approach B_b Z
    _assert_no_band_at_the_threshold(want)
    assert relerr(want[1][3][0], want[1][3][1]) > 1e-4           # the bands' solutions differ
    api = request.getfixturevalue("api")
    got = run_interval(api, b, sky, ivls, FREQS5, 2, B, Bi, rhok, uvmin, **kw)
    assert_close(got, want, 1e-9, 1e-7, 1e-6, 1e-6)


def _noisy(ivls, chans, scale=10.0, seed=5):
    """about `scale` times the noise on channels `chans`, flagged rows kept zero"""
    rng = np.random.default_rng(seed)
    for ivl in ivls:
        for mb in range(NMB):
            for c in chans:
                x = ivl.x[mb, c]
                sig = 1e-2 * np.median(np.abs(x[x != 0]))
                x += rng.normal(0, scale * sig, x.shape)
                x.reshape(-1, 8)[ivl.flag[mb] != 0] = 0.0


@pytest.mark.parametrize("noisy_band,scale", [(1, 10.0), (0, 20.0)], ids=["band-1", "band-0"])
def test_noisy_band_is_flagged(ref, request, noisy_band, scale):
    """5 channels in bands of 2, 2 and 1; one band's channels 10 or 20 times noisier.  The reference
    flags that band in the last minibatch of both intervals: it leaves the band's Y out of the update,
    yet band 0's Y is summed into z whatever its flag.  A band's cost includes its consensus terms,
    which can make it negative (resband 1e12), so the flags depend on rho as much as on the noise; at
    ADMM rho 0.1 they follow the noise"""
    b, sky, ivls = problem(FREQS5)
    c0, nc = bands(5, 3)[noisy_band]
    _noisy(ivls, range(c0, c0 + nc), scale)
    uvmin = uv_cut(b.pr, FREQS5)
    kw = dict(ccid=1, **LBFGS)
    B, Bi, rhok = consensus_setup(ref, FREQS5, 3, sky.Mt, 2, rho=0.1)
    want = run_driver(ref, ref_step(ref, b.pr.N), b, sky, ivls, FREQS5, 3, B, Bi, rhok, uvmin, **kw)
    expect = np.zeros(3, dtype=np.int32)
    expect[noisy_band] = 1
    for iv in want:
        assert np.array_equal(iv[7], expect), iv[7]
    _assert_no_band_at_the_threshold(want)
    api = request.getfixturevalue("api")
    got = run_interval(api, b, sky, ivls, FREQS5, 3, B, Bi, rhok, uvmin, **kw)
    assert_close(got, want, 1e-9, 1e-7, 1e-6, 1e-6)


def test_band_without_channels(ref, request):
    """9 channels in 4 bands: 3, 3, 3 and 0 channels, one interval.  The empty band has no data, only
    the consensus terms, so its costs are (consensus) x 1/0 and its Jones move towards B_b Z; the
    interval call matches the reference"""
    b, sky, ivls = problem(FREQS9)
    ivls = ivls[:1]
    uvmin = uv_cut(b.pr, FREQS9)
    kw = dict(ccid=1, **LBFGS)
    B, Bi, rhok = consensus_setup(ref, FREQS9, 4, sky.Mt, 3)
    want = run_driver(ref, ref_step(ref, b.pr.N), b, sky, ivls, FREQS9, 4, B, Bi, rhok, uvmin, **kw)
    for iv in want:
        assert not np.isfinite(iv[1][..., 3]).any() and np.isfinite(iv[1][..., :3]).all()
    api = request.getfixturevalue("api")
    got = run_interval(api, b, sky, ivls, FREQS9, 4, B, Bi, rhok, uvmin, **kw)
    assert_close(got, want, 1e-9, 1e-7, 1e-6, 1e-6)


def test_use_global(api):
    """-U: every band's returned Jones are B_b Z, and the residuals are those of these Jones"""
    from sagecal_b200 import consensus as cons
    b, sky, ivls = problem(FREQS5)
    pr = b.pr
    uvmin = uv_cut(pr, FREQS5)
    B = cons.basis(api, band_freqs(FREQS5, 2), float(np.mean(FREQS5)), 2, POLYTYPE)
    rhok = np.full((2, sky.Mt), ADMM_RHO)
    Bi = cons.prod_inverse(api, B, rhok)
    got = run_interval(api, b, sky, ivls[:1], FREQS5, 2, B, Bi, rhok, uvmin, use_global=1, ccid=1,
                       **LBFGS)
    xo, _, _, pfreq, Z = got[0][:5]
    assert np.abs(Z).max() > 0
    ivl = ivls[0]
    for bi, (c0, nc) in enumerate(bands(5, 2)):
        assert np.array_equal(pfreq[bi], bz(Z, B[bi]))
        for mb in range(NMB):
            xr = np.ascontiguousarray(ivl.x[mb, c0:c0 + nc])
            assert api.calculate_residuals_multifreq(
                ivl.u[mb], ivl.v[mb], ivl.w[mb], pfreq[bi], xr.reshape(-1), pr.N, pr.Nbase, TMB,
                ivl.barr(mb), sky, FREQS5[c0:c0 + nc], pr.fdelta * nc, ccid=1) == 0
            assert np.max(np.abs(xo[mb, c0:c0 + nc] - xr)) <= 1e-12 * np.max(np.abs(xr))


@pytest.mark.parametrize("max_lbfgs", [0, 3])
def test_zero_rho_is_the_plain_interval(api, max_lbfgs):
    """rhok = 0 with Y and Z zero: the consensus terms add exactly zero, so 2 ADMM iterations of 1
    epoch are the plain interval's 2 epochs (the same loop order, the uv cut in the first pass only)
    and Z stays zero: to the bit without LBFGS iterations, as two runs of one fit otherwise"""
    from test_gpu_stochastic import run_interval as run_plain
    b, sky, ivls = problem(FREQS5)
    uvmin = uv_cut(b.pr, FREQS5)
    kw = dict(LBFGS, max_lbfgs=max_lbfgs, ccid=1)
    B = np.array([[1.0, 0.0], [0.0, 1.0]])
    rhok = np.zeros((2, sky.Mt))
    Bi = np.zeros((sky.Mt, 2, 2))
    got = run_interval(api, b, sky, ivls, FREQS5, 2, B, Bi, rhok, uvmin, nadmm=2, nepochs=1, **kw)
    want = run_plain(api, b, sky, ivls, FREQS5, 2, 2, uvmin, **kw)
    for g, w in zip(got, want):
        assert not g[4].any()
        assert not g[7].any()
        if max_lbfgs == 0:
            assert np.array_equal(g[0], w[0])
            assert np.array_equal(g[3], w[3])
            assert np.array_equal(g[1].reshape(w[1].shape), w[1])
            assert np.array_equal(g[2].reshape(w[2].shape), w[2])
        else:
            assert relerr(g[0], w[0]) <= RERUN_TOL
            assert relerr(g[3], w[3]) <= RERUN_TOL
            assert relerr(g[1].reshape(w[1].shape), w[1]) <= RERUN_TOL
            assert relerr(g[2].reshape(w[2].shape), w[2]) <= RERUN_TOL


def test_interval_equals_the_reference_named_loop(api):
    """keeping the coherencies on the device changes nothing: the interval call and this library's
    own reference-named calls with its host ADMM step agree as closely as two runs of one of them;
    the interval uploads the sky once and moves no coherencies"""
    from sagecal_b200 import consensus as cons
    b, sky, ivls = problem(FREQS5)
    uvmin = uv_cut(b.pr, FREQS5)
    kw = dict(ccid=1, rho=1e-9, **LBFGS)
    B = cons.basis(api, band_freqs(FREQS5, 2), float(np.mean(FREQS5)), 2, POLYTYPE)
    rhok = np.full((2, sky.Mt), ADMM_RHO)
    Bi = cons.prod_inverse(api, B, rhok)
    want = run_driver(api, api_step(api, b.pr.N), b, sky, ivls, FREQS5, 2, B, Bi, rhok, uvmin, **kw)
    api.transfer_stats(reset=True)
    run_interval(api, b, sky, ivls[:1], FREQS5, 2, B, Bi, rhok, uvmin, **kw)
    assert api.transfer_stats(reset=True) == (1, 0)
    got = run_interval(api, b, sky, ivls, FREQS5, 2, B, Bi, rhok, uvmin, **kw)
    assert_close(got, want, RERUN_TOL, RERUN_TOL, RERUN_TOL, RERUN_TOL)


@pytest.mark.parametrize("nsolbw,nadmm,Npoly", [(6, 2, 2), (0, 2, 2), (2, 0, 2), (2, 2, 0)],
                         ids=["more-bands-than-channels", "no-bands", "no-admm", "no-poly"])
def test_refusals(api, nsolbw, nadmm, Npoly):
    """-1 before any work, no output touched"""
    b, sky, ivls = problem(FREQS5)
    pr = b.pr
    ivl = ivls[0]
    nb = max(nsolbw, 1)
    pts = api.persist_init_array(nb, NMB, b.m, 8 * ivl.R, 5)
    pfreq = np.tile(pr.pp0, (nb, 1)) + 0.25
    xo = ivl.x.copy()
    B = np.ones((nb, max(Npoly, 0)))
    Z = np.full((sky.Mt, max(Npoly, 1), 8 * pr.N), 0.5)
    rv, r0, r1, q0, q1, fb = api.stochastic_consensus_interval(
        ivl.u, ivl.v, ivl.w, xo, pr.N, pr.Nbase, TMB, ivl.barr(), sky, FREQS5, pr.fdelta * 5, pts,
        pfreq, nsolbw, 2, nadmm, B, np.ones((sky.Mt, max(Npoly, 1), max(Npoly, 1))),
        np.ones((nb, sky.Mt)), Z, **LBFGS)
    assert rv == -1
    assert not r0.any() and not r1.any() and q0 == 0.0 and q1 == 0.0 and not fb.any()
    assert np.array_equal(xo, ivl.x)
    assert np.array_equal(pfreq, np.tile(pr.pp0, (nb, 1)) + 0.25)
    assert (Z == 0.5).all()
    for i in range(nb):
        api.lib.lbfgs_persist_clear(C.byref(pts[i]))
