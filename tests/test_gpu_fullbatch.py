"""Full-batch calibration of one tile in one call (dirac_b200_fullbatch_tile(_withbeam); sagecal's default
mode, fullbatch_mode.cpp:371-530) against the driver's chain of reference-named calls:
precalculate_coherencies(_withbeam) -> sagefit_visibilities -> calculate_residuals_multifreq(_withbeam),
or with -b 1 the per-channel loop of precalculate_coherencies, bfgsfit_visibilities and
calculate_residuals.  Against this library's own chain (the same kernels in the same order), against the
compiled reference at a small shape, with array and wide-band full beams, sharded over two ranks, and the
refusals.

The LBFGS gradient kernels sum with atomics, so two runs of the same fit differ in the last bits and a
few iterations amplify that (RERUN_TOL, as test_gpu_channels.py measured it).  Everything that no atomic
touches is compared bit for bit: the flags and the cost before the fit.

The tests that compare with the reference call it first and ask for the product library afterwards,
so that the reference's answers can be recorded on a machine without a GPU."""
import copy
import os
import subprocess
import sys

import numpy as np
import pytest

from util import relerr, small_problem
from sagecal_b200.dirac_api import BeamSetup, SkyModel, barr_to_numpy
from test_gpu_beam import beam_problem
from test_gpu_channels import channel_problem, NO_CCID, RERUN_TOL, JONES_TOL, FREQS

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FREQ0 = float(np.mean(FREQS))
FIT = dict(max_emiter=3, max_iter=2, max_lbfgs=8, lbfgs_m=5)


def tile_problem(nchunk=None, seed=41):
    """test_gpu_channels.py's 4-channel problem (9 stations, 3 clusters with ids -1, 1, 2, 8 timeslots,
    spectral indices); x is the channel average of the data"""
    b, sky, xo = channel_problem(nchunk, seed=seed)
    return b, sky, np.ascontiguousarray(xo.mean(axis=0)), np.ascontiguousarray(xo)


def uv_limits(pr):
    uvd = np.sqrt(pr.u * pr.u + pr.v * pr.v)[pr.flag == 0] * FREQ0
    return float(np.quantile(uvd, 0.1)), float(np.quantile(uvd, 0.9))


def chain(lib, b, sky, x, xo, freqs, p0, beam=None, uvmin=0.0, uvmax=1e9, do_chan=0, ccid=NO_CCID,
          rho=1e-9, phase_only=0, solver_mode=1, **fit):
    """the driver's tile (fullbatch_mode.cpp:371-530) through the reference-named calls of `lib`"""
    pr = b.pr
    barr = b.fresh_barr()
    x, xo, p = x.copy(), xo.copy(), p0.copy()
    n = len(freqs)
    deltaf = pr.fdelta * n
    if beam is None:
        coh = lib.precalculate_coherencies(pr.u, pr.v, pr.w, pr.N, pr.Nbase1, barr, sky, FREQ0, deltaf,
                                           uvmin=uvmin, uvmax=uvmax)
    else:
        coh = lib.precalculate_coherencies_withbeam(pr.u, pr.v, pr.w, pr.N, pr.Nbase1, barr, sky, FREQ0,
                                                    deltaf, beam, uvmin=uvmin, uvmax=uvmax)
    fk = dict(fit, max_lbfgs=0 if do_chan else fit["max_lbfgs"])
    _, nu, r0, r1 = lib.sagefit_visibilities(pr.u, pr.v, pr.w, x, pr.N, pr.Nbase, pr.tilesz, barr, sky,
                                             coh, p, freq0=FREQ0, fdelta=deltaf, solver_mode=solver_mode,
                                             **fk)
    r00 = r01 = None
    if do_chan:   # fullbatch_mode.cpp:464-497: no beam, no phase_only
        r00, r01 = np.zeros(n), np.zeros(n)
        pf = p
        for ci, f in enumerate(freqs):
            pf = p.copy()
            cohc = lib.precalculate_coherencies(pr.u, pr.v, pr.w, pr.N, pr.Nbase1, barr, sky, f,
                                                deltaf / n, uvmin=uvmin, uvmax=uvmax)
            xf = xo[ci].copy()
            _, r00[ci], r01[ci] = lib.bfgsfit_visibilities(
                pr.u, pr.v, pr.w, xf, pr.N, pr.Nbase, pr.tilesz, barr, sky, cohc, pf, freq0=f,
                fdelta=deltaf / n, max_lbfgs=fit["max_lbfgs"], lbfgs_m=fit["lbfgs_m"],
                solver_mode=solver_mode, mean_nu=nu)
            assert lib.calculate_residuals(pr.u, pr.v, pr.w, pf, xo[ci], pr.N, pr.Nbase, pr.tilesz, barr,
                                           sky, f, deltaf / n, ccid=ccid, rho=rho) == 0
        p = pf
    elif beam is None:
        assert lib.calculate_residuals_multifreq(pr.u, pr.v, pr.w, p, xo, pr.N, pr.Nbase, pr.tilesz, barr,
                                                 sky, freqs, deltaf, ccid=ccid, rho=rho,
                                                 phase_only=phase_only) == 0
    else:
        assert lib.calculate_residuals_multifreq_withbeam(pr.u, pr.v, pr.w, p, xo, pr.N, pr.Nbase,
                                                          pr.tilesz, barr, sky, freqs, deltaf, beam,
                                                          ccid=ccid, rho=rho, phase_only=phase_only) == 0
    return dict(x=x, xo=xo, p=p, flag=barr_to_numpy(barr, pr.Nbase1)[2], nu=nu, r0=r0, r1=r1, r00=r00,
                r01=r01)


def tile(api, b, sky, x, xo, freqs, p0, beam=None, do_chan=0, **kw):
    """one dirac_b200_fullbatch_tile(_withbeam) call"""
    pr = b.pr
    barr = b.fresh_barr()
    x, xo, p = x.copy(), xo.copy(), p0.copy()
    rv, nu, r0, r1, r00, r01 = api.fullbatch_tile(pr.u, pr.v, pr.w, x, xo, pr.N, pr.Nbase, pr.tilesz,
                                                  barr, sky, FREQ0, pr.fdelta * len(freqs), freqs, p,
                                                  beam=beam, do_chan=do_chan, **kw)
    assert rv == 0
    return dict(x=x, xo=xo, p=p, flag=barr_to_numpy(barr, pr.Nbase1)[2], nu=nu, r0=r0, r1=r1,
                r00=r00 if do_chan else None, r01=r01 if do_chan else None)


def diffs(got, want):
    """largest differences, relative to the largest value of the answer"""
    out = {k: relerr(got[k], want[k]) for k in ("x", "xo", "p")}
    for k in ("nu", "r0", "r1"):
        out[k] = abs(got[k] - want[k]) / abs(want[k])
    if want["r00"] is not None:
        out["r00"] = relerr(got["r00"], want["r00"])
        out["r01"] = relerr(got["r01"], want["r01"])
    print("DIFF", {k: float("%.3g" % v) for k, v in out.items()})
    return out


def assert_same(got, want, tol):
    assert np.array_equal(got["flag"], want["flag"])
    d = diffs(got, want)
    assert d["r0"] <= 1e-14, d
    for k, v in d.items():
        assert v <= tol, (k, d)


# (solver_mode, nchunk, ccid, phase_only, uv cut)
CASES = [(1, None, NO_CCID, 0, False), (3, [1, 3, 2], 1, 0, False), (5, [2, 1, 3], 2, 1, False),
         (1, [1, 3, 2], 1, 1, True)]
IDS = ["lm", "oslm-robust-hybrid-ccid", "rtr-robust-hybrid-phase_only", "lm-uvcut-phase_only"]


@pytest.mark.parametrize("mode,nchunk,ccid,phase_only,cut", CASES, ids=IDS)
def test_tile_equals_the_chain(api, mode, nchunk, ccid, phase_only, cut):
    """the same kernels in the same order: outputs as close as two runs of the chain, the flags and the
    cost before the fit bit for bit; the chain uploads the sky twice and moves the coherencies down and
    up, the tile uploads the sky once and moves no coherency"""
    b, sky, x, xo = tile_problem(nchunk)
    pr = b.pr
    uvmin, uvmax = uv_limits(pr) if cut else (0.0, 1e9)
    kw = dict(uvmin=uvmin, uvmax=uvmax, ccid=ccid, rho=1e-9, phase_only=phase_only, solver_mode=mode,
              **FIT)
    api.transfer_stats(reset=True)
    want = chain(api, b, sky, x, xo, FREQS, pr.pp0, **kw)
    assert api.transfer_stats(reset=True) == (2, 2 * pr.M * pr.Nbase1 * 64)
    got = tile(api, b, sky, x, xo, FREQS, pr.pp0, **kw)
    assert api.transfer_stats(reset=True) == (1, 0)
    assert want["r1"] < want["r0"]
    assert_same(got, want, RERUN_TOL)
    if cut:
        assert (want["flag"] == 2).sum() > 0
    if ccid != NO_CCID:   # the correction is applied
        plain = chain(api, b, sky, x, xo, FREQS, pr.pp0, **dict(kw, ccid=NO_CCID))
        assert relerr(plain["xo"], want["xo"]) > 1e-3


def test_tile_against_the_reference(ref, request):
    """the compiled reference's chain at a small shape: Jones within 1e-5, residuals likewise"""
    b, sky, x, xo = tile_problem()
    pr = b.pr
    kw = dict(ccid=1, rho=1e-9, solver_mode=1, **FIT)
    want = chain(ref, b, sky, x, xo, FREQS, pr.pp0, **kw)
    api = request.getfixturevalue("api")
    got = tile(api, b, sky, x, xo, FREQS, pr.pp0, **kw)
    assert np.array_equal(got["flag"], want["flag"])
    d = diffs(got, want)
    assert d["r0"] < 1e-10 and d["r1"] < 1e-5, d
    assert d["p"] < JONES_TOL and d["x"] < 1e-5 and d["xo"] < 1e-5, d


BEAM_CASES = [("array", True, 0), ("full_wb", False, 0), ("array", True, 1)]
BEAM_IDS = ["array-tile", "full_wb-single", "array-tile-do_chan"]


@pytest.mark.parametrize("mode,tiled,do_chan", BEAM_CASES, ids=BEAM_IDS)
def test_withbeam_equals_the_chain(ref, request, mode, tiled, do_chan):
    """precalculate_coherencies_withbeam_gpu -> sagefit_visibilities ->
    calculate_residuals_multifreq_withbeam_gpu, with coefficient set c in channel c for the wide-band
    element beam; with do_chan the driver's -b 1 loop, which predicts without the beam"""
    freqs = FREQS
    b, sky, beam = beam_problem(ref, mode, tiled, seed=37, freqs=freqs, tilesz=6)
    api = request.getfixturevalue("api")
    pr = b.pr
    rng = np.random.default_rng(5)
    xo = np.ascontiguousarray(np.stack([pr.x + rng.normal(0, 0.02, pr.x.shape) for _ in freqs]))
    x = np.ascontiguousarray(xo.mean(axis=0))
    kw = dict(ccid=1, rho=1e-9, phase_only=0, solver_mode=1, do_chan=do_chan, uvmin=30.0, uvmax=1e5,
              **FIT)
    want = chain(api, b, sky, x, xo, freqs, pr.pp0, beam=beam, **kw)
    got = tile(api, b, sky, x, xo, freqs, pr.pp0, beam=beam, **kw)
    assert_same(got, want, RERUN_TOL)
    plain = tile(api, b, sky, x, xo, freqs, pr.pp0, **kw)   # the beam matters
    assert relerr(plain["p"], got["p"]) > 1e-4


def test_do_chan_equals_the_loop_and_bfgsfit_channels(api):
    """-b 1: the fit with max_lbfgs 0, then per channel coherencies, LBFGS and the residual on the same
    resident problem; against the driver's reference-named loop and dirac_b200_bfgsfit_channels"""
    b, sky, x, xo = tile_problem([1, 3, 2])
    pr = b.pr
    uvmin, uvmax = uv_limits(pr)
    kw = dict(ccid=2, rho=1e-9, solver_mode=1, uvmin=uvmin, uvmax=uvmax, **FIT)
    api.transfer_stats(reset=True)
    got = tile(api, b, sky, x, xo, FREQS, pr.pp0, do_chan=1, **kw)
    assert api.transfer_stats(reset=True) == (1, 0)
    want = chain(api, b, sky, x, xo, FREQS, pr.pp0, do_chan=1, **kw)
    assert_same(got, want, RERUN_TOL)
    assert relerr(want["p"], chain(api, b, sky, x, xo, FREQS, pr.pp0, **kw)["p"]) > 1e-6
    # dirac_b200_bfgsfit_channels from the fit's Jones, flags and mean_nu
    fit = chain(api, b, sky, x, xo, FREQS, pr.pp0, **dict(kw, max_lbfgs=0))
    from sagecal_b200.dirac_api import make_barr
    barr = make_barr(pr.sta1, pr.sta2, fit["flag"])
    xc, p = xo.copy(), fit["p"].copy()
    rv, r00, r01, _ = api.bfgsfit_channels(pr.u, pr.v, pr.w, xc.reshape(-1), pr.N, pr.Nbase, pr.tilesz,
                                           barr, sky, FREQS, pr.fdelta, p, uvmin=uvmin, uvmax=uvmax,
                                           max_lbfgs=FIT["max_lbfgs"], lbfgs_m=FIT["lbfgs_m"],
                                           solver_mode=1, mean_nu=fit["nu"], ccid=2, rho=1e-9,
                                           keep_pfreq=False)
    assert rv == 0
    assert np.array_equal(barr_to_numpy(barr, pr.Nbase1)[2], got["flag"])
    assert relerr(got["p"], p) <= RERUN_TOL and relerr(got["xo"], xc) <= RERUN_TOL
    assert relerr(got["r00"], r00) <= 1e-14 and relerr(got["r01"], r01) <= RERUN_TOL


def test_world_one_with_a_callback_is_the_one_gpu_call(api):
    """world 1 never calls the exchange: a callback changes nothing"""
    from sagecal_b200.dist import ALLREDUCE_FN
    calls = []
    cb = ALLREDUCE_FN(lambda *a: calls.append(a))
    b, sky, x, xo = tile_problem()
    pr = b.pr
    kw = dict(ccid=1, rho=1e-9, solver_mode=1, **FIT)
    one = tile(api, b, sky, x, xo, FREQS, pr.pp0, **kw)
    cbk = tile(api, b, sky, x, xo, FREQS, pr.pp0, rank=0, world=1, allreduce=cb, **kw)
    assert not calls
    assert_same(cbk, one, RERUN_TOL)


def _refusal_args(case):
    b, sky, x, xo = tile_problem()
    kw, freqs, beam = {}, FREQS, None
    if case == "no-channels":
        freqs, xo = FREQS[:0], xo[:0]
    elif case == "rank-is-world":
        kw = dict(rank=1, world=1)
    elif case == "world-above-M":
        kw = dict(rank=0, world=4)
    elif case == "empty-last-block":   # 4 clusters over 3 ranks: 2, 2 and none
        b = small_problem(N=9, M=4, tilesz=8, seed=41)
        sky = SkyModel(b.pr.clusters, b.pr.N)
        x = np.ascontiguousarray(b.pr.x.copy())
        xo = np.ascontiguousarray(np.stack([x] * len(freqs)))
        kw = dict(rank=0, world=3, allreduce="cb")
    elif case == "no-communicator":
        kw = dict(rank=0, world=2)
    elif case == "do_chan-sharded":
        kw = dict(rank=0, world=2, allreduce="cb", do_chan=1)
    elif case == "bad-beam":
        pr = b.pr
        beam = BeamSetup(1, 1.2, 1.0, 1.2, 1.0, FREQ0, np.zeros(pr.N), np.zeros(pr.N),
                         np.zeros(pr.tilesz), [np.zeros((4, 3))] * pr.N, None, 7)
    return b, sky, x, xo, freqs, beam, kw


@pytest.mark.parametrize("case", ["no-channels", "rank-is-world", "world-above-M", "empty-last-block",
                                  "no-communicator", "do_chan-sharded", "bad-beam", "too-large"])
def test_refusals(api, case, capfd):
    """-1 before any device work, no output touched"""
    from sagecal_b200.dist import ALLREDUCE_FN
    cb = ALLREDUCE_FN(lambda *a: None)
    b, sky, x, xo, freqs, beam, kw = _refusal_args(case)
    if kw.get("allreduce") == "cb":
        kw["allreduce"] = cb
    pr = b.pr
    barr = b.fresh_barr()
    tilesz = pr.tilesz
    if case == "too-large":   # 10^8 timeslots: terabytes of coherencies; nothing is read before the check
        tilesz = 10 ** 8
    x1, xo1, p1 = x.copy(), xo.copy(), pr.pp0.copy()
    rv, nu, r0, r1, _, _ = api.fullbatch_tile(pr.u, pr.v, pr.w, x1, xo1, pr.N, pr.Nbase, tilesz, barr,
                                              sky, FREQ0, pr.fdelta * max(len(freqs), 1), freqs, p1,
                                              beam=beam, **kw)
    assert rv == -1
    assert "dirac_b200_fullbatch_tile" in capfd.readouterr().err
    assert np.array_equal(x1, x) and np.array_equal(xo1, xo) and np.array_equal(p1, pr.pp0)
    assert np.array_equal(barr_to_numpy(barr, pr.Nbase1)[2], pr.flag)
    assert (nu, r0, r1) == (0.0, 0.0, 0.0)


# ---- two ranks ---------------------------------------------------------------------------------------

def sharded_setup():
    """the problem every rank solves: 4 clusters (two per rank, the second rank's with a hybrid
    chunk), the correction by a cluster of rank 0, a uv cut"""
    b = small_problem(N=9, M=4, tilesz=8, seed=47, kmean=1.0, gaussian_frac=0.3, nchunk=[1, 2, 1, 3],
                      flag_frac=0.05)
    pr = b.pr
    for k, cl in enumerate(pr.clusters):
        cl["id"] = (-1, 1, 2, 3)[k]
    sky = SkyModel(pr.clusters, pr.N)
    rng = np.random.default_rng(48)
    xo = np.ascontiguousarray(np.stack([pr.x + rng.normal(0, 0.02, pr.x.shape) for _ in FREQS]))
    x = np.ascontiguousarray(xo.mean(axis=0))
    kw = dict(ccid=1, rho=1e-9, phase_only=1, solver_mode=1, uvmin=uv_limits(pr)[0], uvmax=1e9, **FIT)
    return b, sky, x, xo, kw


def emulate_rank(api, rank, world, b, sky, x, kw):
    """this rank's fit through the existing sharded path: dirac_b200_create_shard, the coherencies by
    dirac_b200_precalculate, dirac_b200_sagefit"""
    from sagecal_b200.dist import ShardedProblem
    pr = copy.copy(b.pr)
    pr.coh, pr.x = None, x
    barr = b.fresh_barr()
    sp = ShardedProblem(api, pr, barr, rank, world, use_callback=True)
    sp.precalculate(pr.u, pr.v, pr.w, FREQ0, pr.fdelta * len(FREQS), kw["uvmin"], kw["uvmax"])
    p, xs = pr.pp0.copy(), np.zeros_like(x)
    fit = {k: kw[k] for k in ("max_emiter", "max_iter", "max_lbfgs", "lbfgs_m", "solver_mode")}
    rv, nu, r0, r1 = sp.sagefit(p, xs, **fit)
    sp.close()
    return p, xs, np.array([nu, r0, r1])


def _two_ranks(tmp_path, backend, port):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(HERE, "fullbatch_check.py"), backend, str(tmp_path)]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    print(out.stdout[-3000:], out.stderr[-3000:])
    assert out.returncode == 0 and out.stdout.count("FULLBATCH_CHECK OK") == 2
    return [dict(np.load(os.path.join(str(tmp_path), "rank%d.npz" % r))) for r in range(2)]


@pytest.mark.parametrize("backend", ["gloo", "nccl"])
def test_two_ranks(api, tmp_path, backend):
    """two ranks through the gloo callback on one device or NCCL on two: identical outputs on both ranks;
    the fit as the existing sharded path makes it; the residual equal to calculate_residuals_multifreq of
    the whole sky with the returned Jones up to the order of the sum over the ranks"""
    import torch
    if backend == "nccl" and torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    got = _two_ranks(tmp_path, backend, 29651 if backend == "gloo" else 29653)
    for k in ("x", "xo", "p", "flag", "stats"):
        assert np.array_equal(got[0][k], got[1][k]), k
    b, sky, x, xo, kw = sharded_setup()
    pr = b.pr
    g = got[0]
    assert (g["flag"] == 2).sum() > 0
    for r in range(2):   # the fit of the existing sharded path, run in the same processes
        assert relerr(g["p"], got[r]["emu_p"]) <= RERUN_TOL
        assert relerr(g["x"], got[r]["emu_x"]) <= RERUN_TOL
        assert abs(g["stats"][1] - got[r]["emu_stats"][1]) <= 1e-14 * g["stats"][1]
        assert abs(g["stats"][2] - got[r]["emu_stats"][2]) <= RERUN_TOL * g["stats"][2]
    want = xo.copy()
    assert api.calculate_residuals_multifreq(pr.u, pr.v, pr.w, g["p"].copy(), want, pr.N, pr.Nbase,
                                             pr.tilesz, b.fresh_barr(), sky, FREQS,
                                             pr.fdelta * len(FREQS), ccid=kw["ccid"], rho=kw["rho"],
                                             phase_only=kw["phase_only"]) == 0
    print("DIFF sharded residual", relerr(g["xo"], want))
    assert relerr(g["xo"], want) <= 1e-12
    assert relerr(want, xo) > 1e-3
