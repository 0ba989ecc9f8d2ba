"""Federated stochastic calibration, one interval call per rank (dirac_b200_stochastic_federated_interval;
sagecal-mpi -N -M -w -A, the stochastic slave sagecal_stochastic_slave.cpp:650-881 and the master's
exchange sagecal_stochastic_master.cpp:334-354), no beam.  One rank: the call against the slave's loop
restated with the reference's bfgsfit_minibatch_consensus, update_global_z_multi and projectback
(Nf = 1), and against the same loop made of this library's reference-named calls; with alpha = 0, no
flagged band and no uv cut, against dirac_b200_stochastic_consensus_interval.  Two ranks under
torch.distributed.run (tests/federated_check.py) against a one-process emulation of the two slaves and
the master.  Also a band without channels, use_global, a hybrid sky (Mt > M) and the refusals.

The tests that compare with the reference call it first and ask for the product library afterwards,
so that the reference's answers can be recorded."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from util import relerr
from test_gpu_stochastic import FREQS5, FREQS9, LBFGS, NMB, RERUN_TOL, TMB, bands, problem, uv_cut
from test_gpu_stochastic_consensus import POLYTYPE, band_freqs, bz

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
NADMM, NEPOCHS, ADMM_RHO, ALPHA = 3, 1, 5.0, 2.0
RES_RATIO, CLM_DBL_MAX = 1.5, 1e12
KW = dict(ccid=1, rho=1e-9, **LBFGS)
vp = C.c_void_p


def _p(a):
    return a.ctypes.data_as(vp)


class Setup:
    def __init__(self, freqs, nsolbw, Npoly, B, Bi, rhok, alphak, uvmin):
        self.freqs, self.nsolbw, self.Npoly = freqs, nsolbw, Npoly
        self.B, self.Bi, self.rhok, self.alphak, self.uvmin = B, Bi, rhok, alphak, uvmin


def fed_setup(lib, world, freqs=FREQS5, nsolbw=2, Npoly=2, alpha=ALPHA, cut=True):
    """the shared problem (every rank observes the same band, as one MS each); B from
    dirac_b200_consensus_basis over the bands' mean frequencies, Bi from the fed inverse"""
    from sagecal_b200 import consensus as cons
    b, sky, ivls = problem(freqs)
    B = cons.basis(lib, band_freqs(freqs, nsolbw), float(np.mean(freqs)), Npoly, POLYTYPE)
    rhok = np.full((nsolbw, sky.Mt), ADMM_RHO)
    alphak = np.full(sky.Mt, alpha)
    Bi = lib.consensus_prod_inverse_fed(B, rhok, alphak)
    uvmin = uv_cut(b.pr, freqs) if cut else 0.0
    return b, sky, ivls, Setup(freqs, nsolbw, Npoly, B, Bi, rhok, alphak, uvmin)


def run_call(api, b, sky, ivl, s, rank=0, world=1, allreduce=None, use_global=0):
    """one interval call: (residuals, res_00, res_01, pfreq, Z, res_0, res_1, fband)"""
    pr = b.pr
    pts = api.persist_init_array(s.nsolbw, NMB, b.m, 8 * ivl.R, LBFGS["lbfgs_m"])
    pfreq = np.tile(pr.pp0, (s.nsolbw, 1))
    Z = np.zeros((sky.Mt, s.Npoly, 8 * pr.N))
    xo = ivl.x.copy()
    rv, r0, r1, q0, q1, fb = api.stochastic_federated_interval(
        ivl.u, ivl.v, ivl.w, xo, pr.N, pr.Nbase, TMB, ivl.barr(), sky, s.freqs,
        pr.fdelta * len(s.freqs), pts, pfreq, s.nsolbw, NEPOCHS, NADMM, s.B, s.Bi, s.rhok, s.alphak, Z,
        use_global=use_global, rank=rank, world=world, allreduce=allreduce, uvmin=s.uvmin, **KW)
    assert rv == 0
    for i in range(s.nsolbw):
        api.lib.lbfgs_persist_clear(C.byref(pts[i]))
    return xo, r0, r1, pfreq, Z, np.array(q0), np.array(q1), fb.copy()


def api_step(api, N):
    def step(ad, r00, r01, J, B, Bi, rhok, alphak, Zavg, X, Y, Z):
        rv, q0, q1, fb = api.federated_bands_update(N, ad, r00, r01, J, B, Bi, rhok, alphak, Zavg, X,
                                                    Y, Z)
        assert rv == 0
        return q0, q1, fb
    return step


def ref_step(ref, N):
    """sagecal_stochastic_slave.cpp:731-852 in numpy around the reference's update_global_z_multi"""
    def step(ad, r00, r01, J, B, Bi, rhok, alphak, Zavg, X, Y, Z):
        nsolbw, Npoly = B.shape
        Mt = Bi.shape[0]
        with np.errstate(invalid="ignore"):
            q0, q1 = np.sum(r00) / nsolbw, np.sum(r01) / nsolbw
            resband = np.where((r00 > 0.0) & (r01 > 0.0), r01, CLM_DBL_MAX)
            fb = (resband > RES_RATIO * q1).astype(np.int32)
        rho_i = np.repeat(rhok, 8 * N, axis=1)
        for b in range(nsolbw):
            if not fb[b]:
                Y[b] += rho_i[b] * J[b]
        z = B[0][:, None] * Y[0][None, :] if not fb[0] else np.zeros((Npoly, Y.shape[1]))
        for b in range(1, nsolbw):
            if not fb[b]:
                z += B[b][:, None] * Y[b][None, :]
        z = z.reshape(Npoly, Mt, 8 * N)
        if ad > 0:
            for ci in range(Mt):
                for p in range(Npoly):
                    z[p, ci] += alphak[ci] * Zavg[ci, p]
                    z[p, ci] += -1.0 * X[ci, p]
        z = np.ascontiguousarray(z)
        ref.lib.update_global_z_multi.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp, vp, C.c_int]
        ref.lib.update_global_z_multi(_p(Z), N, Mt, Npoly, _p(z), _p(np.ascontiguousarray(Bi)), 4)
        for b in range(nsolbw):
            if not fb[b]:
                Y[b] -= rho_i[b] * bz(Z, B[b])
        return q0, q1, fb
    return step


def api_average(api):
    def avg(Zall, niter):
        assert api.manifold_projectback(Zall, niter, 0) == 0
    return avg


def ref_average(ref):
    def avg(Zall, niter):
        Nf, Mt, n8 = Zall.shape
        ref.lib.calculate_manifold_average_projectback.argtypes = [C.c_int] * 3 + [vp] + [C.c_int] * 3
        ref.lib.calculate_manifold_average_projectback(n8 // 8, Mt, Nf, _p(Zall), niter, 0, 1)
    return avg


def emulate(lib, step, average, b, sky, ivls, s, use_global=0):
    """the slaves of sagecal_stochastic_slave.cpp:650-881, one per interval of `ivls` (one MS each),
    and the master's exchange, in one process through the reference-named calls of `lib`; the uv cut
    holds in every pass (the slave reloads the flags and predicts again, :675-723).  One tuple per
    slave, as run_call returns"""
    pr = b.pr
    S, nsolbw, Npoly, Mt = len(ivls), s.nsolbw, s.Npoly, sky.Mt
    nchan = len(s.freqs)
    bl = bands(nchan, nsolbw)
    R, M = ivls[0].R, sky.M
    L = Mt * Npoly * 8 * pr.N
    st = []
    for ivl in ivls:
        barrs = [ivl.barr(mb) for mb in range(NMB)]
        coh = [lib.precalculate_coherencies_multifreq(ivl.u[mb], ivl.v[mb], ivl.w[mb], pr.N, R, barrs[mb],
                                                      sky, s.freqs, pr.fdelta * nchan, uvmin=s.uvmin)
               for mb in range(NMB)]
        st.append(dict(ivl=ivl, barrs=barrs, coh=coh, pfreq=np.tile(pr.pp0, (nsolbw, 1)),
                       pts=[lib.persist_init(NMB, b.m, 8 * R, LBFGS["lbfgs_m"]) for _ in range(nsolbw)],
                       Z=np.zeros((Mt, Npoly, 8 * pr.N)), Y=np.zeros((nsolbw, b.m)),
                       X=np.zeros((Mt, Npoly, 8 * pr.N)), Zavg=np.zeros((Mt, Npoly, 8 * pr.N)),
                       r0=np.zeros((NADMM, NEPOCHS, NMB, nsolbw)),
                       r1=np.zeros((NADMM, NEPOCHS, NMB, nsolbw))))
    for ad in range(NADMM):
        for sl in st:
            ivl = sl["ivl"]
            for ep in range(NEPOCHS):
                for mb in range(NMB):
                    for bi, (c0, nc) in enumerate(bl):
                        z = bz(sl["Z"], s.B[bi])
                        coh = np.ascontiguousarray(sl["coh"][mb][c0 * R * M * 4:(c0 + nc) * R * M * 4])
                        x = np.ascontiguousarray(ivl.x[mb, c0:c0 + nc]).reshape(-1)
                        sl["r0"][ad, ep, mb, bi], sl["r1"][ad, ep, mb, bi] = lib.bfgsfit_minibatch(
                            ivl.u[mb], ivl.v[mb], ivl.w[mb], x, pr.N, pr.Nbase, TMB, sl["barrs"][mb],
                            sky, coh, sl["pfreq"][bi], s.freqs[c0:c0 + nc], sl["pts"][bi],
                            fdelta=pr.fdelta * nc, nmb=mb, totalmb=NMB, Y=sl["Y"][bi], Z=z,
                            rho=np.ascontiguousarray(s.rhok[bi]), **LBFGS)
                    sl["q"] = step(ad, sl["r0"][ad, ep, mb], sl["r1"][ad, ep, mb], sl["pfreq"], s.B, s.Bi,
                                   s.rhok, s.alphak, sl["Zavg"], sl["X"], sl["Y"], sl["Z"])
        Zall = np.ascontiguousarray(np.stack([sl["Z"].reshape(Mt, -1) for sl in st]))
        average(Zall, 10 if ad == 0 else 2)
        for f, sl in enumerate(st):
            sl["Zavg"] = Zall[f].reshape(Mt, Npoly, 8 * pr.N).copy()
            for k in range(Mt):
                sl["X"][k] += s.alphak[k] * (sl["Z"][k] - sl["Zavg"][k])
    out = []
    for sl in st:
        ivl = sl["ivl"]
        if use_global:
            for bi in range(nsolbw):
                sl["pfreq"][bi] = bz(sl["Z"], s.B[bi])
        res = ivl.x.copy()
        for mb in range(NMB):
            for bi, (c0, nc) in enumerate(bl):
                if nc == 0:
                    continue
                xr = np.ascontiguousarray(res[mb, c0:c0 + nc])
                assert lib.calculate_residuals_multifreq(
                    ivl.u[mb], ivl.v[mb], ivl.w[mb], sl["pfreq"][bi], xr.reshape(-1), pr.N, pr.Nbase,
                    TMB, ivl.barr(mb), sky, s.freqs[c0:c0 + nc], pr.fdelta * nc, ccid=KW["ccid"],
                    rho=KW["rho"]) == 0
                res[mb, c0:c0 + nc] = xr
        for pt in sl["pts"]:
            lib.persist_clear(pt)
        q0, q1, fb = sl["q"]
        out.append((res, sl["r0"], sl["r1"], sl["pfreq"], sl["Z"], np.array(q0), np.array(q1),
                    np.array(fb)))
    return out


def _costs_close(g, w, tol):
    fin = np.isfinite(w)
    assert np.array_equal(fin, np.isfinite(g))
    if fin.any():
        assert np.max(np.abs(g[fin] - w[fin]) / np.abs(w[fin])) <= tol


def assert_close(g, w, tol_r0, tol_r1, tol_p, tol_x):
    xg, g0, g1, pg, Zg, q0g, q1g, fbg = g
    xw, w0, w1, pw, Zw, q0w, q1w, fbw = w
    _costs_close(g0, w0, tol_r0)
    _costs_close(g1, w1, tol_r1)
    _costs_close(np.atleast_1d(q1g), np.atleast_1d(q1w), tol_r1)
    assert np.array_equal(fbg, fbw), (fbg, fbw)
    for bi in range(len(pw)):
        assert relerr(pg[bi], pw[bi]) <= tol_p, (bi, relerr(pg[bi], pw[bi]))
    assert relerr(Zg, Zw) <= tol_p, relerr(Zg, Zw)
    assert np.max(np.abs(xg - xw)) <= tol_x * np.max(np.abs(xw)), np.max(np.abs(xg - xw))


def test_one_rank_against_the_reference(ref, request):
    """world 1 on the hybrid sky (3 clusters, 4 chunks), with the uv cut and alpha 2: the call against
    the slave's loop on the reference's calls and the reference's projectback with Nf = 1; the bounds
    of the consensus interval against its reference loop"""
    api = request.getfixturevalue("api")
    b, sky, ivls, s = fed_setup(api, 1)
    assert sky.Mt > sky.M
    want = emulate(ref, ref_step(ref, b.pr.N), ref_average(ref), b, sky, ivls[:1], s)[0]
    got = run_call(api, b, sky, ivls[0], s)
    assert_close(got, want, 1e-9, 1e-7, 1e-6, 1e-6)


def test_one_rank_equals_the_library_loop(api):
    """the same loop on this library's reference-named calls: as close as two runs of one of them"""
    b, sky, ivls, s = fed_setup(api, 1)
    want = emulate(api, api_step(api, b.pr.N), api_average(api), b, sky, ivls[:1], s)[0]
    got = run_call(api, b, sky, ivls[0], s)
    assert np.abs(got[4]).max() > 0
    assert_close(got, want, RERUN_TOL, RERUN_TOL, RERUN_TOL, RERUN_TOL)


def test_zero_alpha_is_the_consensus_interval(api):
    """alpha 0, no uv cut, no flagged band: the federated term is zero and the fed inverse is the plain
    one, so the call is dirac_b200_stochastic_consensus_interval"""
    from sagecal_b200 import consensus as cons
    from test_gpu_stochastic_consensus import run_interval
    b, sky, ivls, s = fed_setup(api, 1, alpha=0.0, cut=False)
    Bi = cons.prod_inverse(api, s.B, s.rhok)
    assert relerr(Bi, s.Bi) < 1e-12
    got = run_call(api, b, sky, ivls[0], s)
    want = run_interval(api, b, sky, ivls[:1], FREQS5, 2, s.B, Bi, s.rhok, 0.0, nadmm=NADMM,
                        nepochs=NEPOCHS, **KW)[0]
    assert not got[7].any() and not want[7].any()
    _costs_close(got[1], want[1].reshape(got[1].shape), RERUN_TOL)
    _costs_close(got[2], want[2].reshape(got[2].shape), RERUN_TOL)
    assert relerr(got[3], want[3]) <= RERUN_TOL and relerr(got[4], want[4]) <= RERUN_TOL
    assert np.max(np.abs(got[0] - want[0])) <= RERUN_TOL * np.max(np.abs(want[0]))


def test_band_without_channels_and_use_global(api):
    """9 channels in 4 bands (3, 3, 3, 0), use_global: against the library loop; every band's Jones is
    its B_b Z"""
    b, sky, ivls, s = fed_setup(api, 1, freqs=FREQS9, nsolbw=4)
    want = emulate(api, api_step(api, b.pr.N), api_average(api), b, sky, ivls[:1], s, use_global=1)[0]
    got = run_call(api, b, sky, ivls[0], s, use_global=1)
    assert not np.isfinite(got[1][..., 3]).any()      # consensus terms x 1/0
    assert_close(got, want, RERUN_TOL, RERUN_TOL, RERUN_TOL, RERUN_TOL)
    for bi in range(4):
        assert np.array_equal(got[3][bi], bz(got[4], s.B[bi]))


def _two_ranks(tmp_path, backend, port):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(HERE, "federated_check.py"), backend, str(tmp_path)]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    print(out.stdout[-3000:], out.stderr[-3000:])
    assert out.returncode == 0 and out.stdout.count("FEDERATED_CHECK OK") == 2
    return [list(np.load(os.path.join(str(tmp_path), "rank%d.npz" % r)).values()) for r in range(2)]


@pytest.mark.parametrize("backend", ["gloo", "nccl"])
def test_two_ranks_equal_the_emulated_slaves_and_master(api, tmp_path, backend):
    """two ranks, one MS each, exchanging through the gloo callback on one device or NCCL on two:
    every rank's outputs equal the one-process emulation of the two slaves and the master"""
    import torch
    if backend == "nccl" and torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    got = _two_ranks(tmp_path, backend, 29641 if backend == "gloo" else 29643)
    b, sky, ivls, s = fed_setup(api, 2)
    want = emulate(api, api_step(api, b.pr.N), api_average(api), b, sky, ivls, s)
    assert relerr(want[0][4], want[1][4]) > 1e-6       # the ranks' solutions differ
    for r in range(2):
        assert_close(tuple(got[r]), want[r], RERUN_TOL, RERUN_TOL, RERUN_TOL, RERUN_TOL)


@pytest.mark.parametrize("nsolbw,nadmm,Npoly,rank,world", [
    (6, 2, 2, 0, 1), (2, 0, 2, 0, 1), (2, 2, 0, 0, 1), (2, 2, 2, 1, 1), (2, 2, 2, -1, 2),
    (2, 2, 2, 0, 2)], ids=["more-bands-than-channels", "no-admm", "no-poly", "rank-is-world",
                           "negative-rank", "no-communicator"])
def test_refusals(api, nsolbw, nadmm, Npoly, rank, world):
    """-1 before any work, no output touched (world 2 with no callback and no communicator)"""
    api.lib.dirac_b200_nccl_finalize()
    b, sky, ivls = problem(FREQS5)
    pr = b.pr
    ivl = ivls[0]
    nb = max(nsolbw, 1)
    pts = api.persist_init_array(nb, NMB, b.m, 8 * ivl.R, 5)
    pfreq = np.tile(pr.pp0, (nb, 1)) + 0.25
    xo = ivl.x.copy()
    P = max(Npoly, 1)
    Z = np.full((sky.Mt, P, 8 * pr.N), 0.5)
    rv, r0, r1, q0, q1, fb = api.stochastic_federated_interval(
        ivl.u, ivl.v, ivl.w, xo, pr.N, pr.Nbase, TMB, ivl.barr(), sky, FREQS5, pr.fdelta * 5, pts,
        pfreq, nsolbw, 1, nadmm, np.ones((nb, max(Npoly, 0))), np.ones((sky.Mt, P, P)),
        np.ones((nb, sky.Mt)), np.ones(sky.Mt), Z, rank=rank, world=world, **LBFGS)
    assert rv == -1
    assert not r0.any() and not r1.any() and q0 == 0.0 and q1 == 0.0 and not fb.any()
    assert np.array_equal(xo, ivl.x)
    assert np.array_equal(pfreq, np.tile(pr.pp0, (nb, 1)) + 0.25)
    assert (Z == 0.5).all()
    for i in range(nb):
        api.lib.lbfgs_persist_clear(C.byref(pts[i]))
