"""Influence-function diagnostics on the GPU (calculate_diagnostics_gpu, driver option -i 1): the
reference's own fp32 kernels (oracle/_ref/libinfluence_ref.so, built by oracle/influence.mk) against
the float64 restatement of tests/influence_ref.py, the library's fp64 kernels against the same through
the test hook dirac_b200_diagnostics_eval, and the whole call against the restatement."""
import ctypes as C
import os

import numpy as np
import pytest

import influence_ref as ir
from util import small_problem, perturbed_jones
from sagecal_b200.dirac_api import BeamSetup, SkyModel, make_barr

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libinfluence_ref.so")


def kernel_case(N=7, T=10, nchunk=1, flag_frac=0.15, dead=None, weak=False, seed=5):
    """random coherencies, residual, Jones and X on canonical rows; dead: a station whose rows are
    all flagged; weak: a cluster faint enough that its Hessian's diagonal falls below 1"""
    rng = np.random.default_rng(seed)
    pairs = [(p, q) for p in range(N) for q in range(p + 1, N)]
    Nbase = len(pairs)
    R = Nbase * T
    sta1 = np.tile([p for p, _ in pairs], T).astype(np.int32)
    sta2 = np.tile([q for _, q in pairs], T).astype(np.int32)
    flag = (rng.random(R) < flag_frac).astype(np.uint8)
    if dead is not None:
        flag[(sta1 == dead) | (sta2 == dead)] = 1
    cz = lambda *s: rng.normal(size=s) + 1j * rng.normal(size=s)
    scale = 0.05 if weak else 1.0
    coh = scale * cz(R, 4)
    res = cz(R, 4)
    p = np.tile(np.array([1, 0, 0, 0, 0, 0, 1, 0], dtype=np.float64), N * nchunk) \
        + 0.3 * rng.normal(size=8 * N * nchunk)
    X = cz(4 * N, Nbase)
    return dict(N=N, Nbase=Nbase, T=T, sta1=sta1, sta2=sta2, flag=flag, p=p, nchunk=nchunk,
                coh=coh, res=res, X=X)


def restated(c):
    a = (c["N"], c["Nbase"], c["T"], c["sta1"], c["sta2"])
    H = ir.hessian(*a, c["flag"], c["p"], c["nchunk"], c["coh"], c["res"])
    A = ir.adv(*a, c["flag"], c["p"], c["nchunk"], c["coh"])
    dR = ir.d_residuals(*a, c["p"], c["nchunk"], c["coh"], c["X"])
    return H, A, dR


def rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


CASES = [dict(nchunk=1), dict(nchunk=3), dict(nchunk=3, dead=2), dict(weak=True, nchunk=2)]
IDS = ["nchunk1", "nchunk3-boundary-in-timeslot", "flagged-station", "weak-cluster"]


def test_chunk_boundary_falls_inside_a_timeslot():
    c = kernel_case(nchunk=3)
    per = -(-c["Nbase"] * c["T"] // 3)
    assert per % c["Nbase"] != 0


@pytest.mark.parametrize("kw", CASES, ids=IDS)
def test_reference_kernels_match_the_restatement(kw):
    """the reference's cudakernel_hessian, cudakernel_d_solutions and cudakernel_d_residuals on the
    H100, on the same inputs cast to fp32, against the float64 restatement: 1e-4 of the max norm
    (fp32 with atomics)"""
    import torch
    if not os.path.exists(REF_SO):
        pytest.skip("oracle/_ref/libinfluence_ref.so not built")
    L = C.CDLL(REF_SO)
    c = kernel_case(**kw)
    N, Nbase, T = c["N"], c["Nbase"], c["T"]
    R = Nbase * T
    dev = torch.device("cuda")
    barr = np.zeros((R, 3), dtype=np.int32)
    barr[:, 0], barr[:, 1], barr[:, 2] = c["sta1"], c["sta2"], c["flag"]
    f32 = lambda z: torch.from_numpy(np.ascontiguousarray(z.view(np.float64).reshape(-1), dtype=np.float32)).to(dev)
    d_barr = torch.from_numpy(barr).to(dev)
    d_p = torch.from_numpy(c["p"]).to(dev)
    d_coh, d_res = f32(c["coh"]), f32(c["res"])
    d_X = f32(np.asfortranarray(c["X"]).T.copy())   # column major
    d_H = torch.zeros(2 * 16 * N * N, dtype=torch.float32, device=dev)
    d_A = torch.zeros(2 * 4 * N * Nbase, dtype=torch.float32, device=dev)
    d_dR = torch.zeros(2 * 4 * Nbase * Nbase, dtype=torch.float32, device=dev)
    vp = lambda t: C.c_void_p(t.data_ptr())
    torch.cuda.synchronize()
    L.cudakernel_hessian(R, N, T, 1, vp(d_barr), vp(d_p), c["nchunk"], vp(d_coh), vp(d_res), vp(d_H))
    L.cudakernel_d_solutions(R, N, T, 1, vp(d_barr), vp(d_p), c["nchunk"], vp(d_coh), vp(d_A))
    L.cudakernel_d_residuals(R, N, T, 1, vp(d_barr), vp(d_p), c["nchunk"], vp(d_coh), vp(d_X), vp(d_dR))
    torch.cuda.synchronize()
    cplx = lambda t: t.cpu().numpy().astype(np.float64).view(np.complex128)
    H = cplx(d_H).reshape(4 * N, 4 * N).T       # column major
    A = cplx(d_A).reshape(Nbase, 4 * N).T
    dR = cplx(d_dR).reshape(Nbase, Nbase, 4)     # [bl][row][corr]
    dR = np.transpose(dR, (2, 1, 0))
    Hr, Ar, dRr = restated(c)
    assert rel(H, Hr) < 1e-4, rel(H, Hr)
    assert rel(A, Ar) < 1e-4, rel(A, Ar)
    assert rel(dR, dRr) < 1e-4, rel(dR, dRr)
    if kw.get("weak"):
        assert (np.abs(np.real(np.diag(Hr))) < 1).any()


def _barr(c):
    return make_barr(c["sta1"], c["sta2"], c["flag"])


@pytest.mark.parametrize("kw", CASES + [dict(N=62, T=10, nchunk=2)], ids=IDS + ["62-stations"])
def test_product_kernels_match_the_restatement(api, kw):
    """the fp64 kernels through dirac_b200_diagnostics_eval against the restatement to 1e-11, and
    bit-identical from run to run (no atomics)"""
    c = kernel_case(**kw)
    run = lambda: api.diagnostics_eval(c["N"], c["Nbase"], c["T"], _barr(c), c["p"], c["nchunk"],
                                       c["coh"], c["res"], c["X"])
    H, A, dR = run()
    Hr, Ar, dRr = restated(c)
    assert rel(H, Hr) < 1e-11, rel(H, Hr)
    assert rel(A, Ar) < 1e-11, rel(A, Ar)
    assert rel(dR, dRr) < 1e-11, rel(dR, dRr)
    H2, A2, dR2 = run()
    assert np.array_equal(H, H2) and np.array_equal(A, A2) and np.array_equal(dR, dR2)


FREQS = np.array([150e6, 152e6, 154e6])


def call_case(N=7, M=3, T=10, nchunk=None, seed=17):
    b = small_problem(N=N, M=M, tilesz=T, seed=seed, kmean=2.0, nchunk=nchunk, flag_frac=0.1)
    pr = b.pr
    for k, cl in enumerate(pr.clusters):
        cl["id"] = k if k != 1 else -1     # every cluster counts, whatever its id
    sky = SkyModel(pr.clusters, pr.N)
    rng = np.random.default_rng(seed)
    x0 = rng.normal(0, 1, 8 * pr.Nbase1 * len(FREQS))
    pp = perturbed_jones(pr, amp=0.2)
    return b, sky, x0, pp


def restated_call(api, b, sky, x0, pp, fdelta, hadd=None):
    """steps 1-6: the residual by the library's own simulation call (subtract every cluster), the
    channel-0 coherencies by its multi-channel prediction, then the restatement"""
    pr = b.pr
    R = pr.Nbase1
    res = x0.copy()
    assert api.predict_visibilities_multifreq_withsol(pr.u, pr.v, pr.w, pp.copy(), res, pr.N, pr.Nbase,
                                                      pr.tilesz, b.fresh_barr(), sky, FREQS, fdelta,
                                                      add_to_data=3) == 0
    coh = api.precalculate_coherencies_multifreq(pr.u, pr.v, pr.w, pr.N, R, b.fresh_barr(), sky,
                                                 FREQS[:1], fdelta / len(FREQS), uvmax=1e300)
    coh = coh.reshape(R, sky.M, 4)
    clusters, off = [], 0
    for k in range(sky.M):
        nch = pr.nchunk[k]
        clusters.append(dict(p=pp[off:off + 8 * pr.N * nch], nchunk=nch, coh=coh[:, k]))
        off += 8 * pr.N * nch
    r0 = res[:8 * R].view(np.complex128).reshape(R, 4)
    dR, _, _ = ir.diagnostics(pr.N, pr.Nbase, pr.tilesz, pr.sta1, pr.sta2, pr.flag, clusters, r0, hadd)
    return res, dR


def match_multiset(got, want, tol):
    want = list(want)
    for g in got:
        j = int(np.argmin(np.abs(np.array(want) - g)))
        assert abs(want[j] - g) <= tol, (g, want[j], tol)
        want.pop(j)


def run_call(api, b, sky, x0, pp, fdelta, **kw):
    pr = b.pr
    x = x0.copy()
    rv = api.calculate_diagnostics_gpu(pr.u, pr.v, pr.w, pp.copy(), x, pr.N, pr.Nbase, pr.tilesz,
                                       b.fresh_barr(), sky, FREQS, fdelta, **kw)
    return rv, x


@pytest.mark.parametrize("nchunk", [None, [1, 3, 2]], ids=["nchunk1", "hybrid"])
def test_whole_call_matches_the_restatement(api, nchunk):
    b, sky, x0, pp = call_case(nchunk=nchunk)
    pr = b.pr
    fdelta = pr.fdelta * len(FREQS)
    rv, x = run_call(api, b, sky, x0, pp, fdelta)
    assert rv == 0
    res, dR = restated_call(api, b, sky, x0, pp, fdelta)
    R, Nbase = pr.Nbase1, pr.Nbase
    x0c = x[:8 * R]
    for t in range(1, pr.tilesz):
        assert np.array_equal(x0c[8 * Nbase * t:8 * Nbase * (t + 1)], x0c[:8 * Nbase])
    E = ir.x_to_eig(x0c, Nbase)
    for c in range(4):
        want = np.linalg.eigvals(dR[c])
        match_multiset(E[c], want, 1e-8 * np.abs(want).max())
    assert np.abs(x[8 * R:] - res[8 * R:]).max() <= 1e-12 * np.abs(res[8 * R:]).max()


def test_consensus_form(api):
    """rho, Bpoly and Bi given (the MPI slave, sagecal_slave.cpp:968) with Mt > M: 0.5 rho_k Fd1 on the
    Hessian's real diagonal"""
    b, sky, x0, pp = call_case(nchunk=[1, 2, 1], seed=19)
    pr = b.pr
    M, Npoly = sky.M, 3
    rng = np.random.default_rng(2)
    rho = rng.uniform(1.0, 5.0, M)
    Bpoly = rng.uniform(0.2, 0.6, Npoly)
    Bi = np.stack([np.linalg.inv(np.eye(Npoly) * 3 + 0.1 * np.ones((Npoly, Npoly))) for _ in range(M)])
    fdelta = pr.fdelta * len(FREQS)
    rv, x = run_call(api, b, sky, x0, pp, fdelta, rho=rho, Bpoly=Bpoly, Bi=Bi, Npoly=Npoly)
    assert rv == 0
    hadd = [ir.consensus_hadd(rho[k], Bpoly, Bi[k].reshape(-1)) for k in range(M)]
    assert min(hadd) > 0
    _, dR = restated_call(api, b, sky, x0, pp, fdelta, hadd)
    E = ir.x_to_eig(x[:8 * pr.Nbase], pr.Nbase)
    for c in range(4):
        want = np.linalg.eigvals(dR[c])
        match_multiset(E[c], want, 1e-8 * np.abs(want).max())


def test_62_stations(api):
    """the production launch shapes (N 62, Nbase 1891, M 8, T 10): every eigenvalue sum equals the
    trace of the restatement's dR, every timeslot holds timeslot 0"""
    b, sky, x0, pp = call_case(N=62, M=8, T=10, seed=23)
    pr = b.pr
    fdelta = pr.fdelta * len(FREQS)
    rv, x = run_call(api, b, sky, x0, pp, fdelta)
    assert rv == 0
    _, dR = restated_call(api, b, sky, x0, pp, fdelta)
    Nbase = pr.Nbase
    E = ir.x_to_eig(x[:8 * Nbase], Nbase)
    for c in range(4):
        tr = np.trace(dR[c])
        assert abs(E[c].sum() - tr) <= 1e-8 * np.abs(dR[c]).sum(), (E[c].sum(), tr)
    assert np.array_equal(x[8 * Nbase:16 * Nbase], x[:8 * Nbase])


@pytest.mark.parametrize("tile", [False, True], ids=["array-single", "array-tile"])
def test_beam_residual_matches_the_library(api, tile):
    """with array beams, channels >= 1 hold the library's own calculate_residuals_multifreq_withbeam
    without correction; channel 0 holds finite eigenvalues copied to every timeslot"""
    b, sky, x0, pp = call_case(T=5, seed=29)
    pr = b.pr
    for cl in pr.clusters:
        cl["id"] = 0
    sky = SkyModel(pr.clusters, pr.N)
    rng = np.random.default_rng(31)
    ra0, dec0 = 1.2, np.deg2rad(58.0)
    for cl in pr.clusters:
        K = len(cl["ll"])
        cl["ra"] = ra0 + np.deg2rad(rng.uniform(-4, 4, K))
        cl["dec"] = dec0 + np.deg2rad(rng.uniform(-4, 4, K))
    sky = SkyModel(pr.clusters, pr.N)
    lon = np.deg2rad(6.87 + rng.uniform(-0.5, 0.5, pr.N))
    lat = np.deg2rad(52.9 + rng.uniform(-0.3, 0.3, pr.N))
    t = 2456789.3 + np.arange(pr.tilesz) * 10.0 / 86400.0
    elems = []
    for n in range(pr.N):
        if tile:
            g = (np.arange(4) - 1.5) * 1.25
            dip = np.array([[xx, yy, 0.0] for xx in g for yy in g])
            cen = np.c_[rng.uniform(-15, 15, (20, 2)), rng.normal(0, 0.05, 20)]
            elems.append(np.vstack([dip, cen]))
        else:
            elems.append(np.c_[rng.uniform(-40, 40, (40, 2)), rng.normal(0, 0.1, 40)])
    beam = BeamSetup(2 if tile else 1, ra0 + 0.01, dec0 - 0.01, ra0, dec0, 148e6, lon, lat, t, elems,
                     None, 1)
    fdelta = pr.fdelta * len(FREQS)
    rv, x = run_call(api, b, sky, x0, pp, fdelta, beam=beam)
    assert rv == 0
    res = x0.copy()
    assert api.calculate_residuals_multifreq_withbeam(pr.u, pr.v, pr.w, pp.copy(), res, pr.N, pr.Nbase,
                                                      pr.tilesz, b.fresh_barr(), sky, FREQS, fdelta,
                                                      beam) == 0
    R, Nbase = pr.Nbase1, pr.Nbase
    assert np.array_equal(x[8 * R:], res[8 * R:])
    assert np.isfinite(x[:8 * R]).all()
    assert np.array_equal(x[8 * Nbase:16 * Nbase], x[:8 * Nbase])


def test_beyond_device_memory_is_refused(api, capfd):
    """512 stations: the four dR matrices alone take 64 Nbase^2 bytes (about 1.1 TB); -1 and a message
    before any device work, x untouched"""
    N, T = 512, 1
    pairs = [(p, q) for p in range(N) for q in range(p + 1, N)]
    Nbase = len(pairs)
    sta1 = np.array([p for p, _ in pairs], dtype=np.int32)
    sta2 = np.array([q for _, q in pairs], dtype=np.int32)
    b = small_problem(N=7, M=1, tilesz=1, seed=3)
    sky = SkyModel(b.pr.clusters, N)
    u = np.zeros(Nbase)
    x = np.ones(8 * Nbase)
    pp = np.tile(np.array([1, 0, 0, 0, 0, 0, 1, 0], dtype=np.float64), N * sum(sky.nchunk))
    rv = api.calculate_diagnostics_gpu(u, u, u, pp, x, N, Nbase, T, make_barr(sta1, sta2, np.zeros(Nbase)),
                                       sky, FREQS[:1], 1e5)
    assert rv == -1
    assert "free" in capfd.readouterr().err
    assert (x == 1).all()
