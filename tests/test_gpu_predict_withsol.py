"""Simulation with solutions on the GPU (driver option -a 1|2|3 with -p): the model of every cluster not
in the ignore list, J_p C_k(chan) J_q^H with the solved Jones, written, added or subtracted, then the
optional correction by one cluster's inverse Jones.  predict_visibilities_multifreq_withsol and
predict_visibilities_multifreq_withsol_withbeam against the compiled reference (residual.c:1342-1740,
predict_withbeam.c:1452-1680), exact identities with the other multifreq calls, the beam variant's
correction against numpy, and its GPU-build twin."""
import numpy as np
import pytest

from util import small_problem, relerr, perturbed_jones
from sagecal_b200.dirac_api import SkyModel

pytestmark = pytest.mark.gpu

SIMUL_ONLY, SIMUL_ADD, SIMUL_SUB = 1, 2, 3
NO_CCID = -99999
FREQS = np.array([146e6, 150e6, 154e6, 158e6])


def withsol_problem(nchunk=None, seed=23):
    """9 stations, 3 clusters (the first with a negative id), 6 timeslots, 4 channels, spectral
    indices, Gaussians, 10 % flagged rows, data x0 and perturbed Jones pp"""
    b = small_problem(N=9, M=3, tilesz=6, seed=seed, kmean=2.0, gaussian_frac=0.3, nchunk=nchunk,
                      flag_frac=0.1)
    pr = b.pr
    assert (pr.flag != 0).any()
    for k, cl in enumerate(pr.clusters):
        K = len(cl["ll"])
        cl["spec_idx"] = np.where(np.arange(K) % 2 == 0, -0.7, 0.0)
        cl["spec_idx1"] = np.full(K, 0.05)
        cl["spec_idx2"] = np.full(K, -0.01)
        cl["f0"] = np.full(K, 140e6)
        cl["id"] = k if k != 0 else -1
    sky = SkyModel(pr.clusters, pr.N)
    rng = np.random.default_rng(4)
    x0 = rng.normal(0, 1, 8 * pr.Nbase1 * len(FREQS))
    pp = perturbed_jones(pr, amp=0.2)
    return b, sky, x0, pp


def simulate(lib, b, sky, x0, pp, **kw):
    pr = b.pr
    x = x0.copy()
    rv = lib.predict_visibilities_multifreq_withsol(pr.u, pr.v, pr.w, pp.copy(), x, pr.N, pr.Nbase,
                                                    pr.tilesz, b.fresh_barr(), sky, FREQS,
                                                    pr.fdelta * len(FREQS), **kw)
    assert rv == 0
    return x


# (add_to_data, ignorelist, ccid, nchunk, phase_only)
CASES = [(SIMUL_ONLY, None, NO_CCID, None, 0), (SIMUL_ADD, None, NO_CCID, None, 0),
         (SIMUL_SUB, None, NO_CCID, None, 0), (SIMUL_ONLY, [0, 1, 0], NO_CCID, None, 0),
         (SIMUL_ADD, [0, 1, 0], NO_CCID, None, 0), (SIMUL_SUB, [0, 1, 0], NO_CCID, None, 0),
         (SIMUL_ADD, None, 1, None, 0), (SIMUL_SUB, None, 2, [1, 2, 3], 0),
         (SIMUL_ONLY, None, 1, None, 1), (SIMUL_ADD, None, 2, [1, 2, 3], 1),
         (SIMUL_ONLY, [0, 1, 0], 1, None, 0)]
IDS = ["only", "add", "sub", "only-ignore-1", "add-ignore-1", "sub-ignore-1", "add-correct-by-1",
       "sub-hybrid-correct-by-2", "only-phase-only-1", "add-phase-only-hybrid-2",
       "only-correct-by-ignored-1"]


@pytest.mark.parametrize("add,ign,ccid,nchunk,phase_only", CASES, ids=IDS)
def test_withsol_against_reference(api, ref, add, ign, ccid, nchunk, phase_only):
    b, sky, x0, pp = withsol_problem(nchunk)
    kw = dict(ignorelist=ign, add_to_data=add, ccid=ccid, rho=1e-9, phase_only=phase_only)
    xa = simulate(ref, b, sky, x0, pp, **kw)
    xb = simulate(api, b, sky, x0, pp, **kw)
    # (phase_only: the correction goes through a joint diagonalisation by Jacobi rotations,
    # manifold_average.c:399-610, restated on the host with its own 3x3 eigen-solver)
    assert relerr(xb, xa) < (1e-9 if phase_only else 1e-11), relerr(xb, xa)
    assert relerr(xa, x0) > 1e-3   # the model (or the correction) changed the data


def test_sub_equals_the_residual(api):
    """SIMUL_SUB ignoring the clusters with a negative id is calculate_residuals_multifreq, bit for bit"""
    b, sky, x0, pp = withsol_problem([1, 2, 3])
    pr = b.pr
    ign = [1 if cl["id"] < 0 else 0 for cl in pr.clusters]
    xs = simulate(api, b, sky, x0, pp, ignorelist=ign, add_to_data=SIMUL_SUB)
    xr = x0.copy()
    assert api.calculate_residuals_multifreq(pr.u, pr.v, pr.w, pp.copy(), xr, pr.N, pr.Nbase,
                                             pr.tilesz, b.fresh_barr(), sky, FREQS,
                                             pr.fdelta * len(FREQS)) == 0
    assert np.array_equal(xs, xr)
    assert relerr(xs, x0) > 1e-3


def test_unit_jones_only_equals_the_plain_predict(api):
    """with unit Jones and no cluster ignored, SIMUL_ONLY is predict_visibilities_multifreq"""
    b, sky, x0, _ = withsol_problem()
    pr = b.pr
    unit = np.zeros_like(pr.pp0)
    unit[0::8] = 1.0
    unit[6::8] = 1.0
    xs = simulate(api, b, sky, x0, unit, add_to_data=SIMUL_ONLY)
    xp = x0.copy()
    api.predict_visibilities_multifreq(pr.u, pr.v, pr.w, xp, pr.N, pr.Nbase, pr.tilesz, b.barr, sky,
                                       FREQS, pr.fdelta * len(FREQS), add_to_data=1)
    assert relerr(xs, xp) < 1e-12
    assert np.max(np.abs(xp)) > 0


@pytest.mark.parametrize("ign", [None, [0, 1, 0]], ids=["all", "ignore-1"])
def test_add_and_sub_are_only_plus_minus_data(api, ign):
    """ADD(x0) - x0 == ONLY and SUB(x0) == x0 - ONLY to rounding"""
    b, sky, x0, pp = withsol_problem([2, 1, 3])
    only = simulate(api, b, sky, x0, pp, ignorelist=ign, add_to_data=SIMUL_ONLY)
    add = simulate(api, b, sky, x0, pp, ignorelist=ign, add_to_data=SIMUL_ADD)
    sub = simulate(api, b, sky, x0, pp, ignorelist=ign, add_to_data=SIMUL_SUB)
    scale = np.max(np.abs(x0)) + np.max(np.abs(only))
    eps = np.finfo(np.float64).eps
    assert np.max(np.abs((add - x0) - only)) <= 4 * eps * scale
    assert np.max(np.abs(sub - (x0 - only))) <= 4 * eps * scale
    assert np.max(np.abs(only)) > 1e-3 * scale


def test_all_ignored_gives_zeros(api):
    b, sky, x0, pp = withsol_problem()
    x = simulate(api, b, sky, x0, pp, ignorelist=[1, 1, 1], add_to_data=SIMUL_ONLY)
    assert not x.any()


def test_withsol_segmented_clusters(api, ref):
    """clusters staged in several segments of at most 96 sources (1, 95, 96, 97, 192, 200 sources
    and an empty one), 3 channels, one cluster ignored and a correction, against the reference"""
    from test_gpu_kernels import _segment_sky
    b, clusters, sky = _segment_sky()
    pr = b.pr
    freqs = FREQS[:3]
    rng = np.random.default_rng(8)
    p = np.tile(np.array([1.0, 0, 0, 0, 0, 0, 1.0, 0]), pr.N * sky.Mt)
    p += 0.1 * rng.normal(0, 1, p.shape)
    x0 = rng.normal(0, 1, 8 * pr.Nbase1 * len(freqs))
    ign = [0, 0, 1, 0, 0, 0, 0]
    out = []
    for lib in (ref, api):
        x = x0.copy()
        assert lib.predict_visibilities_multifreq_withsol(
            pr.u, pr.v, pr.w, p.copy(), x, pr.N, pr.Nbase, pr.tilesz, b.fresh_barr(), sky, freqs,
            pr.fdelta * 3, ignorelist=ign, add_to_data=SIMUL_ADD, ccid=4) == 0
        out.append(x)
    assert relerr(out[1], out[0]) < 1e-11, relerr(out[1], out[0])
    assert relerr(out[0], x0) > 1e-3


# ---- station beams ---------------------------------------------------------------------------------

BEAM_CASES = [("full", False), ("full_wb", True), ("array", True)]
BEAM_IDS = ["full-single", "full_wb-tile", "array-tile"]


def _beam_setup(ref, mode, tile, seed=37):
    from test_gpu_beam import beam_problem
    freqs = np.array([146e6, 152e6])
    b, sky, beam = beam_problem(ref, mode, tile, seed=seed, freqs=freqs)
    pr = b.pr
    pp = perturbed_jones(pr, seed=4, amp=0.1)
    x0 = np.random.default_rng(2).normal(0, 0.1, 8 * pr.Nbase1 * len(freqs))
    return b, sky, beam, freqs, pp, x0


def simulate_beam(lib, b, sky, beam, freqs, pp, x0, **kw):
    pr = b.pr
    x = x0.copy()
    rv = lib.predict_visibilities_multifreq_withsol_withbeam(pr.u, pr.v, pr.w, pp.copy(), x, pr.N,
                                                             pr.Nbase, pr.tilesz, b.fresh_barr(), sky,
                                                             freqs, pr.fdelta * len(freqs), beam, **kw)
    assert rv == 0
    return x


@pytest.mark.parametrize("mode,tile", BEAM_CASES, ids=BEAM_IDS)
def test_withsol_withbeam_against_reference(api, ref, mode, tile):
    """no correction: the reference's CPU variant and this library agree"""
    b, sky, beam, freqs, pp, x0 = _beam_setup(ref, mode, tile)
    for add, ign in ((SIMUL_ONLY, None), (SIMUL_SUB, [0, 1, 0])):
        kw = dict(ignorelist=ign, add_to_data=add)
        xa = simulate_beam(ref, b, sky, beam, freqs, pp, x0, **kw)
        xb = simulate_beam(api, b, sky, beam, freqs, pp, x0, **kw)
        assert relerr(xb, xa) < 1e-10, (add, relerr(xb, xa))
        assert relerr(xa, x0) > 1e-3
        # the GPU-build twin is the same call
        xt = simulate_beam(api, b, sky, beam, freqs, pp, x0, gpu_twin=True, **kw)
        assert np.array_equal(xt, xb)


@pytest.mark.parametrize("mode,tile", BEAM_CASES, ids=BEAM_IDS)
def test_withsol_withbeam_one_cluster_corrected(api, ref, mode, tile):
    """with exactly one cluster not ignored the reference's CPU variant corrects once, as this
    library always does: the two agree with a correction"""
    b, sky, beam, freqs, pp, x0 = _beam_setup(ref, mode, tile)
    kw = dict(ignorelist=[1, 0, 1], add_to_data=SIMUL_ADD, ccid=2, rho=1e-9)
    xa = simulate_beam(ref, b, sky, beam, freqs, pp, x0, **kw)
    xb = simulate_beam(api, b, sky, beam, freqs, pp, x0, **kw)
    assert relerr(xb, xa) < 1e-9, relerr(xb, xa)
    xt = simulate_beam(api, b, sky, beam, freqs, pp, x0, gpu_twin=True, **kw)
    assert np.array_equal(xt, xb)


def correct_once(x, pr, pp, k, nchan, rho=1e-9):
    """x[chan][row][8] corrected by (J + rho I)^-1 of cluster k (one chunk): Jinv_p X Jinv_q^H"""
    J = pp[8 * pr.N * k:8 * pr.N * (k + 1)].reshape(pr.N, 4, 2)
    J = (J[..., 0] + 1j * J[..., 1]).reshape(pr.N, 2, 2) + rho * np.eye(2)
    Ji = np.linalg.inv(J)
    X = x.reshape(nchan, pr.Nbase1, 4, 2)
    X = (X[..., 0] + 1j * X[..., 1]).reshape(nchan, pr.Nbase1, 2, 2)
    Y = Ji[pr.sta1] @ X @ np.conj(np.swapaxes(Ji[pr.sta2], -1, -2))
    out = np.empty((nchan, pr.Nbase1, 4, 2))
    out[..., 0] = Y.reshape(nchan, pr.Nbase1, 4).real
    out[..., 1] = Y.reshape(nchan, pr.Nbase1, 4).imag
    return out.reshape(-1)


@pytest.mark.parametrize("mode,tile", BEAM_CASES, ids=BEAM_IDS)
def test_withsol_withbeam_corrects_once(api, ref, mode, tile):
    """several clusters: the corrected output is the uncorrected one corrected once by the inverse
    Jones of cluster ccid (the reference's CPU variant would correct once per cluster, DESIGN.md 7)"""
    b, sky, beam, freqs, pp, x0 = _beam_setup(ref, mode, tile)
    pr = b.pr
    plain = simulate_beam(api, b, sky, beam, freqs, pp, x0, add_to_data=SIMUL_ADD)
    corr = simulate_beam(api, b, sky, beam, freqs, pp, x0, add_to_data=SIMUL_ADD, ccid=1)
    want = correct_once(plain, pr, pp, 1, len(freqs))
    assert relerr(corr, want) < 1e-12, relerr(corr, want)
    assert relerr(corr, plain) > 1e-3
    xt = simulate_beam(api, b, sky, beam, freqs, pp, x0, add_to_data=SIMUL_ADD, ccid=1,
                       gpu_twin=True)
    assert np.array_equal(xt, corr)
