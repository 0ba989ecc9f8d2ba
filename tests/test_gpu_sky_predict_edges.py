"""The sky-prediction kernel (k_sky_predict, kernels_coh.cu) element by element at its edges.

MODE 0 (precalculate_coherencies) and MODE 1 (predict_visibilities_multifreq) against the long-double
restatement util.sky_predict_ref, every visibility against its own error budget
SKY_C eps sum_s w_s (not against the brightest row): long baselines with |phase| up to 1e6 rad, a
source at the phase centre and rows with u = v = w = 0, wide and tiny smearing widths, Gaussians of
zero and of vanishing extent, disks and rings on Bessel zeros, negative and zero spectral fluxes.
The uv cut with rows exactly on uvmin / uvmax and one ulp either side.  Then the walks of the
staging ring and of the station-beam tables against the compiled reference (relerr per channel
and per cluster): clusters across several staging segments under every beam kind, 1-17 channels
over 11 segments, 1-33 timeslots, and row counts around one CTA.  test_cpu_sky_restatement.py pins
the restatement against the reference.  Each test prints the largest error / bound it saw."""
from fractions import Fraction

import numpy as np
import pytest

from util import (SKY_C, SKY_EDGE_CASES, big_cluster_sky, perturbed_jones, relerr, sky_edge_case,
                  sky_predict_ref, small_problem)
from test_cpu_sky_restatement import check_elementwise, uvcut_calls
from test_gpu_beam import beam_problem
from sagecal_b200.dirac_api import SkyModel, barr_to_numpy

pytestmark = pytest.mark.gpu

N, TILESZ = 6, 4
#: relerr bound of the beam walks, per channel, cluster or timeslot
BEAM_TOL = 1e-11


@pytest.mark.parametrize("case", SKY_EDGE_CASES)
def test_edges_coherencies(api, case):
    """MODE 0: per-cluster coherencies at the first channel"""
    u, v, w, cls, freqs, fdelta = sky_edge_case(case)
    b = small_problem(N=N, M=2, tilesz=TILESZ, seed=5)
    got = api.precalculate_coherencies(u, v, w, N, b.pr.Nbase1, b.fresh_barr(), SkyModel(cls, N),
                                       freqs[0], fdelta)
    want, budget = sky_predict_ref(u, v, w, cls, freqs[0], 0.5 * fdelta, spectral=False)
    print("RATIO coherencies-%s %.3g" % (case, check_elementwise(got.reshape(want.shape), want,
                                                                  budget)))


@pytest.mark.parametrize("case", SKY_EDGE_CASES)
def test_edges_predict_multifreq(api, case):
    """MODE 1: sum over clusters per channel with spectral-index fluxes"""
    u, v, w, cls, freqs, fdelta = sky_edge_case(case)
    b = small_problem(N=N, M=2, tilesz=TILESZ, seed=5)
    pr = b.pr
    x = np.full(8 * pr.Nbase1 * len(freqs), np.nan)   # SIMUL_ONLY overwrites every element
    api.predict_visibilities_multifreq(u, v, w, x, N, pr.Nbase, TILESZ, b.fresh_barr(),
                                       SkyModel(cls, N), freqs, fdelta, add_to_data=1)
    got = x.reshape(len(freqs), pr.Nbase1, 4, 2)
    got = got[..., 0] + 1j * got[..., 1]
    worst = 0.0
    for c, f in enumerate(freqs):
        want, budget = sky_predict_ref(u, v, w, cls, f, 0.5 * fdelta / len(freqs), spectral=True)
        worst = max(worst, check_elementwise(got[c], want.sum(axis=1), budget.sum(axis=1)))
    print("RATIO predict-%s %.3g" % (case, worst))


def _fused(u, v, f):
    """sqrt(fma(u, u, v v)) f, the uv distance as a contracting compiler may evaluate it"""
    s = float(Fraction(u) * Fraction(u) + Fraction(v * v))
    return np.sqrt(s) * f


def test_uvcut_edges(api):
    """rows exactly on uvmin and uvmax and one ulp either side: the flags equal those of the plain
    double rule of the reference (test_cpu_sky_restatement.test_restatement_uvcut), row for row.
    Some of the edge rows are ones whose uv distance a fused multiply-add rounds differently."""
    b = small_problem(N=N, M=2, tilesz=TILESZ, seed=5)
    pr = b.pr
    uvd = np.sqrt(pr.u * pr.u + pr.v * pr.v) * pr.freq0
    fused = np.array([[_fused(a, c, pr.freq0), _fused(c, a, pr.freq0)] for a, c in zip(pr.u, pr.v)])
    calls = uvcut_calls(pr)
    differ = np.flatnonzero(((fused[:, 0] != uvd) | (fused[:, 1] != uvd)) & (pr.flag == 0))
    assert len(differ) >= 2
    for r in differ[:6]:   # each such row on both limits, exactly and one ulp either side
        d = float(uvd[r])
        for e in (d, float(np.nextafter(d, 0)), float(np.nextafter(d, np.inf))):
            calls += [(e, 1e12), (0.0, e)]
    for uvmin, uvmax in calls:
        barr = b.fresh_barr()
        api.precalculate_coherencies(pr.u, pr.v, pr.w, N, pr.Nbase1, barr, b.sky, pr.freq0, pr.fdelta,
                                     uvmin=uvmin, uvmax=uvmax)
        want = np.where(pr.flag != 0, pr.flag, np.where((uvd < uvmin) | (uvd > uvmax), 2, 0))
        got = barr_to_numpy(barr, pr.Nbase1)[2]
        assert np.array_equal(got, want), (uvmin, uvmax, np.flatnonzero(got != want))


# ---- walks of the staging ring and the beam tables, against the compiled reference -----------------

def _radec(cls, seed):
    rng = np.random.default_rng(seed)
    for cl in cls:
        K = len(cl["ll"])
        cl["ra"] = 1.2 + np.deg2rad(rng.uniform(-4, 4, K))
        cl["dec"] = np.deg2rad(58.0) + np.deg2rad(rng.uniform(-4, 4, K))
    return cls


def _per_channel(got, want, nchan, tol, what):
    g, w_ = got.reshape(nchan, -1), want.reshape(nchan, -1)
    worst = 0.0
    for c in range(nchan):
        e = relerr(g[c], w_[c])
        assert e <= tol, (what, c, e)
        worst = max(worst, e)
    return worst


BEAMS = [("array", False), ("element", False), ("full", True), ("array_wb", True), ("full_wb", False)]


@pytest.mark.parametrize("mode,tile", BEAMS, ids=["%s-%s" % (m, "tile" if t else "single")
                                                  for m, t in BEAMS])
def test_segmented_clusters_withbeam(api, ref, mode, tile):
    """clusters of 1, 95, 96, 97, 192 and 200 sources and an empty one (11 staging segments of at
    most 96) under station beams: predict, residual and simulation with solutions, relerr per channel;
    the simulation also per cluster (every other cluster ignored)"""
    freqs = np.array([146e6, 152e6, 158e6])
    b, _, beam = beam_problem(ref, mode, tile, seed=47, freqs=freqs, tilesz=3)
    pr = b.pr
    cls = _radec(big_cluster_sky(seed=13), 47)
    sky = SkyModel(cls, pr.N)
    M = len(cls)
    nx = 8 * pr.Nbase1 * len(freqs)
    xa, xb = np.zeros(nx), np.zeros(nx)
    fd = pr.fdelta * 3
    ref.predict_visibilities_multifreq_withbeam(pr.u, pr.v, pr.w, xa, pr.N, pr.Nbase, pr.tilesz,
                                                b.fresh_barr(), sky, freqs, fd, beam)
    api.predict_visibilities_multifreq_withbeam(pr.u, pr.v, pr.w, xb, pr.N, pr.Nbase, pr.tilesz,
                                                b.fresh_barr(), sky, freqs, fd, beam)
    worst = _per_channel(xb, xa, len(freqs), BEAM_TOL, "predict")
    rng = np.random.default_rng(5)
    J = np.concatenate([pr.pp0[:8 * pr.N] + 0.1 * rng.normal(0, 1, 8 * pr.N) for _ in range(M)])
    x0 = xa + rng.normal(0, 0.01, nx)
    ra, rb = x0.copy(), x0.copy()
    ref.calculate_residuals_multifreq_withbeam(pr.u, pr.v, pr.w, J, ra, pr.N, pr.Nbase, pr.tilesz,
                                               b.fresh_barr(), sky, freqs, fd, beam)
    api.calculate_residuals_multifreq_withbeam(pr.u, pr.v, pr.w, J, rb, pr.N, pr.Nbase, pr.tilesz,
                                               b.fresh_barr(), sky, freqs, fd, beam)
    worst = max(worst, _per_channel(rb - x0, ra - x0, len(freqs), BEAM_TOL, "residual"))
    for k in range(M - 1):   # the last cluster is empty: its model is zero
        ign = np.ones(M, dtype=np.int32)
        ign[k] = 0
        sa, sb = np.zeros(nx), np.zeros(nx)
        ref.predict_visibilities_multifreq_withsol_withbeam(pr.u, pr.v, pr.w, J, sa, pr.N, pr.Nbase,
                                                            pr.tilesz, b.fresh_barr(), sky, freqs, fd,
                                                            beam, ignorelist=ign)
        api.predict_visibilities_multifreq_withsol_withbeam(pr.u, pr.v, pr.w, J, sb, pr.N, pr.Nbase,
                                                            pr.tilesz, b.fresh_barr(), sky, freqs, fd,
                                                            beam, ignorelist=ign)
        worst = max(worst, _per_channel(sb, sa, len(freqs), BEAM_TOL, "withsol cluster %d" % k))
    print("RATIO segmented-%s-%s %.3g" % (mode, tile, worst / BEAM_TOL))


CHANNELS = [(1, "array", True), (3, "array", True), (8, "array", True), (17, "array", True),
            (8, "element_wb", False)]


@pytest.mark.parametrize("nchan,mode,tile", CHANNELS, ids=["%d-%s" % (n, m) for n, m, _ in CHANNELS])
def test_channel_walk_withbeam(api, ref, nchan, mode, tile):
    """nchan channels over the 11 staging segments of big_cluster_sky: the double-buffer parity
    cf nseg + sgi takes both values at every segment; a wide-band element beam reads one coefficient
    set per channel"""
    freqs = 140e6 + 1.3e6 * np.arange(nchan)
    b, _, beam = beam_problem(ref, mode, tile, seed=53, freqs=freqs, tilesz=2)
    pr = b.pr
    sky = SkyModel(_radec(big_cluster_sky(seed=17), 53), pr.N)
    nx = 8 * pr.Nbase1 * nchan
    xa, xb = np.zeros(nx), np.zeros(nx)
    ref.predict_visibilities_multifreq_withbeam(pr.u, pr.v, pr.w, xa, pr.N, pr.Nbase, pr.tilesz,
                                                b.fresh_barr(), sky, freqs, pr.fdelta * nchan, beam)
    api.predict_visibilities_multifreq_withbeam(pr.u, pr.v, pr.w, xb, pr.N, pr.Nbase, pr.tilesz,
                                                b.fresh_barr(), sky, freqs, pr.fdelta * nchan, beam)
    print("RATIO channels-%d-%s %.3g" % (nchan, mode, _per_channel(xb, xa, nchan, BEAM_TOL, "predict")
                                         / BEAM_TOL))


@pytest.mark.parametrize("tilesz", [1, 7, 33])
def test_timeslot_walk_withbeam(api, ref, tilesz):
    """the beam tables' timeslot index walks 1, 7 and 33 timeslots (full beam of a tile
    beam-former), across a staged cluster of 97 sources"""
    freqs = np.array([147e6, 153e6])
    b, _, beam = beam_problem(ref, "full", True, seed=59, freqs=freqs, tilesz=tilesz)
    pr = b.pr
    sky = SkyModel(_radec(big_cluster_sky(seed=19, sizes=(3, 97, 0)), 59), pr.N)
    nx = 8 * pr.Nbase1 * len(freqs)
    xa, xb = np.zeros(nx), np.zeros(nx)
    ref.predict_visibilities_multifreq_withbeam(pr.u, pr.v, pr.w, xa, pr.N, pr.Nbase, pr.tilesz,
                                                b.fresh_barr(), sky, freqs, pr.fdelta * 2, beam)
    api.predict_visibilities_multifreq_withbeam(pr.u, pr.v, pr.w, xb, pr.N, pr.Nbase, pr.tilesz,
                                                b.fresh_barr(), sky, freqs, pr.fdelta * 2, beam)
    g, w_ = xb.reshape(len(freqs), tilesz, -1), xa.reshape(len(freqs), tilesz, -1)
    worst = 0.0
    for c in range(len(freqs)):   # per channel and timeslot
        for t in range(tilesz):
            e = relerr(g[c, t], w_[c, t])
            assert e <= BEAM_TOL, (c, t, e)
            worst = max(worst, e)
    print("RATIO timeslots-%d %.3g" % (tilesz, worst / BEAM_TOL))


ROWS = [(2, 1), (2, 127), (2, 128), (3, 43)]   # (N, tilesz): R = 1, 127, 128, 129


@pytest.mark.parametrize("n,tilesz", ROWS, ids=["R%d" % (n * (n - 1) // 2 * t) for n, t in ROWS])
def test_row_counts(api, ref, n, tilesz):
    """row counts of one, just below, at and just above one CTA of 128 rows in all three modes:
    MODE 0 and 1 element-wise against the restatement, MODE 2 (the residual) against the reference"""
    b = small_problem(N=n, M=3, tilesz=tilesz, seed=61, kmean=2.0, gaussian_frac=0.5)
    pr = b.pr
    freqs = np.array([148e6, 151e6, 155e6])
    got = api.precalculate_coherencies(pr.u, pr.v, pr.w, n, pr.Nbase1, b.fresh_barr(), b.sky,
                                       pr.freq0, pr.fdelta)
    want, budget = sky_predict_ref(pr.u, pr.v, pr.w, pr.clusters, pr.freq0, 0.5 * pr.fdelta, False)
    worst = check_elementwise(got.reshape(want.shape), want, budget)
    nx = 8 * pr.Nbase1 * len(freqs)
    x = np.full(nx, np.nan)
    api.predict_visibilities_multifreq(pr.u, pr.v, pr.w, x, n, pr.Nbase, tilesz, b.fresh_barr(), b.sky,
                                       freqs, pr.fdelta, add_to_data=1)
    xg = x.reshape(len(freqs), pr.Nbase1, 4, 2)
    xg = xg[..., 0] + 1j * xg[..., 1]
    for c, f in enumerate(freqs):
        want, budget = sky_predict_ref(pr.u, pr.v, pr.w, pr.clusters, f, 0.5 * pr.fdelta / 3, True)
        worst = max(worst, check_elementwise(xg[c], want.sum(axis=1), budget.sum(axis=1)))
    pp = perturbed_jones(pr, seed=6, amp=0.2)
    x0 = np.random.default_rng(7).normal(0, 1, nx)
    ra, rb = x0.copy(), x0.copy()
    ref.calculate_residuals_multifreq(pr.u, pr.v, pr.w, pp, ra, n, pr.Nbase, tilesz, b.fresh_barr(),
                                      b.sky, freqs, pr.fdelta)
    api.calculate_residuals_multifreq(pr.u, pr.v, pr.w, pp, rb, n, pr.Nbase, tilesz, b.fresh_barr(),
                                      b.sky, freqs, pr.fdelta)
    e = _per_channel(rb - x0, ra - x0, len(freqs), 1e-11, "residual")
    print("RATIO rows-%d %.3g (residual relerr %.3g)" % (pr.Nbase1, worst, e))
