"""CPU: the long-double restatement of the sky prediction (util.sky_predict_ref) against the compiled
reference, element by element, on the edge inputs the GPU tests feed the coherency kernel
(util.sky_edge_case): precalculate_coherencies (predict.c:345-497) and
predict_visibilities_multifreq (residual.c:1067-1248).  This pins the oracle of
test_gpu_sky_predict_edges.py without a GPU.  Shapelets are not restated; their Fourier-plane factor
is pinned against the reference's shapelet_contrib by test_oracle_coh_math.py."""
import numpy as np
import pytest

from util import (SKY_C, SKY_EDGE_CASES, sky_edge_case, sky_predict_ref, small_problem,
                  split_cluster)
from sagecal_b200.dirac_api import SkyModel, barr_to_numpy

EPS = np.finfo(np.float64).eps
N, TILESZ = 6, 4


def _rows():
    b = small_problem(N=N, M=2, tilesz=TILESZ, seed=5)
    return b, b.pr.Nbase


def check_elementwise(got, want, budget):
    """|got - want| <= SKY_C eps budget element-wise (complex [..., 4] against budget [...]).  The
    bound must stay far below the values it checks: on the median row it is under 1e-7 of the row's
    largest correlation (a phase of 1e6 rad alone allows SKY_C eps 1e6 ~ 4e-9 of the flux).
    returns the largest error / bound"""
    err = np.abs(np.asarray(got, dtype=np.complex128) - want.astype(np.complex128))
    tol = SKY_C * EPS * budget[..., None]
    scale = np.max(np.abs(want.astype(np.complex128)), axis=-1)
    assert np.median(tol[..., 0] / np.maximum(scale, 1e-300)) < 1e-7, "vacuous bound"
    bad = ~(err <= tol)   # NaN is an error too
    assert not bad.any(), (np.argwhere(bad)[:5], err[bad][:5], tol[bad][:5])
    return float(np.max(err / tol))


@pytest.mark.parametrize("case", SKY_EDGE_CASES)
def test_restatement_coherencies(ref, case):
    """MODE 0: per-cluster coherencies at the first channel, fluxes as given"""
    u, v, w, cls, freqs, fdelta = sky_edge_case(case)
    b, Nbase = _rows()
    got = ref.precalculate_coherencies(u, v, w, N, Nbase * TILESZ, b.fresh_barr(), SkyModel(cls, N),
                                       freqs[0], fdelta)
    want, budget = sky_predict_ref(u, v, w, cls, freqs[0], 0.5 * fdelta, spectral=False)
    check_elementwise(got.reshape(want.shape), want, budget)


@pytest.mark.parametrize("case", SKY_EDGE_CASES)
def test_restatement_predict_multifreq(ref, case):
    """MODE 1: the sum over clusters per channel, spectral-index fluxes, smearing width fdelta / Nchan"""
    u, v, w, cls, freqs, fdelta = sky_edge_case(case)
    b, Nbase = _rows()
    R = Nbase * TILESZ
    x = np.zeros(8 * R * len(freqs))
    ref.predict_visibilities_multifreq(u, v, w, x, N, Nbase, TILESZ, b.fresh_barr(), SkyModel(cls, N),
                                       freqs, fdelta, add_to_data=1)
    got = x.reshape(len(freqs), R, 4, 2)
    got = got[..., 0] + 1j * got[..., 1]
    for c, f in enumerate(freqs):
        want, budget = sky_predict_ref(u, v, w, cls, f, 0.5 * fdelta / len(freqs), spectral=True)
        check_elementwise(got[c], want.sum(axis=1), budget.sum(axis=1))


def test_restatement_sees_the_edges():
    """the edge cases reach what they are named for"""
    u, v, w, cls, freqs, _ = sky_edge_case("long")
    phase = [2 * np.pi * freqs[-1] * np.abs(u[:, None] * c["ll"] + v[:, None] * c["mm"]
                                            + w[:, None] * c["nn"]) for c in cls]
    assert 1e5 < max(np.max(p) for p in phase) < 2e6
    u, v, w, cls, freqs, fdelta = sky_edge_case("widefd")
    want, _ = sky_predict_ref(u, v, w, cls, freqs[0], 0.5 * fdelta, spectral=False)
    plain, _ = sky_predict_ref(u, v, w, cls, freqs[0], 1e-9, spectral=False)
    ratio = np.abs(want[..., 0]) / np.abs(plain[..., 0])
    assert np.min(ratio) < 0.2
    u, v, w, cls, freqs, _ = sky_edge_case("gauss")
    wide = split_cluster(cls[0], (2, 2))[1]   # the two Gaussians of 1 rad vanish to underflow
    want, _ = sky_predict_ref(u, v, w, [wide], freqs[0], 1e-9, spectral=False)
    assert np.all(want == 0)
    u, v, w, cls, freqs, fdelta = sky_edge_case("bessel")
    for cl in cls:   # every disk and ring sits on a Bessel zero at one row
        one = split_cluster(cl, (1, 1, 1, 1))
        for s, c1 in enumerate(one):
            c1["disk"] = {0: cl["disk"][s]}
        want, _ = sky_predict_ref(u, v, w, one, freqs[0], 1e-9, spectral=False)
        a = np.abs(want[..., 0].astype(np.complex128))
        assert np.all(np.min(a, axis=0) < 1e-12 * np.max(a, axis=0))


def _uv_edges(pr, freq, rows):
    """for each of the rows: its uv distance as the reference computes it (plain double, no fused
    multiply-add), one ulp below and one above"""
    d = np.sqrt(pr.u[rows] * pr.u[rows] + pr.v[rows] * pr.v[rows]) * freq
    return [(float(x), float(np.nextafter(x, 0)), float(np.nextafter(x, np.inf))) for x in d]


def uvcut_calls(pr):
    """(uvmin, uvmax) pairs that put rows exactly on, and one ulp either side of, both limits"""
    rows = np.argsort(np.hypot(pr.u, pr.v))
    lo, hi = rows[len(rows) // 4: len(rows) // 4 + 3], rows[-len(rows) // 4 - 3: -len(rows) // 4]
    out = []
    for a, z in zip(_uv_edges(pr, pr.freq0, lo), _uv_edges(pr, pr.freq0, hi)):
        for i in range(3):
            out.append((a[i], z[i]))
    return out


def test_restatement_uvcut(ref):
    """the uv cut of precalculate_coherencies at its limits: flag 2 exactly where
    sqrt(u u + v v) f < uvmin or > uvmax in plain double arithmetic, 1 kept, 0 otherwise"""
    b = small_problem(N=N, M=2, tilesz=TILESZ, seed=5)
    pr = b.pr
    uvd = np.sqrt(pr.u * pr.u + pr.v * pr.v) * pr.freq0
    for uvmin, uvmax in uvcut_calls(pr):
        barr = b.fresh_barr()
        ref.precalculate_coherencies(pr.u, pr.v, pr.w, N, pr.Nbase1, barr, b.sky, pr.freq0, pr.fdelta,
                                     uvmin=uvmin, uvmax=uvmax)
        want = np.where(pr.flag != 0, pr.flag, np.where((uvd < uvmin) | (uvd > uvmax), 2, 0))
        assert np.array_equal(barr_to_numpy(barr, pr.Nbase1)[2], want), (uvmin, uvmax)
