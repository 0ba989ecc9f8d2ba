"""Diffuse-cluster coherencies on the GPU (recalculate_diffuse_coherencies, diffuse_predict.c:295-586)
against the compiled reference's CPU path, and the resident form dirac_b200_diffuse_coherencies.  Every
case checks the rewritten cluster per row within 1e-11 of its largest value and every other cluster
bit for bit unchanged.  (Large answers of the reference are stored as a sample: the comparisons use
the recorded entries.)"""
import ctypes as C

import numpy as np
import pytest

from sagecal_b200.dirac_api import SkyModel, dptr, make_barr
from test_oracle_diffuse_math import FDELTA, FREQ0, diffuse_problem, run_diffuse

pytestmark = pytest.mark.gpu


def check_against_reference(request, ref, pb):
    want = run_diffuse(ref, pb)       # the reference first: its answers are recorded without a GPU
    api = request.getfixturevalue("api")
    got = run_diffuse(api, pb)
    cid, M, R = pb["cid"], pb["M"], pb["R"]
    x0 = pb["x0"].reshape(R, M, 4)
    others = [k for k in range(M) if k != cid]
    assert np.array_equal(got[:, others], x0[:, others])
    known = np.isfinite(want[:, cid]).all(axis=1)
    assert known.sum() > 0
    w, g = want[known, cid], got[known, cid]
    scale = np.max(np.abs(w))
    assert scale > 0
    err = np.max(np.abs(g - w), axis=1) / scale
    assert np.max(err) <= 1e-11, np.max(err)
    return got


CASES = {
    "cid-first": dict(N=9, T=3, M=3, cid=0, n0s=(8,), sh=2),
    "cid-middle": dict(N=9, T=3, M=3, cid=1, n0s=(8,), sh=2),
    "cid-last": dict(N=9, T=3, M=3, cid=2, n0s=(8,), sh=2),
    "flagged": dict(N=9, T=3, M=3, cid=1, n0s=(6,), sh=2, flag_frac=0.3),
    "T1": dict(N=9, T=1, n0s=(5,), sh=2),
    "T7": dict(N=9, T=7, n0s=(5,), sh=2),
    "T33": dict(N=9, T=33, n0s=(5,), sh=2),
    "N2": dict(N=2, T=3, n0s=(4,), sh=2, zero_row=True),
    "N33": dict(N=33, T=2, n0s=(4,), sh=2),
    "N62": dict(N=62, T=2, M=2, cid=1, n0s=(4,), sh=2),
    "n0-1": dict(N=6, T=3, n0s=(1,), sh=1),
    "n0-20": dict(N=4, T=2, n0s=(20,), sh=3),
    "n0-32": dict(N=3, T=2, n0s=(32,), sh=2),
    "sh1": dict(N=7, T=2, n0s=(6,), sh=1),
    "sh4": dict(N=7, T=2, n0s=(6,), sh=4),
    "sources-3": dict(N=8, T=3, n0s=(5, 3, 7), sh=3, zero_row=True),
}


@pytest.mark.parametrize("case", list(CASES.values()), ids=list(CASES))
def test_diffuse_against_reference(request, ref, case):
    check_against_reference(request, ref, diffuse_problem(seed=len(request.node.name), **case))


def test_zero_source_cluster_is_left_untouched(api):
    pb = diffuse_problem(N=5, T=2, n0s=(), sh=2)
    got = run_diffuse(api, pb)
    assert np.array_equal(got.reshape(-1), pb["x0"])


def _create(api, pb, coh):
    from sagecal_b200.lib import DeviceProblem
    sky = SkyModel(pb["clusters"], pb["N"])
    barr = make_barr(pb["sta1"], pb["sta2"], pb["flag"])
    x = np.random.default_rng(9).normal(0, 1, 8 * pb["R"])
    return DeviceProblem(api, pb["N"], pb["Nb"], pb["T"], barr, sky, coh.reshape(-1).copy(), x), sky


def _admm(api, dp, pb, sky):
    L = api.lib
    L.dirac_b200_sagefit_admm.restype = C.c_int
    L.dirac_b200_sagefit_admm.argtypes = [C.c_void_p] + [C.POINTER(C.c_double)] * 5 + [C.c_int] * 4 + \
        [C.POINTER(C.c_double)] * 2
    npar = 8 * pb["N"] * sky.Mt
    pp = np.tile(np.array([1.0, 0, 0, 0, 0, 0, 1.0, 0]), pb["N"] * sky.Mt)
    Y = np.zeros(npar)
    BZ = pp.copy()
    rho = np.full(pb["M"], 2.0)
    xo = np.zeros(8 * pb["R"])
    r0, r1 = C.c_double(0), C.c_double(0)
    assert L.dirac_b200_sagefit_admm(dp.h, dptr(pp), dptr(xo), dptr(Y), dptr(BZ), dptr(rho), 2, 3, 0, 0,
                                     C.byref(r0), C.byref(r1)) == 0
    return pp, xo, r0.value, r1.value


def test_resident_equals_the_reference_named_call_and_feeds_admm(api):
    """dirac_b200_diffuse_coherencies gives the bits of recalculate_diffuse_coherencies, and an ADMM
    solve after it runs on the new coherencies: the answer of a problem created with them"""
    pb = diffuse_problem(N=9, T=4, M=3, cid=1, n0s=(6, 4), sh=2)
    new = run_diffuse(api, pb)
    dp, sky = _create(api, pb, pb["x0"])
    assert dp.diffuse_coherencies(pb["u"], pb["v"], pb["w"], FREQ0, FDELTA, 1, pb["sh"], pb["sh_beta"],
                                  pb["Z"]) == 0
    assert np.array_equal(dp.get_coherencies(), new.reshape(-1))
    a = _admm(api, dp, pb, sky)
    dp.close()
    dq, sky2 = _create(api, pb, new)
    b = _admm(api, dq, pb, sky2)
    dq.close()
    # (the solver's reductions are not bit-reproducible from run to run: agreement to rounding)
    rel = lambda x, y: np.max(np.abs(x - y)) / np.max(np.abs(y))
    assert rel(a[0], b[0]) < 1e-9 and rel(a[1], b[1]) < 1e-9, (rel(a[0], b[0]), rel(a[1], b[1]))
    assert abs(a[3] - b[3]) <= 1e-9 * abs(b[3])
    dz, sky3 = _create(api, pb, pb["x0"])
    c = _admm(api, dz, pb, sky3)
    dz.close()
    assert rel(a[1], c[1]) > 1e-3  # the old coherencies give another answer
