"""The tiled assembly of J^T J at 512 stations (8N = 4096) and the in-place damping of the cuSOLVER
Cholesky path: the lower triangle (column-major) of J^T J + mu I against the full undamped matrix and
the O(rows) restatement, a damp-factor-rebuild cycle against scipy's Cholesky, and the batched form
of the sweep's first systems over cluster lists of several lengths."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from util import relerr

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

dp_ = C.POINTER(C.c_double)
ip_ = C.POINTER(C.c_int)


def _ptr(a, t=dp_):
    return a.ctypes.data_as(t)


@pytest.fixture(scope="module")
def setup(api):
    import make_golden_n512 as gen
    from sagecal_b200 import lib as blib
    from sagecal_b200.dirac_api import SkyModel, make_barr
    pr = gen.build()
    L = api.lib
    L.dirac_b200_assemble_damped.restype = None
    L.dirac_b200_assemble_damped.argtypes = [C.c_void_p, C.c_int, C.c_int, dp_, C.c_int, dp_, C.c_int,
                                             dp_, ip_]
    L.dirac_b200_assemble_batch.restype = None
    L.dirac_b200_assemble_batch.argtypes = [C.c_void_p, dp_, ip_, C.c_int, C.c_double, C.c_int, dp_, dp_]
    dp = blib.DeviceProblem(api, pr.N, pr.Nbase, pr.tilesz, make_barr(pr.sta1, pr.sta2, pr.flag),
                            SkyModel(pr.clusters, pr.N), pr.coh, pr.x)
    rng = np.random.default_rng(11)
    n8 = 8 * pr.N
    pblk = np.ascontiguousarray(pr.pp0[:n8] + 0.1 * rng.normal(0, 1, n8))
    _, JTJ, _ = dp.normal_eq(0, 0, pblk, pr.x)
    yield pr, L, dp, pblk, JTJ
    dp.close()


def _damped(L, dp, pblk, mus, factor):
    n8 = pblk.size
    mus = np.asarray(mus, dtype=np.float64)
    out = np.zeros((len(mus), n8, n8))
    info = np.zeros(len(mus), dtype=np.int32)
    L.dirac_b200_assemble_damped(dp.h, 0, 0, _ptr(pblk), len(mus), _ptr(mus), 1 if factor else 0,
                                 _ptr(out), _ptr(info, ip_))
    return out, info


def _lower(A):
    """the column-major lower triangle of a row-major buffer: its upper triangle as numpy sees it"""
    return np.triu(A)


def test_full_matrix_symmetric_and_matches_restatement(setup):
    import orcdirac
    pr, L, dp, pblk, JTJ = setup
    assert np.array_equal(JTJ, JTJ.T)
    if not orcdirac.available():
        pytest.skip("oracle/liboracle.so not built")
    _, JTJ_o, _ = orcdirac.Oracle(pr).normal_eq(0, 0, pr.tilesz, pblk, pr.x)
    assert relerr(JTJ, JTJ_o) < 1e-11


def test_lower_triangle_damped(setup):
    pr, L, dp, pblk, JTJ = setup
    mu = 0.37 * np.max(np.abs(np.diag(JTJ)))
    out, _ = _damped(L, dp, pblk, [mu], False)
    want = JTJ + mu * np.eye(JTJ.shape[0])
    assert np.array_equal(_lower(out[0]), _lower(want))


def test_damped_factor_rebuild_cycle(setup):
    """factor at mu1 in place, rebuild over the factor at mu2 and factor again"""
    from scipy.linalg import cho_factor
    pr, L, dp, pblk, JTJ = setup
    dmax = np.max(np.abs(np.diag(JTJ)))
    mus = [1e-3 * dmax, 8e-3 * dmax, 2e-3 * dmax]
    out, info = _damped(L, dp, pblk, mus, True)
    assert list(info) == [0, 0, 0]
    n8 = JTJ.shape[0]
    for k, mu in enumerate(mus):
        c, low = cho_factor(JTJ + mu * np.eye(n8), lower=True)
        # row-major buffer = column-major factor transposed: numpy's upper triangle is L^T
        got = _lower(out[k]).T
        want = np.tril(c)
        assert relerr(got, want) < 1e-11, (k, relerr(got, want))


@pytest.mark.parametrize("lst", [[0], [1], [1, 0], [0, 1]])
def test_batched_lists(setup, lst):
    pr, L, dp, pblk, JTJ = setup
    n8 = 8 * pr.N
    tau = 1e-3
    nb = len(lst)
    pp = np.ascontiguousarray(pr.pp0 + 0.1 * np.random.default_rng(5).normal(0, 1, pr.pp0.size))
    li = np.asarray(lst, dtype=np.int32)
    mu = np.zeros(nb)
    low = np.zeros((nb, n8, n8))
    full = np.zeros((nb, n8, n8))
    L.dirac_b200_assemble_batch(dp.h, _ptr(pp), _ptr(li, ip_), nb, tau, 1, _ptr(mu), _ptr(low))
    mu2 = np.zeros(nb)
    L.dirac_b200_assemble_batch(dp.h, _ptr(pp), _ptr(li, ip_), nb, tau, 0, _ptr(mu2), _ptr(full))
    assert np.array_equal(mu, mu2)
    for y, k in enumerate(lst):
        # cluster k's block of pp (one chunk per cluster at this shape)
        _, ref, _ = dp.normal_eq(k, 0, np.ascontiguousarray(pp[k * n8:(k + 1) * n8]), pr.x)
        assert np.array_equal(full[y], ref)
        d = np.diag(ref)
        assert mu[y] == tau * d[np.argmax(np.abs(d))]
        assert np.array_equal(_lower(low[y]), _lower(ref + mu[y] * np.eye(n8)))
