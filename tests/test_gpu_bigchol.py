"""The blocked batch Cholesky of the sweep's first large LM systems (bigchol.cu: 8N > 1024, C4:
4096 x 4096): the factor against LAPACK by backward error, alone and in batches, the status of non-SPD
systems against LAPACK's index, the factor of a damped J^T J of the 512-station problem, and the factor
fed to the blocked substitutions (kernels_bigtri.cu) against scipy's cho_solve."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import scipy.linalg as sla

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

dp_ = C.POINTER(C.c_double)
ip_ = C.POINTER(C.c_int)


def _factor(api, mats):
    """factor the list of symmetric matrices in place on the device; returns (lower factors, info)"""
    L = api.lib
    L.dirac_b200_big_factor.restype = C.c_int
    L.dirac_b200_big_factor.argtypes = [C.c_int, C.c_int, dp_, ip_]
    n = mats[0].shape[0]
    # column-major systems back to back: the row-major buffer of each transposed (A is symmetric)
    buf = np.ascontiguousarray(np.stack(mats))
    info = np.full(len(mats), -99, dtype=np.int32)
    rc = L.dirac_b200_big_factor(n, len(mats), buf.ctypes.data_as(dp_), info.ctypes.data_as(ip_))
    assert rc == 0
    # row-major view of a column-major lower factor is L^T: its upper triangle
    return [np.tril(b.T) for b in buf], info


def _spd(n, seed):
    rng = np.random.default_rng(seed)
    G = rng.standard_normal((n, n))
    return G @ G.T / n + np.eye(n)


def _backward(Lf, A):
    return np.linalg.norm(Lf @ Lf.T - A) / np.linalg.norm(A)


def _lapack_backward(A):
    c, info = sla.lapack.dpotrf(A, lower=1)
    assert info == 0
    return _backward(np.tril(c), A)


@pytest.mark.parametrize("n", [1032, 2056, 4096])
def test_factor_backward_error(api, n):
    A = _spd(n, n)
    (Lf,), info = _factor(api, [A])
    assert list(info) == [0]
    err = _backward(Lf, A)
    assert err < 1e-13, (err, _lapack_backward(A))


@pytest.mark.parametrize("n,nb", [(1032, 32), (2056, 5), (4096, 3)])
def test_batch_backward_error(api, n, nb):
    mats = [_spd(n, 100 * n + b) for b in range(nb)]
    Ls, info = _factor(api, mats)
    assert list(info) == [0] * nb
    for Lf, A in zip(Ls, mats):
        assert _backward(Lf, A) < 1e-13


def test_damped_jtj_of_512_stations(api):
    """J^T J + mu I of cluster 0 of the 512-station golden problem (8N = 4096), mu as LM's first"""
    import make_golden_n512 as gen
    from sagecal_b200 import lib as blib
    from sagecal_b200.dirac_api import SkyModel, make_barr
    pr = gen.build()
    dp = blib.DeviceProblem(api, pr.N, pr.Nbase, pr.tilesz, make_barr(pr.sta1, pr.sta2, pr.flag),
                            SkyModel(pr.clusters, pr.N), pr.coh, pr.x)
    try:
        _, JTJ, _ = dp.normal_eq(0, 0, np.ascontiguousarray(pr.pp0[:8 * pr.N]), pr.x)
    finally:
        dp.close()
    A = JTJ + 1e-3 * np.max(np.diag(JTJ)) * np.eye(JTJ.shape[0])
    (Lf,), info = _factor(api, [A])
    assert list(info) == [0]
    assert _backward(Lf, A) < 1e-13


def _spoiled(n, k, seed):
    """diagonally dominant SPD, made indefinite at pivot k (0-based): LAPACK's info is k + 1"""
    rng = np.random.default_rng(seed)
    S = rng.uniform(-1, 1, (n, n))
    A = (S + S.T) / n + 4 * np.eye(n)
    A[k, k] = -1.0
    return A


@pytest.mark.parametrize("k", [5, 600, 1030])
def test_info_matches_lapack(api, k):
    """first block, a middle block and the ragged last block (n = 1032: panels of 256, last of 8)"""
    n = 1032
    A = _spoiled(n, k, k)
    _, want = sla.lapack.dpotrf(A, lower=1)
    assert want == k + 1
    _, info = _factor(api, [A])
    assert list(info) == [want]


def test_info_flags_only_the_bad_system(api):
    n = 1032
    mats = [_spd(n, 7), _spoiled(n, 600, 1), _spd(n, 8), _spoiled(n, 1030, 2)]
    _, info = _factor(api, mats)
    assert list(info) == [0, 601, 0, 1031]


def test_factor_feeds_blocked_substitutions(api):
    """the factor as the LM's substitutions read it (column-major lower, ld = n)"""
    from sagecal_b200.dirac_api import dptr
    n = 4096
    A = _spd(n, 3)
    (Lf,), info = _factor(api, [A])
    assert list(info) == [0]
    b = np.random.default_rng(4).standard_normal(n)
    Lcol = np.asfortranarray(Lf)
    x = np.zeros(n)
    us = C.c_double(0.0)
    api.lib.dirac_b200_bigtri_solve.restype = C.c_int
    rc = api.lib.dirac_b200_bigtri_solve(n, Lcol.ctypes.data_as(dp_), dptr(b), dptr(x), 0, C.byref(us))
    assert rc == 0
    want = sla.cho_solve(sla.cho_factor(A, lower=True), b)
    assert np.max(np.abs(x - want)) <= 1e-10 * np.max(np.abs(want))
