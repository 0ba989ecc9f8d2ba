"""Cluster Cholesky solver (kernels_chol.cu) against numpy on SPD systems of the sizes the LM uses."""
import ctypes as C

import numpy as np
import pytest

from sagecal_b200 import lib as blib

pytestmark = pytest.mark.gpu


def _solve(n, A, b, mu):
    api = blib.load()
    L = api.lib
    L.dirac_b200_spd_solve.restype = C.c_int
    L.dirac_b200_spd_solve.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_void_p]
    x = np.zeros(n)
    info = np.zeros(2, dtype=np.int32)
    A = np.asfortranarray(A)
    rc = L.dirac_b200_spd_solve(n, A.ctypes.data, b.ctypes.data, mu, x.ctypes.data, info.ctypes.data)
    return rc, x, int(info[0])


@pytest.mark.parametrize("n", [8, 31, 32, 33, 64, 200, 496, 512])
def test_spd_solve_matches_numpy(n):
    rng = np.random.default_rng(n)
    J = rng.standard_normal((2 * n, n))
    A = J.T @ J
    b = rng.standard_normal(n)
    mu = 1e-3 * np.max(np.diag(A))
    rc, x, info = _solve(n, A, b, mu)
    assert rc == 0 and info == 0
    ref = np.linalg.solve(A + mu * np.eye(n), b)
    # tolerance: backward-stable factorisation, cond ~1e3..1e4
    assert np.max(np.abs(x - ref)) <= 1e-10 * np.max(np.abs(ref))


def test_spd_solve_only_reads_lower_triangle():
    n = 100
    rng = np.random.default_rng(1)
    J = rng.standard_normal((3 * n, n))
    A = J.T @ J
    b = rng.standard_normal(n)
    Al = np.tril(A) + np.triu(np.full((n, n), np.nan), 1)
    rc, x, info = _solve(n, Al, b, 0.5)
    assert rc == 0 and info == 0
    ref = np.linalg.solve(A + 0.5 * np.eye(n), b)
    assert np.allclose(x, ref, rtol=1e-10, atol=1e-12)


def test_spd_solve_reports_failing_pivot():
    n = 96
    A = np.eye(n)
    A[40, 40] = -1.0
    b = np.ones(n)
    rc, x, info = _solve(n, A, b, 0.0)
    assert rc == 0 and info == 41


def _tri_solve(n, F, b):
    """the solve-only kernel on a column-major factor F: dirac_b200_tri_solve for ld = n,
    dirac_b200_tri_solve_ld for ld = F.shape[0] > n"""
    L = blib.load().lib
    F = np.asfortranarray(F)
    x = np.zeros(n)
    if F.shape[0] == n:
        L.dirac_b200_tri_solve.restype = C.c_int
        L.dirac_b200_tri_solve.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                           C.c_void_p]
        rc = L.dirac_b200_tri_solve(n, F.ctypes.data, b.ctypes.data, x.ctypes.data, 0, None)
    else:
        L.dirac_b200_tri_solve_ld.restype = C.c_int
        L.dirac_b200_tri_solve_ld.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                              C.c_int, C.c_void_p]
        rc = L.dirac_b200_tri_solve_ld(n, F.ctypes.data, F.shape[0], b.ctypes.data, x.ctypes.data, 0,
                                       None)
    return rc, x


def _padded_ld(n):
    return 32 * ((n + 31) // 32)


# ld = n: the factor as LAPACK / cuSOLVER leave it; ld = 32*ceil(n/32): as the batched factorisation
# leaves it (n = 496, the C2 / C3 systems: ld = 512)
TRI_CASES = ([pytest.param(n, n, id=str(n)) for n in (16, 33, 250, 496, 512)]
             + [pytest.param(n, _padded_ld(n), id="%d-ld%d" % (n, _padded_ld(n))) for n in (16, 33, 250, 496)])


@pytest.mark.parametrize("n,ld", TRI_CASES)
def test_tri_solve_matches_numpy(n, ld):
    """Solve-only cluster kernel on a factor laid out as LAPACK/cuSOLVER leave it (lower, ld = n)
    or as the batched factorisation leaves it (ld = 32*ceil(n/32))"""
    rng = np.random.default_rng(100 + n)
    J = rng.standard_normal((2 * n, n))
    A = J.T @ J + 0.1 * np.eye(n)
    fac = np.linalg.cholesky(A)
    # upper triangle and the padding rows poisoned: they must never be read
    Lf = np.full((ld, n), np.nan)
    Lf[:n] = np.tril(fac) + np.triu(np.full((n, n), np.nan), 1)
    b = rng.standard_normal(n)
    rc, x = _tri_solve(n, Lf, b)
    if rc == -1:
        pytest.skip("cluster size on this device too small for the solve-only kernel")
    ref = np.linalg.solve(A, b)
    assert np.max(np.abs(x - ref)) <= 1e-10 * np.max(np.abs(ref))


def _check_factors(n, full, mu, F, info):
    """backward error of every factor and forward error against LAPACK's"""
    eps = np.finfo(np.float64).eps
    for b in range(full.shape[0]):
        assert info[b, 0] == 0, (b, info[b])
        Ad = full[b] + mu[b] * np.eye(n)
        Lg = np.tril(F[b, :n, :n])
        bwd = np.linalg.norm(Lg @ Lg.T - Ad) / np.linalg.norm(Ad)
        assert bwd <= 4 * n * eps, (b, bwd)
        # (make_batch's matrices have eigenvalues in [0.05, ~5]: the forward error is ~cond * eps)
        Lw = np.linalg.cholesky(Ad)
        assert np.linalg.norm(Lg - Lw) <= 1e-12 * np.linalg.norm(Lw), b


BATCHES = ([(n, 34) for n in (8, 24, 32, 40, 264, 496, 504, 512)]
           + [(496, nb) for nb in (1, 33, 64, 100)])


@pytest.mark.parametrize("n,nb", BATCHES, ids=["n%d-nb%d" % c for c in BATCHES])
def test_chol_factor_batched_matches_numpy(n, nb):
    """factor-only k_chol_solve over a batch (more matrices than clusters in flight from 34 on), a
    different damping per matrix read from the device; the factors at ld = 32*ceil(n/32)"""
    from chol_batch_check import factor_batched, make_batch
    A, full, mu = make_batch(n, nb, seed=n + nb)
    rc, F, info = factor_batched(n, A, mu)
    if rc == -1:
        pytest.skip("the device grants no cluster for the batched factorisation")
    _check_factors(n, full, mu, F, info)


def test_chol_factor_batched_failing_matrix_is_isolated():
    """one indefinite matrix in the middle of a batch: its info is dpotrf's pivot, and every other
    factor is bit for bit the one of the batch without it"""
    import scipy.linalg.lapack as lapack
    from chol_batch_check import factor_batched, make_batch
    n, nb, bad = 264, 34, 17
    A, full, mu = make_batch(n, nb, seed=5)
    rc, F0, info0 = factor_batched(n, A, mu)
    if rc == -1:
        pytest.skip("the device grants no cluster for the batched factorisation")
    Abad = A.copy()
    Abad[bad, 150, 150] = -1.0          # column-major: (150, 150)
    assert not info0[:, 0].any()
    rc, F1, info1 = factor_batched(n, Abad, mu)
    want = full[bad] + mu[bad] * np.eye(n)
    want[150, 150] = -1.0 + mu[bad]
    _, piv = lapack.dpotrf(want, lower=1)
    assert piv > 0 and info1[bad, 0] == piv, (info1[bad], piv)
    others = [b for b in range(nb) if b != bad]
    assert np.array_equal(F1[others], F0[others])
    assert not info1[others, 0].any()


def test_chol_factor_then_padded_solve():
    """the LM's chained path: batched factorisation, then the solve-only kernel on each factor at
    the padded leading dimension (n = 496: ld = 512, the C2 / C3 systems)"""
    from chol_batch_check import factor_batched, make_batch
    n, nb = 496, 3
    A, full, mu = make_batch(n, nb, seed=9)
    rc, F, info = factor_batched(n, A, mu)
    if rc == -1:
        pytest.skip("the device grants no cluster for the batched factorisation")
    assert not info[:, 0].any()
    rng = np.random.default_rng(2)
    for b in range(nb):
        rhs = rng.standard_normal(n)
        rc, x = _tri_solve(n, F[b, :, :n], rhs)
        assert rc == 0
        want = np.linalg.solve(full[b] + mu[b] * np.eye(n), rhs)
        assert np.max(np.abs(x - want)) <= 1e-10 * np.max(np.abs(want))


@pytest.mark.parametrize("cl", [1, 2, 8, 16])
def test_chol_factor_batched_cluster_shapes(cl, tmp_path):
    """the batch with 1-, 2-, 8- and 16-CTA clusters per matrix (DIRAC_B200_BATCH_CL, read once
    per process: one subprocess each)"""
    import os
    import subprocess
    import sys
    from chol_batch_check import make_batch
    n, nb = 496, 34
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), "chol_batch_check.py")
    env = dict(os.environ)
    env["DIRAC_B200_BATCH_CL"] = str(cl)
    out_path = str(tmp_path / "f.npz")
    out = subprocess.run([sys.executable, script, str(n), str(nb), out_path], env=env,
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    z = np.load(out_path)
    if int(z["rc"]) == -1:
        pytest.skip("the device grants no cluster for the batched factorisation")
    _, full, mu = make_batch(n, nb, seed=n + nb)
    _check_factors(n, full, mu, z["F"], z["info"])


def test_pivot_rsqrt_accuracy():
    """The branch-free 1/sqrt of the pivot chain (hardware seed + one cubic correction)."""
    api = blib.load()
    L = api.lib
    L.dirac_b200_test_rsqrt.restype = C.c_int
    L.dirac_b200_test_rsqrt.argtypes = [C.c_int, C.c_void_p, C.c_void_p]
    rng = np.random.default_rng(7)
    x = np.concatenate([10.0 ** rng.uniform(-30, 30, 200000), rng.uniform(0.5, 4.0, 200000)])
    y = np.zeros_like(x)
    L.dirac_b200_test_rsqrt(x.size, x.ctypes.data, y.ctypes.data)
    ref = 1.0 / np.sqrt(x.astype(np.longdouble))
    rel = np.max(np.abs((y - ref) / ref).astype(np.float64))
    assert rel <= 4 * np.finfo(np.float64).eps, rel


@pytest.mark.parametrize("n", [576, 1024, 4096])
def test_bigtri_solve_matches_numpy(api, n):
    """blocked dataflow substitutions for systems beyond the cluster kernels (8N > 512) against
    scipy on the same factor"""
    import ctypes as C
    import scipy.linalg as sla
    from sagecal_b200.dirac_api import dptr
    rng = np.random.default_rng(n)
    A = rng.normal(0, 1, (n, n))
    A = A @ A.T / n + np.eye(n) * 0.5
    Lf = np.linalg.cholesky(A)
    b = rng.normal(0, 1, n)
    want = sla.cho_solve((Lf, True), b)
    Lcol = np.asfortranarray(Lf)          # column-major lower, ld = n
    x = np.zeros(n)
    us = C.c_double(0.0)
    api.lib.dirac_b200_bigtri_solve.restype = C.c_int
    rc = api.lib.dirac_b200_bigtri_solve(n, Lcol.ctypes.data_as(C.POINTER(C.c_double)), dptr(b), dptr(x), 20,
                                         C.byref(us))
    assert rc == 0
    assert np.max(np.abs(x - want)) <= 1e-10 * np.max(np.abs(want))
    print("bigtri n=%d: %.1f us per solve" % (n, us.value))
