"""Batched factor-only Cholesky of the LM's per-sweep batch (dirac_b200_chol_factor_batched) on a
seeded batch.  test_chol_solver.py imports `make_batch` / `factor_batched`, and runs this file in a
subprocess to see the batch under DIRAC_B200_BATCH_CL, which the library reads once per process:
`python chol_batch_check.py n nb out.npz`."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from sagecal_b200 import lib as blib  # noqa: E402


def make_batch(n, nb, seed):
    """nb SPD matrices (column-major, upper triangle NaN: it must never be read) and a different
    damping per matrix; returns (A [nb, n, n] as the device reads it, full symmetric A, mu)"""
    rng = np.random.default_rng(seed)
    full = np.empty((nb, n, n))
    for b in range(nb):
        B = rng.standard_normal((n, n + 8))
        full[b] = B @ B.T / (n + 8) + 0.05 * np.eye(n)
    mu = 10.0 ** rng.uniform(-3, 0, nb) * np.einsum("bii->b", full) / n
    poisoned = np.where(np.tril(np.ones((n, n), dtype=bool)), full, np.nan)
    # column-major: element (r, c) of matrix b at b*n*n + c*n + r
    return np.ascontiguousarray(np.swapaxes(poisoned, 1, 2)), full, mu


def factor_batched(n, A, mu):
    """returns (rc, factors [nb, ld, ld] as column-major matrices, info [nb, 2])"""
    L = blib.load().lib
    L.dirac_b200_chol_factor_batched.restype = C.c_int
    L.dirac_b200_chol_factor_batched.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 4
    nb = A.shape[0]
    ld = 32 * ((n + 31) // 32)
    out = np.zeros((nb, ld, ld))
    info = np.full((nb, 2), -7, dtype=np.int32)
    A = np.ascontiguousarray(A, dtype=np.float64)
    mu = np.ascontiguousarray(mu, dtype=np.float64)
    rc = L.dirac_b200_chol_factor_batched(n, nb, A.ctypes.data, mu.ctypes.data, out.ctypes.data,
                                          info.ctypes.data)
    return rc, np.swapaxes(out, 1, 2), info


def main():
    n, nb = int(sys.argv[1]), int(sys.argv[2])
    A, _, mu = make_batch(n, nb, seed=n + nb)
    rc, F, info = factor_batched(n, A, mu)
    np.savez(sys.argv[3], rc=rc, F=F, info=info)


if __name__ == "__main__":
    main()
