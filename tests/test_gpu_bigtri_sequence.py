"""The blocked substitutions (kernels_bigtri.cu) the way the LM issues them: many solves back to back on
one workspace and one output vector, with no host synchronisation in between, alternating two factors
that cuSOLVER's dpotrf leaves on the device and several right-hand sides.  Every answer is checked
against scipy, so a solution slot left over from the previous solve shows up as a wrong answer."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _spd(n, seed):
    g = np.random.default_rng(seed).standard_normal((n, n))
    return g @ g.T / n + 0.5 * np.eye(n)


@pytest.mark.parametrize("n,nsolve", [(576, 9), (1024, 7), (4096, 8)])
def test_back_to_back_solves_alternating_factors(api, n, nsolve):
    import scipy.linalg as sla
    f = api.lib.dirac_b200_bigtri_sequence
    f.restype = C.c_int
    f.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    mats = [_spd(n, 2 * n), _spd(n, 2 * n + 1)]
    A = np.stack([np.asfortranarray(m) for m in mats]).copy()
    rng = np.random.default_rng(n)
    b = rng.standard_normal((nsolve, n))
    b[1] = b[0]          # the same right-hand side on the other factor
    b[3] = 1e3 * b[2]    # and a scaled one: answers differ from their predecessor's everywhere
    x = np.full((nsolve, n), np.nan)
    rc = f(n, 2, A.ctypes.data, nsolve, b.ctypes.data, x.ctypes.data, 0, None)
    assert rc == 0
    facs = [sla.cho_factor(m, lower=True) for m in mats]
    for s in range(nsolve):
        want = sla.cho_solve(facs[s % 2], b[s])
        err = np.max(np.abs(x[s] - want))
        assert err <= 1e-10 * np.max(np.abs(want)), (s, err)


def test_back_to_back_refuses_unhandled_sizes(api):
    f = api.lib.dirac_b200_bigtri_sequence
    f.restype = C.c_int
    f.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    assert f(512, 1, None, 1, None, None, 0, None) == -1
    assert f(600, 1, None, 1, None, None, 0, None) == -1


def test_back_to_back_reports_indefinite_matrix(api):
    n = 576
    f = api.lib.dirac_b200_bigtri_sequence
    f.restype = C.c_int
    f.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    A = np.asfortranarray(_spd(n, 5))
    A[100, 100] = -1.0
    b = np.ones(n)
    x = np.zeros(n)
    assert f(n, 1, A.ctypes.data, 1, b.ctypes.data, x.ctypes.data, 0, None) == -2
