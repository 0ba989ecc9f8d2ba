"""GPU tier of the projectback manifold average (calculate_manifold_average_projectback,
manifold_average.c:809; k_manifold_projectback): the library's export against the compiled reference
with Nt = 1, at small shapes (randomised first projections, a zero block and zero Jones columns, up to
the 64 solutions the kernel takes) and at the C4 shape (N Npoly = 1536, 256 chunks, 8 solutions, 10
rounds), bit-identical from run to run; the device-pointer form against the export; the refusals.

The tests call the reference first and the product library afterwards, so that the reference's answers
can be recorded (tests/golden/ref/test_gpu_federated)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
vp = C.c_void_p
i_ = C.c_int


def _p(a):
    return a.ctypes.data_as(vp)


def _blocks(rng, Nf, M, n, degenerate=False):
    Y = rng.normal(size=(Nf, M, 8 * n))
    if degenerate and Nf > 3:
        Y[1, 0] = 0.0                       # a zero block
        for o in (2, 3, 6, 7):
            Y[2, :, o::8] = 0.0             # a zero second Jones column
        for o in (0, 1, 4, 5):
            Y[3, :, o::8] = 0.0             # a zero first Jones column
    return Y


def ref_projectback(ref, Y, Niter, randomize, seed):
    Nf, M, n8 = Y.shape
    A = Y.copy()
    L = ref.lib
    L.calculate_manifold_average_projectback.restype = i_
    L.calculate_manifold_average_projectback.argtypes = [i_, i_, i_, vp, i_, i_, i_]
    C.CDLL(None).srand(seed)
    assert L.calculate_manifold_average_projectback(n8 // 8, M, Nf, _p(A), Niter, randomize, 1) == 0
    return A


def ours(api, Y, Niter, randomize, seed):
    B = Y.copy()
    C.CDLL(None).srand(seed)
    assert api.manifold_projectback(B, Niter, randomize) == 0
    return B


def _check(got, want, tol=1e-12):
    """to tol of the largest value; a large reference answer is stored as a sample (NaN elsewhere)"""
    m = ~np.isnan(want)
    assert m.any()
    assert np.abs(got[m] - want[m]).max() <= tol * np.abs(want[m]).max()


SMALL = [(1, 62, 4, 10, 0), (2, 62, 4, 10, 1), (3, 124, 5, 10, 1), (4, 186, 3, 2, 0),
         (8, 300, 3, 10, 1), (64, 5, 2, 3, 1)]


@pytest.mark.parametrize("Nf,n,M,Niter,randomize", SMALL)
def test_export_matches_the_reference(ref, api, Nf, n, M, Niter, randomize):
    rng = np.random.default_rng(Nf * 100 + n)
    Y = _blocks(rng, Nf, M, n, degenerate=True)
    want = ref_projectback(ref, Y, Niter, randomize, 17)
    got = ours(api, Y, Niter, randomize, 17)
    _check(got, want)
    again = ours(api, Y, Niter, randomize, 17)
    assert np.array_equal(got, again)


def test_export_at_the_c4_shape(ref, api):
    """N Npoly = 512 x 3, 256 chunks, 8 solutions, 10 rounds (the stochastic master's first ADMM
    iteration at 512 stations): 201 MB in"""
    rng = np.random.default_rng(4)
    Y = _blocks(rng, 8, 256, 1536)
    want = ref_projectback(ref, Y, 10, 1, 99)
    got = ours(api, Y, 10, 1, 99)
    _check(got, want)
    again = ours(api, Y, 10, 1, 99)
    assert np.array_equal(got, again)


def test_device_form_equals_the_export(api):
    """dirac_b200_manifold_projectback_dev on a resident tensor with the same draws as the export"""
    import torch
    rng = np.random.default_rng(8)
    Nf, M, n = 5, 7, 93
    Y = _blocks(rng, Nf, M, n, degenerate=True)
    want = ours(api, Y, 10, 1, 5)
    C.CDLL(None).srand(5)
    libc = C.CDLL(None)
    cr = np.array([libc.rand() % Nf for _ in range(M)], np.int32)
    dY = torch.from_numpy(Y).cuda()
    assert api.manifold_projectback_dev(dY, 10, cr) == 0
    torch.cuda.synchronize()
    assert np.array_equal(dY.cpu().numpy(), want)
    # no draws: every chunk projects onto solution 0, as randomize = 0
    want0 = ours(api, Y, 2, 0, 0)
    dY = torch.from_numpy(Y).cuda()
    assert api.manifold_projectback_dev(dY, 2) == 0
    torch.cuda.synchronize()
    assert np.array_equal(dY.cpu().numpy(), want0)


def test_refusals_touch_nothing(api):
    import torch
    Y = np.full((65, 1, 8), 7.0)
    assert api.manifold_projectback(Y, 10) == -1           # more solutions than the kernel takes
    Y2 = np.full((2, 1, 8), 7.0)
    assert api.manifold_projectback(Y2, -1) == -1
    assert (Y == 7).all() and (Y2 == 7).all()
    dY = torch.full((2, 3, 8), 7.0, dtype=torch.float64, device="cuda")
    assert api.manifold_projectback_dev(dY, 1, np.array([0, 2, 1], np.int32)) == -1   # cr[1] >= Nf
    torch.cuda.synchronize()
    assert (dY == 7).all()
