"""CPU: the arithmetic of the projectback manifold average (sagecal_b200/csrc/manifold_math.cuh, compiled
as host code from oracle/manifold_math_check.cu) against the compiled reference: the 2x2 polar factor
against zgesvd + U*VT as manifold_average.c forms it (my_zgesvd, my_zgemm), degenerate Grams included,
and the whole average against calculate_manifold_average_projectback (manifold_average.c:809) with
Nt = 1.  Also include/dirac_b200_federated.h: its declarations, and a plain C99 caller that links and is
refused before any device work.  Runs without a GPU."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from test_cpu_abi import _c_declarations

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
vp = C.c_void_p
i_ = C.c_int


@pytest.fixture(scope="session")
def chk(tmp_path_factory):
    """the harness, compiled by nvcc as host code into a temporary directory"""
    out = str(tmp_path_factory.mktemp("manifold") / "libmanifold_math_check.so")
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-Xcompiler", "-fPIC", "-shared", "-cudart",
                           "static", "-Wno-deprecated-gpu-targets", "-o", out,
                           os.path.join(ROOT, "oracle", "manifold_math_check.cu")])
    L = C.CDLL(out)
    L.check_polar.argtypes = [vp, vp]
    L.check_projectback.argtypes = [i_, i_, i_, vp, i_, vp]
    L.check_draws.argtypes = [i_, i_, vp]
    return L


def _p(a):
    return a.ctypes.data_as(vp)


def ref_polar(ref, G):
    """zgesvd('A','A') of the 2x2 G, then U*VT, as manifold_average.c:733-736 does"""
    L = ref.lib
    L.my_zgesvd.restype = i_
    L.my_zgesvd.argtypes = [C.c_char, C.c_char, i_, i_, vp, i_, vp, vp, i_, vp, i_, vp, i_, vp]
    A = np.ascontiguousarray(np.asarray(G, dtype=complex).T)  # column-major G
    S = np.zeros(2)
    U = np.zeros((2, 2), complex)    # column-major: U.T and VT.T are the matrices
    VT = np.zeros((2, 2), complex)
    work = np.zeros(64, complex)
    rwork = np.zeros(32)
    assert L.my_zgesvd(b"A", b"A", 2, 2, _p(A), 2, _p(S), _p(U), 2, _p(VT), 2, _p(work), 64,
                       _p(rwork)) == 0
    return U.T @ VT.T


def our_polar(chk, G):
    G = np.ascontiguousarray(G, dtype=complex)
    W = np.zeros((2, 2), complex)
    chk.check_polar(_p(G), _p(W))
    return W


def _cplx(rng, *shape):
    return rng.normal(size=shape) + 1j * rng.normal(size=shape)


# the Grams the average meets when a block is zero or has a zero Jones column: the zero Gram, rank 1
# with a zero second row (Y_f^H X for a zero second column of Y_f), zero first or second column
# (X^H Y_f), a single entry; and general Grams, complex and real
DEGENERATE = ["zero", "row2-zero", "col1-zero", "col2-zero", "single-entry", "general", "real"]


@pytest.mark.parametrize("case", DEGENERATE)
def test_polar_factor_is_zgesvd_s(ref, chk, case):
    rng = np.random.default_rng(DEGENERATE.index(case))
    for t in range(40):
        G = _cplx(rng, 2, 2)
        if case == "zero":
            G[:] = 0
        elif case == "row2-zero":
            G[1, :] = 0
        elif case == "col1-zero":
            G[:, 0] = 0
        elif case == "col2-zero":
            G[:, 1] = 0
        elif case == "single-entry":
            z = G[t % 2, (t // 2) % 2]
            G[:] = 0
            G[t % 2, (t // 2) % 2] = z
        elif case == "real":
            G = G.real + 0j
        want = ref_polar(ref, G)
        got = our_polar(chk, G)
        assert np.abs(got - want).max() <= 1e-12, (case, G, want, got)
        if case == "zero":
            assert np.array_equal(want, np.eye(2)) and np.array_equal(got, np.eye(2))
        if case in ("row2-zero", "col1-zero", "col2-zero", "single-entry"):
            # rank 1, yet the null-space part is zgesvd's: not the polar factor of a perturbed Gram
            assert np.abs(got @ got.conj().T - np.eye(2)).max() < 1e-14


def test_polar_factor_with_a_zero_first_row(ref, chk):
    """G = [[0, 0], [a, b]] (a block with a zero first Jones column projected onto another): zgesvd's
    first reflection leaves a rounding-sized d2 whose phase picks the first row of U V^H, so only the
    second row is defined.  The average multiplies that first row by the block's zero column."""
    rng = np.random.default_rng(11)
    for _ in range(40):
        G = _cplx(rng, 2, 2)
        G[0, :] = 0
        want = ref_polar(ref, G)
        got = our_polar(chk, G)
        assert np.abs(got[1] - want[1]).max() <= 1e-12
        assert np.abs(got @ got.conj().T - np.eye(2)).max() < 1e-14


def _blocks(rng, Nf, M, N, zero_block=False, zero_cols=False):
    Y = rng.normal(size=(Nf, M, 8 * N))
    if zero_block and Nf > 1:
        Y[1, 0] = 0.0
    if zero_cols and Nf > 2:
        for o in (2, 3, 6, 7):    # second Jones column of block 2
            Y[2, :, o::8] = 0.0
    if zero_cols and Nf > 3:
        for o in (0, 1, 4, 5):    # first Jones column of block 3
            Y[3, :, o::8] = 0.0
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


def our_projectback(chk, Y, Niter, randomize, seed):
    Nf, M, n8 = Y.shape
    B = Y.copy()
    cr = np.zeros(M, np.int32)
    if randomize:
        C.CDLL(None).srand(seed)
        chk.check_draws(M, Nf, _p(cr))
    chk.check_projectback(n8 // 8, M, Nf, _p(B), Niter, _p(cr))
    return B


@pytest.mark.parametrize("Nf", [1, 2, 3, 4])
@pytest.mark.parametrize("N", [1, 5, 62])
@pytest.mark.parametrize("randomize", [0, 1])
def test_projectback_matches_the_reference(ref, chk, Nf, N, randomize):
    rng = np.random.default_rng(1000 * Nf + 10 * N + randomize)
    for Niter, kw in ((10, {}), (2, dict(zero_block=True, zero_cols=True)), (0, {})):
        Y = _blocks(rng, Nf, 3, N, **kw)
        want = ref_projectback(ref, Y, Niter, randomize, 4242 + Niter)
        got = our_projectback(chk, Y, Niter, randomize, 4242 + Niter)
        assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max(), (Niter, kw)


def test_projectback_draws_follow_the_reference_order(ref, chk):
    """with randomize, chunk k projects first onto rand() % Nf drawn for k = 0..M-1 in order: a
    different seed gives a different answer, the same seed the reference's"""
    rng = np.random.default_rng(5)
    Y = _blocks(rng, 4, 6, 3)
    a = our_projectback(chk, Y, 0, 1, 1)
    b = our_projectback(chk, Y, 0, 1, 2)
    assert np.abs(a - b).max() > 1e-3
    want = ref_projectback(ref, Y, 0, 1, 2)
    assert np.abs(b - want).max() <= 1e-12 * np.abs(want).max()


# ---- header and C linkage --------------------------------------------------------------------------

def test_federated_header_matches_the_reference_and_the_library():
    """include/dirac_b200_federated.h declares calculate_manifold_average_projectback with the
    reference's own parameter type list (Dirac.h:1384, stored by
    tests/golden/make_golden_federated_signatures.py) and the library's own entry points; dirac_b200.h
    includes the header and declares none of its names"""
    from sagecal_b200 import lib as blib
    ours = _c_declarations(os.path.join(ROOT, "include", "dirac_b200_federated.h"))
    with open(os.path.join(ROOT, "tests", "golden", "ref_signatures_federated.json")) as f:
        refsig = json.load(f)
    assert sorted(ours) == sorted(blib.FEDERATED_EXPORTED)
    name = "calculate_manifold_average_projectback"
    assert sorted(refsig) == [name]
    assert ours[name][0] in refsig[name]
    assert [n for n in ours if not n.startswith("dirac_b200")] == [name]
    main = _c_declarations(os.path.join(ROOT, "include", "dirac_b200.h"))
    assert not set(main) & set(ours)
    assert '#include "dirac_b200_federated.h"' in open(os.path.join(ROOT, "include", "dirac_b200.h")).read()
    if os.path.exists(blib.LIB_PATH):
        L = C.CDLL(blib.LIB_PATH)
        for n in ours:
            assert hasattr(L, n), n


def test_plain_c_host_compiles_links_and_is_refused(tmp_path):
    exe = os.path.join(str(tmp_path), "federated_caller")
    libdir = os.path.join(ROOT, "sagecal_b200")
    subprocess.check_call(["gcc", "-std=c99", "-O1", "-Wall", "-Wextra", "-Werror", "-o", exe,
                           os.path.join(ROOT, "tests", "c_caller", "federated_caller.c"),
                           "-I", os.path.join(ROOT, "include"), "-L", libdir, "-ldirac_b200", "-lm",
                           "-Wl,-rpath," + libdir])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "FEDERATED_CALLER OK" in out.stdout, (out.stdout, out.stderr)
    assert "Nf = 0 must be at least 1" in out.stderr and "Niter = -1 at least 0" in out.stderr
    assert "admm = -1 at least 0" in out.stderr
    assert "nadmm = 0 ADMM iterations" in out.stderr
