"""CPU, no GPU: the stochastic closing stage of sagefit (lbfgs_m < 0 with a robust solver_mode) as
the library runs it on the host, minibatch::lbfgs_fit_robust_wrapper_minibatch (minibatch_algo.h),
against the compiled reference's lbfgs_fit_robust_wrapper_minibatch (robust_batchmode_lbfgs.c:859-930).

The cost and gradient of a row window are supplied by the reference's own full-interval Student's-t
cost and gradient with every row outside the window flagged and its data zeroed: rows outside the
window then contribute nothing, as in robust_cost_func_batch / robust_grad_func_batch, and the
minibatch gradient is the negative of the full-batch one (DESIGN.md §7 item 8)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from util import small_problem, relerr
from sagecal_b200.dirac_api import make_barr, dptr, c_double_p

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COST_FN = C.CFUNCTYPE(C.c_double, c_double_p, C.c_longlong, C.c_longlong)
GRAD_FN = C.CFUNCTYPE(None, c_double_p, c_double_p, C.c_longlong, C.c_longlong)


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("mbwin") / "libminibatch_window.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-Wall", "-Werror", "-shared", "-o", so,
                           os.path.join(ROOT, "tests", "c_caller", "minibatch_window.cpp")])
    L = C.CDLL(so)
    L.window_fit.argtypes = [COST_FN, GRAD_FN, c_double_p, C.c_int, C.c_longlong, C.c_int, C.c_int]
    L.window_table.argtypes = [C.c_longlong, C.c_int, C.POINTER(C.c_longlong),
                               C.POINTER(C.c_longlong)]
    return L


def table(L, n):
    off = (C.c_longlong * 5)()
    ln = (C.c_longlong * 5)()
    L.window_table(n, 5, off, ln)
    return list(zip(off, ln))


def windowed(b, r0, nr):
    """barr and data of the problem with every row outside [r0, r0 + nr) flagged and zeroed"""
    pr = b.pr
    rows = np.arange(pr.Nbase1)
    out = (rows < r0) | (rows >= r0 + nr)
    flag = pr.flag.copy()
    flag[out] = 1
    x = pr.x.reshape(-1, 8).copy()
    x[out] = 0.0
    return make_barr(pr.sta1, pr.sta2, flag), x.reshape(-1)


@pytest.mark.parametrize("n", [1, 3, 4, 5, 6, 7, 11, 360, 396, 2415 * 3])
def test_batch_table(harness, n):
    """lbfgs_persist_init's table over n rows (lbfgs.c:997-1008): ceil(n/5) rows per window, the last
    non-empty one short; with fewer rows than windows the trailing windows are empty"""
    b = (n + 4) // 5
    got = table(harness, n)
    covered = []
    for i, (off, ln) in enumerate(got):
        assert off == i * b
        assert ln == min(b, n - i * b)
        covered += list(range(off, off + max(ln, 0)))
    assert covered == list(range(n))


CASES = [
    # 360 rows, windows of 72 = 2 timeslots; the hybrid cluster's row map and tile map agree
    ("hybrid", dict(N=9, M=3, tilesz=10, seed=91, nchunk=[1, 2, 1], outliers=0.02)),
    # 3 chunks over 11 timeslots, 80-row windows cut timeslots of 36 rows
    ("uneven-cut", dict(N=9, M=3, tilesz=11, seed=92, nchunk=[3, 1, 2], outliers=0.02)),
    # flagged and uv-cut rows, 63-row windows cut timeslots of 45 rows
    ("flags-cut", dict(N=10, M=2, tilesz=7, seed=93, flag_frac=0.3, uvcut_frac=0.05, outliers=0.02)),
]


@pytest.mark.parametrize("name,prob", CASES, ids=[c[0] for c in CASES])
def test_wrapper_matches_reference(harness, ref, name, prob):
    """the product's wrapper on the reference's windowed evaluators against the reference's own
    lbfgs_fit_robust_wrapper_minibatch, max_lbfgs = 10 (3 epochs of 5 windows), memory 7: Jones to
    1e-9"""
    b = small_problem(**prob)
    pr = b.pr
    nu, itmax, M = 4.5, 10, 7
    rng = np.random.default_rng(5)
    p0 = pr.pp0 + 0.05 * rng.normal(0, 1, pr.pp0.shape)
    m, n = len(p0), 8 * pr.Nbase1
    # the reference stage, driven with a me_data_t as lmfit.c:1029 drives it
    L = ref.lib
    L.lbfgs_fit_robust_wrapper_minibatch.restype = C.c_int
    L.lbfgs_fit_robust_wrapper_minibatch.argtypes = [c_double_p, c_double_p, C.c_int, C.c_int, C.c_int,
                                                     C.c_int, C.c_int, C.c_void_p]
    md = ref.me_data(pr.N, pr.Nbase, pr.tilesz, b.fresh_barr(), b.sky, pr.coh, robust_nu=nu)
    p_ref = p0.copy()
    x = pr.x.copy()
    L.lbfgs_fit_robust_wrapper_minibatch(dptr(p_ref), dptr(x), m, n, itmax, M, 0, md)

    # the product's control flow on windowed reference evaluators
    wins = {}
    for off, ln in table(harness, pr.Nbase1):
        if ln > 0:
            barr, xw = windowed(b, off, ln)
            wins[(off, ln)] = (ref.me_data(pr.N, pr.Nbase, pr.tilesz, barr, b.sky, pr.coh, robust_nu=nu),
                               xw)

    def cost(p, r0, nr):
        md_w, xw = wins[(r0, nr)]
        return ref.cost(np.ctypeslib.as_array(p, (m,)).copy(), xw, md_w, robust=True)

    def grad(p, g, r0, nr):
        md_w, xw = wins[(r0, nr)]
        gw = ref.grad(np.ctypeslib.as_array(p, (m,)).copy(), xw, md_w, robust=True)
        np.ctypeslib.as_array(g, (m,))[:] = -gw

    cf, gf = COST_FN(cost), GRAD_FN(grad)
    p_got = p0.copy()
    harness.window_fit(cf, gf, dptr(p_got), m, pr.Nbase1, itmax, M)
    assert relerr(p_ref, p0) > 1e-6            # the stage moved the Jones
    assert relerr(p_got, p_ref) < 1e-9, relerr(p_got, p_ref)
