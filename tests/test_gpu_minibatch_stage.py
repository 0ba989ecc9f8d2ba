"""GPU: the stochastic closing stage of sagefit (lbfgs_m < 0 with a robust solver_mode, lmfit.c:1027-1029).

* the row-window Student's-t cost and gradient (dirac_b200_cost_window / dirac_b200_grad_window, the
  windowed k_stream_all and k_grad_tma_window passes) against the compiled reference's full-interval
  cost and gradient with every row outside the window flagged and zeroed, which is what the
  reference's robust_cost_func_batch / robust_grad_func_batch compute (the gradient negated);
* sagefit_visibilities(..., lbfgs_m=-7) under solver_mode 2, 3, 5 and 6 against the reference, with
  the stage alone (max_emiter=0) and behind a SAGE sweep;
* the sharded stage on two GPUs against one (tests/minibatch_stage_check.py).

The reference calls come before the device is touched, so that their answers can be recorded on a
machine without a GPU."""
import os
import subprocess
import sys

import numpy as np
import pytest

from util import small_problem, perturbed_jones, relerr
from sagecal_b200 import lib as blib
from sagecal_b200.dirac_api import make_barr

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JONES_TOL = 1e-5


def device_api():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return blib.load()


def batch_table(n):
    b = (n + 4) // 5
    return [(i * b, min(b, n - i * b)) for i in range(5)]


def windowed(b, r0, nr):
    pr = b.pr
    rows = np.arange(pr.Nbase1)
    out = (rows < r0) | (rows >= r0 + nr)
    flag = pr.flag.copy()
    flag[out] = 1
    x = pr.x.reshape(-1, 8).copy()
    x[out] = 0.0
    return make_barr(pr.sta1, pr.sta2, flag), x.reshape(-1)


WINDOW_CASES = [
    ("hybrid", dict(N=9, M=3, tilesz=10, seed=91, nchunk=[1, 2, 1], outliers=0.02)),
    ("uneven-cut", dict(N=9, M=3, tilesz=11, seed=92, nchunk=[3, 1, 2], outliers=0.02)),
    ("flags-cut", dict(N=10, M=2, tilesz=7, seed=93, flag_frac=0.3, uvcut_frac=0.05, outliers=0.02)),
    # more than 64 stations: several tiles of stations, windows of 1449 rows cut timeslots of 2415
    ("n70", dict(N=70, M=2, tilesz=3, seed=94, nchunk=[1, 2], outliers=0.02)),
    # 62 stations, windows over one to two of 13 timeslots and a time block of the gradient pass cut
    ("n62-ragged", dict(N=62, M=2, tilesz=13, seed=95, outliers=0.02)),
]


@pytest.mark.parametrize("name,prob", WINDOW_CASES, ids=[c[0] for c in WINDOW_CASES])
def test_window_cost_and_grad(ref, name, prob):
    b = small_problem(**prob)
    pr = b.pr
    pp = perturbed_jones(pr, seed=9)
    nu = 3.5
    wins = [w for w in batch_table(pr.Nbase1) if w[1] > 0] + [(0, pr.Nbase1)]
    want = []
    for r0, nr in wins:
        barr, xw = windowed(b, r0, nr)
        md = ref.me_data(pr.N, pr.Nbase, pr.tilesz, barr, b.sky, pr.coh, robust_nu=nu)
        want.append((ref.cost(pp, xw, md, robust=True), -ref.grad(pp, xw, md, robust=True)))
    api = device_api()
    with blib.DeviceProblem(api, pr.N, pr.Nbase, pr.tilesz, b.barr, b.sky, pr.coh, pr.x) as dp:
        got = [(dp.cost_window(pp, r0, nr, nu), dp.grad_window(pp, r0, nr, nu)) for r0, nr in wins]
        full_c = dp.cost(pp, robust=True, nu=nu)
        full_g = dp.grad(pp, robust=True, nu=nu)
        empty = (dp.cost_window(pp, pr.Nbase1, 0, nu), dp.grad_window(pp, pr.Nbase1, -3, nu))
    for (r0, nr), (cw, gw), (c, g) in zip(wins, want, got):
        assert abs(c - cw) <= 1e-12 * abs(cw), (r0, nr, c, cw)
        assert relerr(g, gw) < 1e-11, (r0, nr, relerr(g, gw))
    # the five windows tile the interval; the full window is the full-interval pass
    assert abs(sum(c for c, _ in got[:-1]) - full_c) <= 1e-12 * full_c
    assert abs(got[-1][0] - full_c) <= 1e-14 * full_c
    assert relerr(got[-1][1], -full_g) < 1e-12
    assert empty[0] == 0.0 and not np.any(empty[1])


def test_window_empty_when_fewer_rows_than_windows():
    """3 rows, 5 windows: the last two windows of the batch table are empty (cost 0, gradient 0)"""
    b = small_problem(N=3, M=1, tilesz=1, seed=96)
    pr = b.pr
    assert pr.Nbase1 == 3
    pp = perturbed_jones(pr, seed=9)
    api = device_api()
    with blib.DeviceProblem(api, pr.N, pr.Nbase, pr.tilesz, b.barr, b.sky, pr.coh, pr.x) as dp:
        tab = batch_table(pr.Nbase1)
        assert [w[1] for w in tab] == [1, 1, 1, 0, -1]
        cs = [dp.cost_window(pp, r0, nr, 2.0) for r0, nr in tab]
        gs = [dp.grad_window(pp, r0, nr, 2.0) for r0, nr in tab]
        full = dp.cost(pp, robust=True, nu=2.0)
        gfull = dp.grad(pp, robust=True, nu=2.0)
    assert cs[3] == 0.0 and cs[4] == 0.0
    assert not np.any(gs[3]) and not np.any(gs[4])
    assert abs(sum(cs) - full) <= 1e-13 * full
    assert relerr(sum(gs), -gfull) < 1e-13


STAGE_CASES = [
    (2, dict(N=9, M=3, tilesz=10, seed=97, nchunk=[1, 2, 1], outliers=0.02)),
    (3, dict(N=9, M=3, tilesz=10, seed=97, nchunk=[1, 2, 1], outliers=0.02)),
    (5, dict(N=9, M=3, tilesz=10, seed=97, nchunk=[1, 2, 1], outliers=0.02)),
    (6, dict(N=9, M=3, tilesz=10, seed=97, nchunk=[1, 2, 1], outliers=0.02)),
]


def run_both(lib_ref, b, kw):
    pr = b.pr
    out = []
    x = pr.x.copy()
    pp = pr.pp0.copy()
    r = lib_ref.sagefit_visibilities(pr.u, pr.v, pr.w, x, pr.N, pr.Nbase, pr.tilesz, b.fresh_barr(),
                                     b.sky, pr.coh, pp, **kw)
    out.append((r, x, pp))
    api = device_api()
    x = pr.x.copy()
    pp = pr.pp0.copy()
    r = api.sagefit_visibilities(pr.u, pr.v, pr.w, x, pr.N, pr.Nbase, pr.tilesz, b.fresh_barr(), b.sky,
                                 pr.coh, pp, **kw)
    out.append((r, x, pp))
    return out


def check_parity(pr, out, tag):
    (rr, xr, ppr), (rg, xg, ppg) = out
    assert rr[0] == rg[0], tag
    assert abs(rr[1] - rg[1]) < 1e-9, tag                    # mean nu
    assert abs(rr[2] - rg[2]) <= 1e-10 * rr[2], tag          # res_0
    assert relerr(ppg, ppr) < JONES_TOL, (tag, relerr(ppg, ppr))
    assert relerr(xg, xr) < 1e-5 * max(1.0, np.max(np.abs(pr.x)) / np.max(np.abs(xr))), tag
    assert abs(rr[3] - rg[3]) <= 1e-5 * rr[3], (tag, rr[3], rg[3])   # res_1


@pytest.mark.parametrize("emiter", [0, 2], ids=["stage", "full"])
@pytest.mark.parametrize("mode,prob", STAGE_CASES, ids=["mode%d" % c[0] for c in STAGE_CASES])
def test_sagefit_minibatch_stage(ref, refser, mode, prob, emiter):
    """lbfgs_m = -7: the reference's stochastic LBFGS over 5 row windows (3 epochs at max_lbfgs = 10);
    robust RTR / NSD (5, 6) against the reference build with serialised worker threads"""
    b = small_problem(**prob)
    kw = dict(max_emiter=emiter, max_iter=2, max_lbfgs=10, lbfgs_m=-7, randomize=0, solver_mode=mode)
    out = run_both(refser if mode in (5, 6) else ref, b, kw)
    check_parity(b.pr, out, (mode, emiter))


def test_sagefit_minibatch_stage_16_stations(ref):
    b = small_problem(N=16, M=3, tilesz=8, seed=98, outliers=0.02, flag_frac=0.1)
    kw = dict(max_emiter=2, max_iter=2, max_lbfgs=10, lbfgs_m=-7, randomize=0, solver_mode=2)
    check_parity(b.pr, run_both(ref, b, kw), "n16")


def test_positive_memory_keeps_the_full_batch_stage(ref):
    """lbfgs_m = +7 still runs the full-batch LBFGS (the reference's answer), and -7 is another stage"""
    b = small_problem(**STAGE_CASES[0][1])
    kw = dict(max_emiter=0, max_iter=2, max_lbfgs=10, lbfgs_m=7, randomize=0, solver_mode=2)
    out = run_both(ref, b, kw)
    check_parity(b.pr, out, "m+7")
    api = device_api()
    pr = b.pr
    pp = pr.pp0.copy()
    x = pr.x.copy()
    api.sagefit_visibilities(pr.u, pr.v, pr.w, x, pr.N, pr.Nbase, pr.tilesz, b.fresh_barr(), b.sky, pr.coh,
                             pp, **dict(kw, lbfgs_m=-7))
    assert relerr(pp, out[1][2]) > 1e-6


def test_sharded_stage_matches_single_gpu():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", "29619",
           os.path.join(ROOT, "tests", "minibatch_stage_check.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    print(out.stdout[-3000:], out.stderr[-3000:])
    assert out.returncode == 0 and "MINIBATCH_STAGE_CHECK OK" in out.stdout
