"""The stochastic LBFGS stage of sagefit (lbfgs_m < 0, robust solver_mode) at the C3 shape (62 stations,
64 clusters, 120 timeslots, robust data): stage time with lbfgs_m = +7 (full-batch LBFGS) and -7 (5 row
windows), its host / device split, and CUDA-event time and bytes/s of one windowed cost and gradient
pass against the full-interval passes.  Prints one JSON line; with --out, writes it there too.

    python profiles/minibatch_stage.py [--reps 20] [--max-lbfgs 10] [--out FILE]

Bytes per pass are what the pass has to move: coherencies of every cluster plus data, flags and (for
the gradient's cost pass) residual of the rows it covers (problem.cu, db_prof_begin)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sagecal_b200 import synth, lib as blib  # noqa: E402
from sagecal_b200.dirac_api import SkyModel, make_barr  # noqa: E402


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        out = "unavailable (%s)" % e
    return name, out


def kernel_ms(api, kind):
    """(launches, ms, bytes) of the passes of one kind timed since profiling was enabled"""
    import ctypes as C
    api.lib.dirac_b200_profile_read.argtypes = [C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double)]
    a, b = C.c_double(0), C.c_double(0)
    n = api.lib.dirac_b200_profile_read(kind, C.byref(a), C.byref(b))
    return n, a.value, b.value


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--max-lbfgs", type=int, default=10)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("minibatch_stage.py measures on a GPU; none is visible")
    api = blib.load()
    api.lib.dirac_b200_profile_enable.argtypes = [__import__("ctypes").c_int]
    pr = synth.make_config("C3")
    barr = make_barr(pr.sta1, pr.sta2, pr.flag)
    sky = SkyModel(pr.clusters, pr.N)
    dp = blib.DeviceProblem(api, pr.N, pr.Nbase, pr.tilesz, barr, sky, pr.coh, pr.x)
    rng = np.random.default_rng(7)
    p0 = pr.pp0 + 0.02 * rng.normal(0, 1, pr.pp0.shape)
    nu = 4.0
    R = pr.Nbase1
    b = (R + 4) // 5
    rep = {"shape": dict(N=pr.N, M=pr.M, Mt=pr.Mt, tilesz=pr.tilesz, rows=R, window_rows=b)}
    rep["card"], rep["power_limit_and_max_sm_clock"] = card()

    # one pass each, CUDA events around every launch (db_prof_begin / end), averaged over reps
    def passes(fn, kind):
        fn()  # warm-up
        api.lib.dirac_b200_profile_enable(1)
        for _ in range(args.reps):
            fn()
        n, ms, by = kernel_ms(api, kind)
        api.lib.dirac_b200_profile_enable(0)
        return dict(ms=ms / n, GBps=by / (ms * 1e-3) / 1e9 if ms > 0 else None, bytes=by / n)

    rep["cost_full"] = passes(lambda: dp.cost(p0, robust=True, nu=nu), 0)
    rep["cost_window"] = passes(lambda: dp.cost_window(p0, b, b, nu), 0)
    rep["grad_full"] = passes(lambda: dp.grad(p0, robust=True, nu=nu), 1)
    rep["grad_window"] = passes(lambda: dp.grad_window(p0, b, b, nu), 1)
    rep["cost_window_over_full"] = rep["cost_window"]["ms"] / rep["cost_full"]["ms"]
    rep["grad_window_over_full"] = rep["grad_window"]["ms"] / rep["grad_full"]["ms"]

    # the LBFGS stage alone (max_emiter = 0), full batch (+7) and stochastic (-7), alternated
    kw = dict(max_emiter=0, max_iter=0, max_lbfgs=args.max_lbfgs, solver_mode=2)
    stage = {7: [], -7: []}
    for rnd in range(3):
        for m in (7, -7):
            p = p0.copy()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            dp.sagefit(p, None, lbfgs_m=m, **kw)
            torch.cuda.synchronize()
            if rnd:  # the first round warms up both
                stage[m].append(time.perf_counter() - t0)
    rep["stage_s"] = {"lbfgs_m=+7": min(stage[7]), "lbfgs_m=-7": min(stage[-7]),
                      "all": {str(k): v for k, v in stage.items()}}
    # host / device split of the -7 stage: device time of the cost and gradient passes it launched
    p = p0.copy()
    api.lib.dirac_b200_profile_enable(1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    dp.sagefit(p, None, lbfgs_m=-7, **kw)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    n0, ms0, _ = kernel_ms(api, 0)
    n1, ms1, _ = kernel_ms(api, 1)
    api.lib.dirac_b200_profile_enable(0)
    dev = (ms0 + ms1) * 1e-3
    rep["stage_m7_split"] = dict(wall_s=wall, cost_passes=n0, grad_passes=n1, device_pass_s=dev,
                                 rest_s=wall - dev, note="rest = host vector algebra, copies, syncs "
                                 "(the wall time includes the two full-interval residual passes of sagefit)")
    dp.close()
    line = json.dumps(rep)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
