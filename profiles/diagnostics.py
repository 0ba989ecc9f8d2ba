"""Influence-function diagnostics (calculate_diagnostics_gpu, driver option -i 1) at the C3 shape: 62
stations (Nbase 1891), 64 clusters, 120 timeslots, one channel.  Reports the CUDA-event times of the
stages (profile kinds 18-23 of problem.cu: the model stage, Hessians and right-hand sides, the LU
solves, k_infl_dr, the four 1891 x 1891 complex geevs, the whole call) and the host wall time of the
call, with the card's name and power limit read in the same run.  Prints one JSON line; with --out,
writes it there too.

    python profiles/diagnostics.py [--reps 3] [--out FILE]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sagecal_b200 import synth, lib as blib  # noqa: E402
from sagecal_b200.dirac_api import SkyModel, make_barr  # noqa: E402
from minibatch_stage import card  # noqa: E402

STAGES = {"model": 18, "hessian_rhs": 19, "solves": 20, "dR": 21, "geev4": 22, "call": 23}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("diagnostics.py measures on a GPU; none is visible")
    api = blib.load()
    pr = synth.make_config("C3")
    sky = SkyModel(pr.clusters, pr.N)
    freqs = np.array([150e6])
    rng = np.random.default_rng(5)
    pp = pr.pp0 + 0.05 * rng.normal(0, 1, pr.pp0.shape)
    x0 = rng.normal(0, 1, 8 * pr.Nbase1)
    rep = {"shape": dict(N=pr.N, Nbase=pr.Nbase, M=pr.M, Mt=pr.Mt, tilesz=pr.tilesz, Nchan=1)}
    rep["card"], rep["power_limit_and_max_sm_clock"] = card()

    def call():
        x = x0.copy()
        rv = api.calculate_diagnostics_gpu(pr.u, pr.v, pr.w, pp.copy(), x, pr.N, pr.Nbase, pr.tilesz,
                                           make_barr(pr.sta1, pr.sta2, pr.flag), sky, freqs, 195.3e3)
        assert rv == 0
        return x

    xw = call()  # warm-up: modules, cuSOLVER
    api.lib.dirac_b200_profile_enable(1)
    walls = []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        x = call()
        walls.append(time.perf_counter() - t0)
    ms = C.c_double(0.0)
    for name, kind in STAGES.items():
        n = api.lib.dirac_b200_profile_read(kind, C.byref(ms), None)
        rep[name + "_ms"] = round(ms.value / max(n, 1), 3)
    api.lib.dirac_b200_profile_enable(0)
    rep["wall_ms_mean"] = round(1e3 * float(np.mean(walls)), 2)
    rep["reps"] = args.reps
    rep["bit_identical_runs"] = bool(np.array_equal(x, xw))
    line = json.dumps(rep)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
