"""Simulation with solutions (predict_visibilities_multifreq_withsol) at the C3 station count: 62 stations,
64 clusters, 120 timeslots, 8 channels, SIMUL_ONLY with the correction by one cluster.  Reports the
CUDA-event time of the coherency kernel (k_sky_predict<2>, profile kind 11), the whole call including
the uploads and the copy back, the reference's CPU call from oracle/_ref on the same host (all host
threads) and the relative difference of the two answers, with the card's name and power limit read
in the same run.  Prints one JSON line; with --out, writes it there too.

    python profiles/predict_withsol.py [--reps 5] [--out FILE]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sagecal_b200 import synth, lib as blib  # noqa: E402
from sagecal_b200.dirac_api import SkyModel, make_barr  # noqa: E402
from minibatch_stage import card, kernel_ms  # noqa: E402

KIND_WITHSOL = 11   # coh_host.cu: residuals_multifreq_impl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("predict_withsol.py measures on a GPU; none is visible")
    api = blib.load()
    api.lib.dirac_b200_profile_enable.argtypes = [C.c_int]
    pr = synth.make_config("C3")
    sky = SkyModel(pr.clusters, pr.N)
    freqs = 150e6 + (np.arange(8) - 3.5) * 195.3e3
    rng = np.random.default_rng(5)
    pp = pr.pp0 + 0.05 * rng.normal(0, 1, pr.pp0.shape)
    n = 8 * pr.Nbase1 * len(freqs)
    kw = dict(add_to_data=1, ccid=3, rho=1e-9)
    rep = {"shape": dict(N=pr.N, M=pr.M, Mt=pr.Mt, tilesz=pr.tilesz, rows=pr.Nbase1,
                         Nchan=len(freqs), sources=int(sum(len(c["ll"]) for c in pr.clusters)))}
    rep["card"], rep["power_limit_and_max_sm_clock"] = card()

    def call(lib, x, Nt=4):
        barr = make_barr(pr.sta1, pr.sta2, pr.flag)
        rv = lib.predict_visibilities_multifreq_withsol(pr.u, pr.v, pr.w, pp, x, pr.N, pr.Nbase,
                                                        pr.tilesz, barr, sky, freqs,
                                                        195.3e3 * len(freqs), Nt=Nt, **kw)
        assert rv == 0

    xb = np.zeros(n)
    call(api, xb)  # warm-up
    api.lib.dirac_b200_profile_enable(1)
    walls = []
    for _ in range(args.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        call(api, xb)
        walls.append(time.perf_counter() - t0)
    nk, ms, by = kernel_ms(api, KIND_WITHSOL)
    api.lib.dirac_b200_profile_enable(0)
    rep["kernel_ms"] = ms / nk
    rep["call_ms"] = {"min": 1e3 * min(walls), "all": [1e3 * t for t in walls]}
    rep["kernel_share_of_call"] = rep["kernel_ms"] / rep["call_ms"]["min"]

    import refdirac
    if refdirac.available():
        nt = os.cpu_count() or 1
        xa = np.zeros(n)
        t0 = time.perf_counter()
        call(refdirac.load(), xa, Nt=nt)
        rep["reference_cpu_ms"] = 1e3 * (time.perf_counter() - t0)
        rep["reference_threads"] = nt
        rep["reference_over_call"] = rep["reference_cpu_ms"] / rep["call_ms"]["min"]
        rep["relerr_vs_reference"] = float(np.max(np.abs(xb - xa)) / np.max(np.abs(xa)))
    else:
        rep["reference_cpu_ms"] = "not measured (oracle/_ref not built)"
    line = json.dumps(rep)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
