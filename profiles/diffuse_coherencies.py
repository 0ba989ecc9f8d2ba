"""Diffuse-cluster coherencies (recalculate_diffuse_coherencies) at the shape of a sagecal-mpi slave with
spatial regularisation: 62 stations, 120 timeslots, 64 clusters, the diffuse cluster with two shapelet
sources of order 20 and 32 and a spatial model of order 3.  Reports the CUDA-event time of the
prediction kernel (k_diffuse_predict, profile kind 12), the whole call (best of --reps after a warm-up,
uploads and the copy back of the cluster's slice included), the reference's CPU call from oracle/_ref
with all host threads at --ref-timeslots timeslots (its pair products do not depend on the timeslots),
this library's answer against it at that shape, and the card's name and power limit read in the same
run.  Prints one JSON line; with --out, writes it there too.

    python profiles/diffuse_coherencies.py [--reps 5] [--ref-timeslots 1] [--out FILE]"""
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
from sagecal_b200 import lib as blib  # noqa: E402
from sagecal_b200.dirac_api import SkyModel, make_barr  # noqa: E402
from minibatch_stage import card, kernel_ms  # noqa: E402

KIND_DIFFUSE = 12   # kernels_diffuse.cu: db_launch_diffuse
N, M, CID, SH = 62, 64, 17, 3
N0S = (20, 32)
FREQ0, FDELTA = 150e6, 195.3e3


def problem(T, seed=3):
    rng = np.random.default_rng(seed)
    p, q = np.triu_indices(N, 1)
    R = len(p) * T
    sta1, sta2 = np.tile(p, T), np.tile(q, T)
    u, v, w = rng.normal(0, 6e-7, R), rng.normal(0, 6e-7, R), rng.normal(0, 1e-7, R)
    clusters = []
    for k in range(M):
        K = len(N0S) if k == CID else 1
        cl = dict(ll=rng.uniform(-0.02, 0.02, K), mm=rng.uniform(-0.02, 0.02, K),
                  sI=rng.uniform(0.5, 2.0, K), sQ=rng.uniform(-0.3, 0.3, K),
                  sU=rng.uniform(-0.3, 0.3, K), sV=rng.uniform(-0.2, 0.2, K))
        if k == CID:
            cl["stype"] = np.full(K, 4)
            cl["shapelet"] = {s: dict(n0=n0, beta=0.02, modes=rng.normal(0, 1, n0 * n0) / n0, eX=1.0,
                                      eY=1.0, eP=0.0) for s, n0 in enumerate(N0S)}
        cl["nn"] = np.sqrt(1.0 - cl["ll"] ** 2 - cl["mm"] ** 2) - 1.0
        clusters.append(cl)
    G = SH * SH
    Z = (rng.normal(0, 1, (2 * N, 2 * G)) + 1j * rng.normal(0, 1, (2 * N, 2 * G))) / G
    return dict(R=R, sta1=sta1, sta2=sta2, u=u, v=v, w=w, sky=SkyModel(clusters, N), Z=Z)


def call(lib, pb, x, Nt=4):
    barr = make_barr(pb["sta1"], pb["sta2"], np.zeros(pb["R"]))
    assert lib.recalculate_diffuse_coherencies(pb["u"], pb["v"], pb["w"], x, N, barr, pb["sky"], FREQ0,
                                               FDELTA, CID, SH, 0.004, pb["Z"], Nt=Nt) == 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--timeslots", type=int, default=120)
    ap.add_argument("--ref-timeslots", type=int, default=1)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("diffuse_coherencies.py measures on a GPU; none is visible")
    api = blib.load()
    api.lib.dirac_b200_profile_enable.argtypes = [C.c_int]
    pb = problem(args.timeslots)
    rep = {"shape": dict(N=N, M=M, timeslots=args.timeslots, rows=pb["R"], n0=list(N0S), sh_n0=SH)}
    rep["card"], rep["power_limit_and_max_sm_clock"] = card()
    x = np.zeros(pb["R"] * M * 4, dtype=np.complex128)
    call(api, pb, x)  # warm-up
    api.lib.dirac_b200_profile_enable(1)
    walls = []
    for _ in range(args.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        call(api, pb, x)
        walls.append(time.perf_counter() - t0)
    nk, ms, _ = kernel_ms(api, KIND_DIFFUSE)
    api.lib.dirac_b200_profile_enable(0)
    rep["kernel_ms"] = ms / nk
    rep["call_ms"] = {"min": 1e3 * min(walls), "all": [1e3 * t for t in walls]}
    del x

    import refdirac
    if refdirac.available():
        nt = os.cpu_count() or 1
        ps = problem(args.ref_timeslots)
        xa = np.zeros(ps["R"] * M * 4, dtype=np.complex128)
        xb = xa.copy()
        t0 = time.perf_counter()
        call(refdirac.load(), ps, xa, Nt=nt)
        rep["reference_cpu_ms"] = 1e3 * (time.perf_counter() - t0)
        rep["reference_threads"] = nt
        rep["reference_timeslots"] = args.ref_timeslots
        t0 = time.perf_counter()
        call(api, ps, xb)
        rep["call_ms_at_reference_shape"] = 1e3 * (time.perf_counter() - t0)
        a = xa.reshape(-1, M, 4)[:, CID]
        b = xb.reshape(-1, M, 4)[:, CID]
        rep["maxerr_over_max_vs_reference"] = float(np.max(np.abs(a - b)) / np.max(np.abs(a)))
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
