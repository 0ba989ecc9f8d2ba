"""The projectback manifold average of federated stochastic calibration (the stochastic master of
sagecal-mpi, calculate_manifold_average_projectback) at the C4 shape: N Npoly = 512 x 3 stations, 256
chunks, 8 solutions, 10 Procrustes rounds (the first ADMM iteration) and 2 (the later ones).  Times
(a) k_manifold_projectback through dirac_b200_manifold_projectback_dev on a resident tensor (CUDA
events over --reps launches after a warm-up), (b) the library's calculate_manifold_average_projectback
with its host copies (wall time), and (c) the compiled reference's threaded projectback (Nt = the CPU
count, wall time) when oracle/_ref is built; reports the bound of one pass over the data at the H100
SXM data-sheet bandwidth and the largest difference from the reference with Nt = 1.  The card's name,
power limit and maximum SM clock are read in the same run.  Prints one JSON line; with --out, writes
it there too.

    python profiles/stochastic_federated.py [--reps 20] [--out FILE]"""
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
from minibatch_stage import card  # noqa: E402

N, NPOLY, MT, NF = 512, 3, 256, 8
HBM = 3.35e12  # bytes/s, H100 SXM data sheet


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("stochastic_federated.py measures on a GPU; none is visible")
    api = blib.load()
    rep = {"shape": dict(N=N, Npoly=NPOLY, Mt=MT, Nf=NF)}
    rep["card"], rep["power_limit_and_max_sm_clock"] = card()
    n = N * NPOLY
    rng = np.random.default_rng(3)
    Y0 = rng.normal(size=(NF, MT, 8 * n))
    nbytes = Y0.nbytes
    rep["data_MB"] = nbytes / 1e6
    rep["bound_ms_per_round_2x_traffic"] = 2 * nbytes / HBM * 1e3
    # the kernel reads the data twice and writes it once, whatever the number of rounds
    rep["bound_ms_kernel_3x_traffic"] = 3 * nbytes / HBM * 1e3
    dY0 = torch.from_numpy(Y0).cuda()
    dY = dY0.clone()
    for niter in (10, 2):
        for _ in range(3):
            dY.copy_(dY0)
            assert api.manifold_projectback_dev(dY, niter) == 0
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2 * args.reps)]
        ms = []
        for r in range(args.reps):
            dY.copy_(dY0)
            ev[2 * r].record()
            assert api.manifold_projectback_dev(dY, niter) == 0
            ev[2 * r + 1].record()
        torch.cuda.synchronize()
        ms = [ev[2 * r].elapsed_time(ev[2 * r + 1]) for r in range(args.reps)]
        rep["kernel_ms_niter%d" % niter] = dict(best=min(ms), median=float(np.median(ms)))
        rep["kernel_GBps_niter%d" % niter] = 3 * nbytes / (min(ms) * 1e-3) / 1e9
    Yg = Y0.copy()
    assert api.manifold_projectback(Yg, 10) == 0
    t = []
    for _ in range(3):
        Yg = Y0.copy()
        t0 = time.perf_counter()
        api.manifold_projectback(Yg, 10)
        t.append(time.perf_counter() - t0)
    rep["export_with_copies_ms_niter10"] = 1e3 * min(t)
    import refdirac
    if refdirac.available():
        L = C.CDLL(refdirac.REF_PATH)
        fn = L.calculate_manifold_average_projectback
        fn.argtypes = [C.c_int] * 3 + [C.c_void_p] + [C.c_int] * 3
        nt = os.cpu_count() or 1
        A = Y0.copy()
        t0 = time.perf_counter()
        fn(n, MT, NF, A.ctypes.data, 10, 0, nt)
        rep["reference_ms_niter10_threads%d" % nt] = 1e3 * (time.perf_counter() - t0)
        A = Y0.copy()
        t0 = time.perf_counter()
        fn(n, MT, NF, A.ctypes.data, 10, 0, 1)
        rep["reference_ms_niter10_threads1"] = 1e3 * (time.perf_counter() - t0)
        rep["max_rel_diff_vs_reference"] = float(np.abs(Yg - A).max() / np.abs(A).max())
    else:
        rep["reference"] = "oracle/_ref not built"
    line = json.dumps(rep)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
