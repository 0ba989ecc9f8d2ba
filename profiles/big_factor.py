"""Factorisation of the large LM systems (8N = 4096 at 512 stations): device time per factor and FP64
rate (n^3 / 3 flops per factor) of cuSOLVER dpotrf one system at a time, dpotrf on four streams side by
side, and the blocked batch (bigchol.cu), by CUDA events on
freshly written SPD matrices (dirac_b200_bench_big_factor).  The card's name, power limit and maximum
SM clock are read in the same run.  Prints one JSON line.

    python profiles/big_factor.py [--n 4096] [--batch 32] [--reps 3]"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sagecal_b200 import lib as blib  # noqa: E402
from minibatch_stage import card  # noqa: E402

VARIANTS = ["dpotrf", "dpotrf_4_streams", "blocked_trsm", "blocked_inv", "blocked_inv_lookahead"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    L = blib.load().lib
    L.dirac_b200_bench_big_factor.restype = C.c_int
    L.dirac_b200_bench_big_factor.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_double)]
    rep = {"n": args.n, "batch": args.batch, "reps": args.reps}
    rep["card"], rep["power_limit_and_max_sm_clock"] = card()
    gflop = args.n ** 3 / 3.0 * 1e-9
    for batch in sorted({1, args.batch}):
        for v, name in enumerate(VARIANTS):
            us = (C.c_double * 4)()
            bad = L.dirac_b200_bench_big_factor(args.n, batch, args.reps, v, us)
            per = us[0] / batch
            r = {"us_per_factor": round(per, 1), "tflops": round(gflop / per * 1e3, 2), "bad_status": bad}
            if v in (2, 3):
                r["us_panels_trailing_per_factor"] = [round(us[i] / batch, 1) for i in (1, 2)]
            rep["%s_x%d" % (name, batch)] = r
    print(json.dumps(rep))


if __name__ == "__main__":
    main()
