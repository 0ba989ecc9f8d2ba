"""The substitution pair of the large LM systems (8N = 4096 at 512 stations) as the LM issues it: every
solve recomputes its diagonal-block products from a fresh factor, and the factor is not resident in L2
(the timed solves alternate over --nfac factors of 67 MB each).  Times `reps` back-to-back solves by
CUDA events (dirac_b200_bigtri_sequence), and cuSOLVER dpotrf at the same n as a yardstick, and checks
the answers of --nfac solves against scipy.  The card's name, power limit and maximum SM clock are read
in the same run.  --lib times another build of the library (e.g. the parent commit's) for a
before / after pair in one session.  Prints one JSON line.

    python profiles/bigtri_solve.py [--n 4096] [--nfac 2] [--reps 400] [--lib path/to/libdirac_b200.so]"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sagecal_b200 import lib as blib  # noqa: E402
from minibatch_stage import card  # noqa: E402


def spd(n, seed):
    g = np.random.default_rng(seed).standard_normal((n, n))
    return g @ g.T / n + 0.5 * np.eye(n)


def main():
    import scipy.linalg as sla
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--nfac", type=int, default=2)
    ap.add_argument("--reps", type=int, default=400)
    ap.add_argument("--lib", default=blib.LIB_PATH)
    args = ap.parse_args()
    n, nfac = args.n, args.nfac
    L = blib.DiracB200(os.path.abspath(args.lib)).lib
    f = L.dirac_b200_bigtri_sequence
    f.restype = C.c_int
    f.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    mats = [spd(n, 10 + i) for i in range(nfac)]
    A = np.stack([np.asfortranarray(m) for m in mats]).copy()
    b = np.random.default_rng(3).standard_normal((nfac, n))
    x = np.zeros((nfac, n))
    us = np.zeros(2)
    rc = f(n, nfac, A.ctypes.data, nfac, b.ctypes.data, x.ctypes.data, args.reps, us.ctypes.data)
    if rc != 0:
        raise SystemExit("dirac_b200_bigtri_sequence returned %d" % rc)
    rel = max(float(np.max(np.abs(x[i] - want)) / np.max(np.abs(want)))
              for i, want in enumerate(sla.cho_solve(sla.cho_factor(m, lower=True), b[i]) for i, m in enumerate(mats)))
    rep = {"lib": os.path.relpath(os.path.abspath(args.lib), ROOT), "n": n, "nfac": nfac, "reps": args.reps}
    rep["card"], rep["power_limit_and_max_sm_clock"] = card()
    rep["us_per_substitution_pair"] = round(float(us[0]), 1)
    rep["us_per_dpotrf"] = round(float(us[1]), 1)
    rep["max_rel_err_vs_scipy"] = rel
    print(json.dumps(rep))


if __name__ == "__main__":
    main()
