"""The LBFGS line model of one seeded problem through the library's test hook
(dirac_b200_line_model).  test_gpu_linemodel.py imports `make_case` / `run_case`, and runs this file
in a subprocess to see the line model under DIRAC_B200_* switches, which the library reads once per
process: `python linemodel_check.py '<case json>' out.npz`."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from sagecal_b200 import lib as blib  # noqa: E402
from util import small_problem  # noqa: E402

ALPHAS = np.array([0.0, 1e-6, 0.37, 1.0, -0.5, 3.0])
NU = 3.5
ALPHA_RES = 0.63


def make_case(case):
    """(bound problem, xk, pk) of a case dict: N, M, tilesz, seed, optional nchunk / kmean"""
    kw = {k: v for k, v in case.items() if k in ("nchunk", "kmean")}
    b = small_problem(N=case["N"], M=case["M"], tilesz=case["tilesz"], seed=case["seed"], **kw)
    rng = np.random.default_rng(case["seed"] + 1000)
    xk = b.pr.pp0 + 0.1 * rng.normal(0, 1, b.pr.pp0.shape)
    pk = 0.05 * rng.normal(0, 1, b.pr.pp0.shape)
    return b, xk, pk


def run_case(api, b, xk, pk):
    pr = b.pr
    with blib.DeviceProblem(api, pr.N, pr.Nbase, pr.tilesz, b.barr, b.sky, pr.coh, pr.x) as dp:
        return dp.line_model(xk, pk, ALPHAS, NU, ALPHA_RES)


def main():
    case = json.loads(sys.argv[1])
    b, xk, pk = make_case(case)
    got = run_case(blib.load(), b, xk, pk)
    got["shape"] = np.array(got["shape"])
    np.savez(sys.argv[2], **got)


if __name__ == "__main__":
    main()
