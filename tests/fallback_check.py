"""Run one small sagefit solve and dump the solved Jones + residual norms (stdout, JSON).  Executed in
a subprocess by test_gpu_solvers.py with and without DIRAC_B200_CUSOLVER: the library reads it once
per process."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from sagecal_b200 import lib as blib  # noqa: E402
from util import small_problem  # noqa: E402


def main():
    api = blib.load()
    b = small_problem(N=20, M=3, tilesz=12, seed=77, kmean=1.5)
    pr = b.pr
    x = pr.x.copy()
    pp = pr.pp0.copy()
    r = api.sagefit_visibilities(pr.u, pr.v, pr.w, x, pr.N, pr.Nbase, pr.tilesz, b.fresh_barr(), b.sky,
                                 pr.coh, pp, max_emiter=3, max_iter=3, max_lbfgs=6, lbfgs_m=5,
                                 solver_mode=1, randomize=0)
    print(json.dumps({"r": [float(v) for v in r], "pp": pp.tolist(),
                      "xn": float(np.linalg.norm(x))}))


if __name__ == "__main__":
    main()
