import sys, os; sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from sagecal_b200 import synth, lib as blib
from sagecal_b200.dirac_api import SkyModel, make_barr
api = blib.load()
shape = dict(N=62, M=64, tilesz=120, radius=40e3, seed=20260923, kmean=2.0)
pr = synth.make_problem(**shape)
barr = make_barr(pr.sta1, pr.sta2, pr.flag); sky = SkyModel(pr.clusters, pr.N)
dp = blib.DeviceProblem(api, pr.N, pr.Nbase, pr.tilesz, barr, sky, pr.coh, pr.x)
pp = pr.pp0.copy()
for it in range(2):
    c = dp.cost(pp)
    g = dp.grad(pp)
r = dp.sagefit(pp, None, max_emiter=1, max_iter=2, max_lbfgs=2, lbfgs_m=7, solver_mode=1)
print(c, r)
