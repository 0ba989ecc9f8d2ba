import sys, os; sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import ctypes as C, numpy as np
from sagecal_b200 import synth, lib as blib
from sagecal_b200.dirac_api import SkyModel, make_barr
api = blib.load(); L = api.lib
L.dirac_b200_bench_cluster_pass.restype = C.c_double
L.dirac_b200_bench_cluster_pass.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
pr = synth.make_problem(N=62, M=64, tilesz=120, radius=40e3, seed=5, kmean=2.0)
barr = make_barr(pr.sta1, pr.sta2, pr.flag); sky = SkyModel(pr.clusters, pr.N)
dp = blib.DeviceProblem(api, pr.N, pr.Nbase, pr.tilesz, barr, sky, pr.coh, pr.x)
dp.cost(pr.pp0)
R = pr.Nbase1
for (mode, grad, wr, name) in [(1,1,0,'TRIAL+grad'), (0,1,1,'INIT'), (3,0,1,'SUB')]:
    us = L.dirac_b200_bench_cluster_pass(dp.h, 0, mode, grad, wr, 300)
    by = R*(129+(64 if wr else 0))
    print(f'{name:16s} {us:7.2f} us  {by/us/1e3:7.1f} GB/s')
