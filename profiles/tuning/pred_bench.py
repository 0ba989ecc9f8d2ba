import sys, os; sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import ctypes as C, numpy as np
from sagecal_b200 import synth, lib as blib
from sagecal_b200.dirac_api import SkyModel, make_barr
api = blib.load()
L = api.lib
L.dirac_b200_bench_predict.restype = C.c_double
L.dirac_b200_bench_predict.argtypes = [C.c_void_p, C.c_int, C.c_int]
pr = synth.make_problem(N=62, M=64, tilesz=120, radius=40e3, seed=5, kmean=2.0)
barr = make_barr(pr.sta1, pr.sta2, pr.flag); sky = SkyModel(pr.clusters, pr.N)
dp = blib.DeviceProblem(api, pr.N, pr.Nbase, pr.tilesz, barr, sky, pr.coh, pr.x)
dp.cost(pr.pp0)
by = pr.Nbase1*(64*pr.M+65)
us = L.dirac_b200_bench_predict(dp.h, 0, 50)
print('cfg', os.environ.get('DIRAC_B200_SA_CFG','0'), 'tma' if not os.environ.get('DIRAC_B200_NO_TMA') else 'regs', f'{us:8.1f} us {by/us/1e3:8.1f} GB/s')
