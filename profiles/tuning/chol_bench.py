import sys, os; sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import ctypes as C, numpy as np
from sagecal_b200 import lib as blib
L = blib.load().lib
L.dirac_b200_bench_spd_solve.restype = C.c_double
L.dirac_b200_bench_spd_solve.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_double, C.c_int]
for n in (496, 256, 128):
    rng = np.random.default_rng(0); J = rng.standard_normal((2*n, n)); A = np.asfortranarray(J.T@J); b = rng.standard_normal(n)
    print('n', n, 'us/solve', L.dirac_b200_bench_spd_solve(n, A.ctypes.data, b.ctypes.data, 1.0, 200))
