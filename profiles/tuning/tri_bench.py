import sys, os; sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import ctypes as C, numpy as np
from sagecal_b200 import lib as blib
L = blib.load().lib
L.dirac_b200_tri_solve.restype = C.c_int
L.dirac_b200_tri_solve.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
for n in (496, 256):
    rng = np.random.default_rng(0); J = rng.standard_normal((2*n, n)); A = J.T@J + np.eye(n); F = np.asfortranarray(np.linalg.cholesky(A)); b = rng.standard_normal(n); x = np.zeros(n)
    us = C.c_double(0)
    rc = L.dirac_b200_tri_solve(n, F.ctypes.data, b.ctypes.data, x.ctypes.data, 200, C.byref(us))
    print('n', n, 'rc', rc, 'us/solve', us.value, 'err', np.max(np.abs(x-np.linalg.solve(A,b))))
