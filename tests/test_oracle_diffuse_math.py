"""CPU: the arithmetic of the diffuse-cluster kernels (sagecal_b200/csrc/diffuse_math.cuh, compiled as
host code from oracle/diffuse_math_check.cu) against the compiled reference: shapelet_product_tensor
(shapelet.c:640), shapelet_product_jones (:864), shapelet_contrib_vector (:199) and the whole of
recalculate_diffuse_coherencies (diffuse_predict.c:295) on its CPU path.  Also the declarations of
include/dirac_b200_diffuse.h and the link order of its entry points.  Runs without a GPU."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from sagecal_b200.dirac_api import SkyModel, cptr, dptr, make_barr

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
d, i, dp = C.c_double, C.c_int, C.POINTER(C.c_double)
STYPE_SHAPELET = 4
FREQ0, FDELTA = 150e6, 2e5


@pytest.fixture(scope="session")
def chk(tmp_path_factory):
    """the harness, compiled by nvcc as host code into a temporary directory"""
    out = str(tmp_path_factory.mktemp("diffuse") / "libdiffuse_math_check.so")
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-Xcompiler", "-fPIC", "-shared", "-cudart",
                           "static", "-o", out, os.path.join(ROOT, "oracle", "diffuse_math_check.cu")])
    L = C.CDLL(out)
    L.check_tensor.restype = i
    L.check_tensor.argtypes = [i, i, i, d, d, d, dp]
    L.check_product.argtypes = [i, i, i, dp, dp, dp, i, dp]
    L.check_contrib.argtypes = [dp, i, d, d, d, dp]
    L.check_pipeline.restype = i
    L.check_pipeline.argtypes = ([i, C.c_longlong, C.POINTER(i), C.POINTER(i), dp, dp, dp, d, d, i,
                                  C.POINTER(i), dp, dp, dp, dp, i, d, dp, dp])
    return L


def _ref_fn(ref, name, restype, argtypes):
    fn = getattr(ref.lib, name)
    fn.restype = restype
    fn.argtypes = argtypes
    return fn


def ref_tensor(ref, L, M, N, a, b, c):
    B = np.zeros(L * M * N)
    _ref_fn(ref, "shapelet_product_tensor", i, [i, i, i, d, d, d, dp])(L, M, N, a, b, c, dptr(B))
    return B


# ---- the diffuse problem the CPU and GPU tests share ------------------------------------------------

def diffuse_problem(N, T, M=3, cid=1, n0s=(4,), sh=2, seed=0, flag_frac=0.0, zero_row=False,
                    nsrc_other=1):
    """N stations, T timeslots of the canonical baselines (p < q); M clusters, cluster cid diffuse with
    one shapelet source per entry of n0s (Stokes I, Q, U, V all non-zero), the others point sources;
    x0: random coherencies [row][M][4]; Z: random 2N x 2G spatial model"""
    rng = np.random.default_rng(seed)
    p, q = np.triu_indices(N, 1)
    Nb = len(p)
    R = Nb * T
    sta1, sta2 = np.tile(p, T), np.tile(q, T)
    flag = (rng.uniform(size=R) < flag_frac).astype(np.uint8)
    # u v w in seconds: |u f| up to a few hundred wavelengths at 150 MHz
    u = rng.normal(0, 6e-7, R)
    v = rng.normal(0, 6e-7, R)
    w = rng.normal(0, 1e-7, R)
    if zero_row:
        u[0] = v[0] = w[0] = 0.0
    clusters = []
    for k in range(M):
        if k == cid:
            K = len(n0s)
            sh_ = {}
            for s, n0 in enumerate(n0s):
                sh_[s] = dict(n0=int(n0), beta=float(rng.uniform(0.01, 0.03)),
                              modes=rng.normal(0, 1, n0 * n0) / n0, eX=1.0, eY=1.0, eP=0.0)
            cl = dict(ll=rng.uniform(-0.02, 0.02, K), mm=rng.uniform(-0.02, 0.02, K),
                      sI=rng.uniform(0.5, 2.0, K), sQ=rng.uniform(-0.3, 0.3, K),
                      sU=rng.uniform(-0.3, 0.3, K), sV=rng.uniform(-0.2, 0.2, K),
                      stype=np.full(K, STYPE_SHAPELET), shapelet=sh_)
        else:
            K = nsrc_other
            cl = dict(ll=rng.uniform(-0.02, 0.02, K), mm=rng.uniform(-0.02, 0.02, K),
                      sI=rng.uniform(0.5, 2.0, K), sQ=np.zeros(K), sU=np.zeros(K), sV=np.zeros(K))
        cl["nn"] = np.sqrt(1.0 - cl["ll"] ** 2 - cl["mm"] ** 2) - 1.0
        clusters.append(cl)
    G = sh * sh
    Z = (rng.normal(0, 1, (2 * N, 2 * G)) + 1j * rng.normal(0, 1, (2 * N, 2 * G))) / G
    x0 = rng.normal(0, 1, R * M * 4) + 1j * rng.normal(0, 1, R * M * 4)
    return dict(N=N, T=T, Nb=Nb, R=R, M=M, cid=cid, sh=sh, sh_beta=float(rng.uniform(0.003, 0.006)),
                sta1=sta1, sta2=sta2, flag=flag, u=u, v=v, w=w, clusters=clusters, Z=Z, x0=x0)


def run_diffuse(lib, pb, sky=None, x=None, cid=None):
    """lib.recalculate_diffuse_coherencies on a copy of x0; returns x [row][M][4]"""
    sky = sky or SkyModel(pb["clusters"], pb["N"])
    x = (pb["x0"] if x is None else x).copy()
    barr = make_barr(pb["sta1"], pb["sta2"], pb["flag"])
    rv = lib.recalculate_diffuse_coherencies(pb["u"], pb["v"], pb["w"], x, pb["N"], barr, sky, FREQ0,
                                             FDELTA, pb["cid"] if cid is None else cid, pb["sh"],
                                             pb["sh_beta"], pb["Z"])
    assert rv == 0
    return x.reshape(pb["R"], pb["M"], 4)


def harness_pipeline(chk, pb):
    cl = pb["clusters"][pb["cid"]]
    ns = len(cl["ll"])
    n0s = np.array([cl["shapelet"][s]["n0"] for s in range(ns)], dtype=np.int32)
    betas = np.array([cl["shapelet"][s]["beta"] for s in range(ns)])
    lmn = np.ascontiguousarray(np.stack([cl["ll"], cl["mm"], cl["nn"]], axis=1).reshape(-1))
    iquv = np.ascontiguousarray(np.stack([cl["sI"], cl["sQ"], cl["sU"], cl["sV"]], axis=1).reshape(-1))
    modes = np.ascontiguousarray(np.concatenate([cl["shapelet"][s]["modes"] for s in range(ns)]))
    s1 = np.ascontiguousarray(pb["sta1"], dtype=np.int32)
    s2 = np.ascontiguousarray(pb["sta2"], dtype=np.int32)
    Zf = np.asfortranarray(pb["Z"]).reshape(-1, order="F")
    out = np.zeros(pb["R"] * 4, dtype=np.complex128)
    ip = lambda a: a.ctypes.data_as(C.POINTER(i))
    rv = chk.check_pipeline(pb["N"], pb["R"], ip(s1), ip(s2), dptr(pb["u"]), dptr(pb["v"]), dptr(pb["w"]),
                            FREQ0, FDELTA, ns, ip(n0s), dptr(betas), dptr(lmn), dptr(iquv), dptr(modes),
                            pb["sh"], pb["sh_beta"], cptr(Zf), cptr(out))
    assert rv == 0
    return out.reshape(pb["R"], 4)


# ---- tensor ---------------------------------------------------------------------------------------

TENSOR_CASES = [(1, 1, 1), (3, 3, 1), (5, 1, 5), (4, 4, 3), (8, 3, 8), (12, 12, 4), (20, 3, 20),
                (20, 20, 3), (32, 4, 32), (32, 32, 4), (32, 1, 32), (32, 32, 32), (17, 29, 32)]


@pytest.mark.parametrize("LMN", TENSOR_CASES, ids=["x".join(map(str, c)) for c in TENSOR_CASES])
def test_product_tensor(ref, chk, LMN):
    """to 1e-14 of the largest entry, including the normalisation of shapelet.c:672 and the rescaling
    by the 2-norm"""
    L, M, N = LMN
    rng = np.random.default_rng(L * 1000 + M * 37 + N)
    a, b, c = rng.uniform(0.002, 0.008, 3)
    want = ref_tensor(ref, L, M, N, a, b, c)
    got = np.zeros(L * M * N)
    assert chk.check_tensor(L, M, N, a, b, c, dptr(got)) == 0
    assert np.all(np.isfinite(want))
    assert np.max(np.abs(got - want)) <= 1e-14 * np.max(np.abs(want)), np.max(np.abs(got - want))


# ---- products -------------------------------------------------------------------------------------

def _cplx(rng, n):
    return rng.normal(0, 1, n) + 1j * rng.normal(0, 1, n)


PRODUCT_CASES = [(1, 1, 1), (4, 4, 2), (6, 2, 6), (8, 8, 3), (12, 4, 12), (10, 10, 1), (7, 3, 9)]


@pytest.mark.parametrize("herm", [1, 0])
@pytest.mark.parametrize("LMN", PRODUCT_CASES, ids=["x".join(map(str, c)) for c in PRODUCT_CASES])
def test_product_jones(ref, chk, LMN, herm):
    """the separable product against the reference's Kronecker sum, within 1e-12 of the same sum taken
    over absolute values"""
    L, M, N = LMN
    rng = np.random.default_rng(7 * L + 3 * M + N + herm)
    Cf = ref_tensor(ref, L, M, N, *rng.uniform(0.002, 0.008, 3))
    f = _cplx(rng, 4 * M * M)
    g = _cplx(rng, 4 * N * N)
    want = np.zeros(4 * L * L, dtype=np.complex128)
    _ref_fn(ref, "shapelet_product_jones", i, [i, i, i, d, d, d, dp, dp, dp, dp, i])(
        L, M, N, 1.0, 1.0, 1.0, cptr(want), cptr(f), cptr(g), dptr(Cf), herm)
    got = np.zeros_like(want)
    chk.check_product(L, M, N, dptr(Cf), cptr(f), cptr(g), herm, cptr(got))
    mag = np.zeros_like(want)
    chk.check_product(L, M, N, dptr(np.abs(Cf)), cptr(np.abs(f).astype(complex)),
                      cptr(np.abs(g).astype(complex)), 0, cptr(mag))
    assert np.all(np.abs(got - want) <= 1e-12 * mag.real + 1e-300), np.max(np.abs(got - want) / mag.real)
    assert np.max(np.abs(want)) > 0


# ---- one row --------------------------------------------------------------------------------------

@pytest.mark.parametrize("n0", [1, 2, 5, 12, 20, 32])
def test_row_contrib(ref, chk, n0):
    rng = np.random.default_rng(n0)
    modes = _cplx(rng, 4 * n0 * n0)
    beta = 0.02
    fn = _ref_fn(ref, "shapelet_contrib_vector", i, [dp, i, d, d, d, d, dp])
    for k in range(6):
        uf, vf = (0.0, 0.0) if k == 0 else rng.normal(0, 80.0, 2)
        want = np.zeros(4, dtype=np.complex128)
        fn(cptr(modes), n0, beta, uf, vf, 0.0, cptr(want))
        got = np.zeros(4, dtype=np.complex128)
        chk.check_contrib(cptr(modes), n0, beta, uf, vf, cptr(got))
        assert np.max(np.abs(got - want)) <= 1e-12 * max(np.max(np.abs(want)), 1e-300), (k, got, want)


# ---- the whole host pipeline ------------------------------------------------------------------------

PIPE_CASES = [dict(N=2, T=3, n0s=(1,), sh=1), dict(N=5, T=2, n0s=(3, 2), sh=2),
              dict(N=7, T=2, n0s=(6,), sh=3, zero_row=True), dict(N=12, T=1, n0s=(12, 4, 8), sh=4),
              dict(N=9, T=2, n0s=(9, 1), sh=1), dict(N=4, T=4, n0s=(5, 5, 3), sh=3, zero_row=True)]
# (every source order is at least sh: the reference allocates n0^3 doubles for its n0 x sh x n0 pair
# tensor, diffuse_predict.c:483, and writes past them when sh > n0)


@pytest.mark.parametrize("case", PIPE_CASES, ids=["N%d-n0%s-sh%d" % (c["N"], "-".join(map(str, c["n0s"])),
                                                                     c["sh"]) for c in PIPE_CASES])
def test_pipeline_against_reference(ref, chk, case):
    """this header's arithmetic in the reference's order against recalculate_diffuse_coherencies with
    use_cuda = 0, to 1e-11 of the cluster's largest value; the other clusters untouched"""
    pb = diffuse_problem(M=3, cid=1, seed=len(case["n0s"]) * 11 + case["N"], **case)
    want = run_diffuse(ref, pb)
    got = harness_pipeline(chk, pb)
    scale = np.max(np.abs(want[:, 1]))
    assert scale > 0
    assert np.max(np.abs(got - want[:, 1])) <= 1e-11 * scale, np.max(np.abs(got - want[:, 1])) / scale
    x0 = pb["x0"].reshape(pb["R"], 3, 4)
    assert np.array_equal(want[:, [0, 2]], x0[:, [0, 2]])


# ---- header and link order --------------------------------------------------------------------------

def test_diffuse_header_matches_the_reference_and_the_library():
    """include/dirac_b200_diffuse.h declares recalculate_diffuse_coherencies with the reference's own
    parameter type list (Dirac_radio.h:228, stored by tests/golden/make_golden_diffuse_signatures.py)
    and the resident form; the library exports both; dirac_b200.h includes the header"""
    from sagecal_b200 import lib as blib
    from test_cpu_abi import _c_declarations
    ours = _c_declarations(os.path.join(ROOT, "include", "dirac_b200_diffuse.h"))
    with open(os.path.join(ROOT, "tests", "golden", "ref_signatures_diffuse.json")) as f:
        refsig = json.load(f)
    assert sorted(ours) == sorted(blib.DIFFUSE_EXPORTED)
    assert sorted(refsig) == ["recalculate_diffuse_coherencies"]
    assert ours["recalculate_diffuse_coherencies"][0] in refsig["recalculate_diffuse_coherencies"]
    main = _c_declarations(os.path.join(ROOT, "include", "dirac_b200.h"))
    assert not set(main) & set(ours)
    assert '#include "dirac_b200_diffuse.h"' in open(os.path.join(ROOT, "include", "dirac_b200.h")).read()
    if os.path.exists(blib.LIB_PATH):
        L = C.CDLL(blib.LIB_PATH)
        for name in ours:
            assert hasattr(L, name), name


def test_link_order_puts_the_diffuse_call_on_this_library(tmp_path):
    """`-ldirac_b200` in front of the reference's library takes recalculate_diffuse_coherencies;
    update_spatialreg_fista (spatial regularisation on the master) stays with the reference.  The
    reference's library is stood in for by one that defines both names."""
    names = ["recalculate_diffuse_coherencies", "update_spatialreg_fista"]
    refdir = str(tmp_path)
    stub = os.path.join(refdir, "dirac_ref_standin.c")
    with open(stub, "w") as f:
        f.write("".join("void %s(void) {}\n" % s for s in names))
    subprocess.check_call(["gcc", "-shared", "-fPIC", "-o", os.path.join(refdir, "libdirac_ref.so"), stub])
    src = os.path.join(refdir, "link_order_diffuse.c")
    with open(src, "w") as f:
        f.write('#define _GNU_SOURCE\n#include <dlfcn.h>\n#include <stdio.h>\n#include <string.h>\n'
                '#include "dirac_b200.h"\nextern void update_spatialreg_fista(void);\n'
                'static void where(const char *n, void *fn) { Dl_info i; dladdr(fn, &i);\n'
                '  const char *b = strrchr(i.dli_fname, 47); printf("%s %s\\n", n, b ? b + 1 : i.dli_fname); }\n'
                'int main(void) { where("recalculate_diffuse_coherencies", (void *)recalculate_diffuse_coherencies);\n'
                '  where("update_spatialreg_fista", (void *)update_spatialreg_fista); return 0; }\n')
    exe = os.path.join(refdir, "link_order_diffuse")
    libdir = os.path.join(ROOT, "sagecal_b200")
    subprocess.check_call(["gcc", "-O1", "-Wall", "-o", exe, src, "-I", os.path.join(ROOT, "include"),
                           "-L", libdir, "-ldirac_b200", "-L", refdir, "-ldirac_ref", "-ldl", "-lm",
                           "-Wl,-rpath," + libdir, "-Wl,-rpath," + refdir, "-Wl,--allow-shlib-undefined"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, (out.stdout, out.stderr)
    got = dict(line.split() for line in out.stdout.strip().splitlines())
    assert got == {"recalculate_diffuse_coherencies": "libdirac_b200.so",
                   "update_spatialreg_fista": "libdirac_ref.so"}, got


# ---- refused arguments -----------------------------------------------------------------------------

_EXIT_SCRIPT = """
import sys
sys.path[:0] = [%r, %r]
import numpy as np
from sagecal_b200 import lib
from test_oracle_diffuse_math import diffuse_problem, run_diffuse
pb = diffuse_problem(N=4, T=1, M=3, cid=1, n0s=(3,), sh=2)
if sys.argv[1] == "point":
    pb["clusters"][1]["stype"] = np.zeros(1)
run_diffuse(lib.load(), pb, cid=7 if sys.argv[1] == "cid" else None)
print("returned")
"""


@pytest.mark.parametrize("what,msg", [("cid", "invalid cluster id"),
                                      ("point", "invalid source type, must be shapelet")])
def test_refused_arguments_exit_1(what, msg):
    """a cluster id outside [0, M) and a source that is not a shapelet print the reference's message
    and exit(1) before any device work (diffuse_predict.c:388-397)"""
    from sagecal_b200 import lib as blib
    if not os.path.exists(blib.LIB_PATH):
        pytest.skip("libdirac_b200.so not built")
    out = subprocess.run([sys.executable, "-c", _EXIT_SCRIPT % (ROOT, HERE), what], capture_output=True,
                         text=True, timeout=300)
    assert out.returncode == 1, (out.returncode, out.stdout, out.stderr)
    assert msg in out.stderr and "returned" not in out.stdout
