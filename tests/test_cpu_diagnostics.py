"""CPU tier of the influence-function diagnostics (calculate_diagnostics_gpu, driver option -i 1): the
header against the reference's parameter type list, the link order of a C host, and identities of the
float64 restatement (tests/influence_ref.py) the GPU tests compare against."""
import json
import os
import subprocess

import numpy as np

import influence_ref as ir

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_diagnostics_header_matches_the_reference_and_the_library():
    """include/dirac_b200_diagnostics.h declares calculate_diagnostics_gpu with the reference's own
    parameter type list (Dirac_radio.h:676, tests/golden/make_golden_diagnostics_signatures.py)"""
    from sagecal_b200 import lib as blib
    from test_cpu_abi import _c_declarations
    ours = _c_declarations(os.path.join(ROOT, "include", "dirac_b200_diagnostics.h"))
    with open(os.path.join(ROOT, "tests", "golden", "ref_signatures_diagnostics.json")) as f:
        ref = json.load(f)
    assert sorted(ours) == sorted(ref) == sorted(blib.DIAGNOSTICS_EXPORTED)
    for name, sigs in ours.items():
        assert len(sigs) == 1 and sigs[0] in ref[name], (name, sigs, ref[name])
    main = _c_declarations(os.path.join(ROOT, "include", "dirac_b200.h"))
    assert not set(main) & set(ours)
    assert '#include "dirac_b200_diagnostics.h"' in open(os.path.join(ROOT, "include", "dirac_b200.h")).read()


def test_link_order_puts_the_diagnostics_on_this_library(tmp_path):
    """a C host compiled against the header and linked `-ldirac_b200` before the reference's library
    resolves calculate_diagnostics_gpu to libdirac_b200.so (the reference is stood in for by a
    library that also defines it)"""
    refdir = str(tmp_path)
    stub = os.path.join(refdir, "dirac_ref_standin.c")
    with open(stub, "w") as f:
        f.write("void calculate_diagnostics_gpu(void) {}\n")
    subprocess.check_call(["gcc", "-shared", "-fPIC", "-o", os.path.join(refdir, "libdirac_ref.so"), stub])
    src = os.path.join(refdir, "caller.c")
    with open(src, "w") as f:
        f.write('#define _GNU_SOURCE\n#include <dlfcn.h>\n#include <stdio.h>\n#include <string.h>\n'
                '#include "dirac_b200_diagnostics.h"\n'
                "int main(void) {\n  Dl_info i;\n"
                "  if (!dladdr((void *)calculate_diagnostics_gpu, &i) || !i.dli_fname) return 1;\n"
                "  const char *b = strrchr(i.dli_fname, '/');\n"
                '  printf("%s\\n", b ? b + 1 : i.dli_fname);\n  return 0;\n}\n')
    exe = os.path.join(refdir, "caller")
    libdir = os.path.join(ROOT, "sagecal_b200")
    subprocess.check_call(["gcc", "-O1", "-Wall", "-std=c99", "-o", exe, src, "-I",
                           os.path.join(ROOT, "include"), "-L", libdir, "-ldirac_b200", "-L", refdir,
                           "-ldirac_ref", "-ldl", "-lm", "-Wl,-rpath," + libdir, "-Wl,-rpath," + refdir,
                           "-Wl,--allow-shlib-undefined"])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, (out.stdout, out.stderr)
    assert out.stdout.strip() == "libdirac_b200.so"


def _case(N=5, T=4, nchunk=2, seed=0):
    rng = np.random.default_rng(seed)
    pairs = [(p, q) for p in range(N) for q in range(p + 1, N)]
    Nbase = len(pairs)
    R = Nbase * T
    sta1 = np.tile([p for p, _ in pairs], T)
    sta2 = np.tile([q for _, q in pairs], T)
    flag = (rng.random(R) < 0.2).astype(np.uint8)
    cz = lambda *s: rng.normal(size=s) + 1j * rng.normal(size=s)
    p = rng.normal(size=8 * N * nchunk)
    return N, Nbase, T, sta1, sta2, flag, p, nchunk, cz(R, 4), cz(R, 4), cz(4 * N, Nbase)


def test_hessian_is_hermitian_before_the_conditioning():
    N, Nbase, T, sta1, sta2, flag, p, nchunk, coh, res, _ = _case()
    H = ir.hessian(N, Nbase, T, sta1, sta2, flag, p, nchunk, coh, res)
    assert np.abs(H).max() > 0
    assert np.abs(H - H.conj().T).max() <= 1e-12 * np.abs(H).max()


def test_integer_abs_conditioning():
    """diagnostics.c:712 applies C's integer abs to a float: 0.7 and -0.7 become 1, 1.3 and 0 -> 1
    and 1.3 stays; imaginary parts and off-diagonal entries are untouched; then + hadd"""
    H = np.diag([0.7, 1.3, -0.7, 0.0, -1.3]).astype(np.complex128) + 0.25j
    got = ir.condition(H)
    assert np.allclose(np.real(np.diag(got)), [1.0, 1.3, 1.0, 1.0, -1.3])
    assert np.allclose(np.imag(got), 0.25)
    assert np.allclose(np.real(np.diag(ir.condition(H, 0.5))), [1.5, 1.8, 1.5, 1.5, -0.8])


def test_eigenvalue_trace_equals_dR_trace():
    N, Nbase, T, sta1, sta2, flag, p, nchunk, coh, res, X = _case()
    dR = ir.d_residuals(N, Nbase, T, sta1, sta2, p, nchunk, coh, X)
    for c in range(4):
        assert abs(np.linalg.eigvals(dR[c]).sum() - np.trace(dR[c])) <= 1e-10 * np.abs(dR[c]).sum()


def test_output_layout_round_trips_odd_nbase():
    for N in (7, 6):   # Nbase 21 (odd) and 15
        Nbase = N * (N - 1) // 2
        rng = np.random.default_rng(N)
        E = [rng.normal(size=Nbase) + 1j * rng.normal(size=Nbase) for _ in range(4)]
        x0 = ir.eig_to_x(E, Nbase, 3)
        assert x0.shape == (3 * 8 * Nbase,)
        assert np.array_equal(x0[:8 * Nbase], x0[8 * Nbase:16 * Nbase])
        back = ir.x_to_eig(x0, Nbase)
        for c in range(4):
            assert np.array_equal(back[c], E[c])


def test_dR_reads_every_row_and_adv_only_unflagged():
    N, Nbase, T, sta1, sta2, flag, p, nchunk, coh, res, X = _case(seed=3)
    all_flagged = np.ones_like(flag)
    assert np.abs(ir.adv(N, Nbase, T, sta1, sta2, all_flagged, p, nchunk, coh)).max() == 0
    assert np.abs(ir.hessian(N, Nbase, T, sta1, sta2, all_flagged, p, nchunk, coh, res)).max() == 0
    assert np.abs(ir.d_residuals(N, Nbase, T, sta1, sta2, p, nchunk, coh, X)).max() > 0
