"""CPU tier of the simulation with solutions (predict_visibilities_multifreq_withsol and its beam
variants): what the reference's CPU beam variant does with a correction, from its recorded answers,
and the link order that puts the three entry points on this library."""
import os
import subprocess

import numpy as np

from util import perturbed_jones, relerr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SIMUL_ADD = 2


def _jinv(pp, N, k, rho):
    J = pp[8 * N * k:8 * N * (k + 1)].reshape(N, 4, 2)
    return np.linalg.inv((J[..., 0] + 1j * J[..., 1]).reshape(N, 2, 2) + rho * np.eye(2))


def _correct(x, pr, Ji, nchan):
    """x[chan][row][8] -> Jinv_p X Jinv_q^H per row"""
    X = x.reshape(nchan, pr.Nbase1, 4, 2)
    X = (X[..., 0] + 1j * X[..., 1]).reshape(nchan, pr.Nbase1, 2, 2)
    Y = (Ji[pr.sta1] @ X @ np.conj(np.swapaxes(Ji[pr.sta2], -1, -2))).reshape(nchan, pr.Nbase1, 4)
    return np.stack([Y.real, Y.imag], axis=-1).reshape(-1)


def test_reference_withbeam_corrects_once_per_cluster(ref):
    """The reference's CPU predict_visibilities_multifreq_withsol_withbeam corrects inside the
    per-cluster loop (predict_withbeam.c:1175-1210, launched per cluster at :1577-1660): with two
    clusters not ignored and a valid ccid its answer is K(K(x0 + M0) + M2), K the correction and Mk
    the model of cluster k, not the K(x0 + M0 + M2) of its beam-less and GPU variants, which this
    library computes in all three entry points (DESIGN.md section 7)."""
    from test_gpu_beam import beam_problem
    freqs = np.array([146e6, 152e6])
    b, sky, beam = beam_problem(ref, "array", True, seed=37, freqs=freqs)
    pr = b.pr
    pp = perturbed_jones(pr, seed=4, amp=0.1)
    x0 = np.random.default_rng(2).normal(0, 0.1, 8 * pr.Nbase1 * len(freqs))

    def run(x, ign, ccid):
        x = x.copy()
        assert ref.predict_visibilities_multifreq_withsol_withbeam(
            pr.u, pr.v, pr.w, pp.copy(), x, pr.N, pr.Nbase, pr.tilesz, b.fresh_barr(), sky, freqs,
            pr.fdelta * len(freqs), beam, ignorelist=ign, add_to_data=SIMUL_ADD, ccid=ccid,
            rho=1e-9) == 0
        return x

    zero = np.zeros_like(x0)
    m0 = run(zero, [0, 1, 1], -99999)
    m2 = run(zero, [1, 1, 0], -99999)
    got = run(x0, [0, 1, 0], 1)
    K = lambda x: _correct(x, pr, _jinv(pp, pr.N, 1, 1e-9), len(freqs))
    assert relerr(got, K(K(x0 + m0) + m2)) < 1e-12
    assert relerr(got, K(x0 + m0 + m2)) > 1e-3


def test_withsol_header_matches_the_reference_and_the_library():
    """include/dirac_b200_withsol.h declares exactly the three simulation entry points, each with the
    reference's own parameter type list (stored from Dirac_radio.h:490,529,666,
    tests/golden/make_golden_withsol_signatures.py), and the library exports them"""
    import json
    from sagecal_b200 import lib as blib
    from test_cpu_abi import _c_declarations
    ours = _c_declarations(os.path.join(ROOT, "include", "dirac_b200_withsol.h"))
    with open(os.path.join(ROOT, "tests", "golden", "ref_signatures_withsol.json")) as f:
        ref = json.load(f)
    assert sorted(ours) == sorted(ref) == sorted(blib.WITHSOL_EXPORTED), (sorted(ours), sorted(ref))
    for name, sigs in ours.items():
        assert len(sigs) == 1 and sigs[0] in ref[name], (name, sigs, ref[name])
    # the main header brings them in, and declares none of them itself
    main = _c_declarations(os.path.join(ROOT, "include", "dirac_b200.h"))
    assert not set(main) & set(ours)
    assert '#include "dirac_b200_withsol.h"' in open(os.path.join(ROOT, "include", "dirac_b200.h")).read()
    if os.path.exists(blib.LIB_PATH):
        import ctypes as C
        L = C.CDLL(blib.LIB_PATH)
        for name in ours:
            assert hasattr(L, name), name


def test_link_order_puts_the_simulation_on_this_library(tmp_path):
    """INTEGRATION.md section 2: `-ldirac_b200` in front of the reference's library takes the three
    simulation entry points and leaves read_solutions and update_ignorelist with the reference.  The
    reference's library is stood in for by one that, like it, defines all five names."""
    names = ["predict_visibilities_multifreq_withsol", "predict_visibilities_multifreq_withsol_withbeam",
             "predict_visibilities_withsol_withbeam_gpu", "read_solutions", "update_ignorelist"]
    refdir = str(tmp_path)
    stub = os.path.join(refdir, "dirac_ref_standin.c")
    with open(stub, "w") as f:
        f.write("".join("void %s(void) {}\n" % s for s in names))
    subprocess.check_call(["gcc", "-shared", "-fPIC", "-o", os.path.join(refdir, "libdirac_ref.so"), stub])
    exe = os.path.join(refdir, "link_order_withsol")
    libdir = os.path.join(ROOT, "sagecal_b200")
    cmd = ["gcc", "-O1", "-Wall", "-o", exe,
           os.path.join(ROOT, "tests", "c_caller", "link_order_withsol.c"),
           "-I", os.path.join(ROOT, "include"), "-L", libdir, "-ldirac_b200", "-L", refdir,
           "-ldirac_ref", "-ldl", "-lm", "-Wl,-rpath," + libdir, "-Wl,-rpath," + refdir,
           "-Wl,--allow-shlib-undefined"]
    subprocess.check_call(cmd)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, (out.stdout, out.stderr)
    got = dict(line.split() for line in out.stdout.strip().splitlines())
    assert got == {n: ("libdirac_ref.so" if n in ("read_solutions", "update_ignorelist")
                       else "libdirac_b200.so") for n in names}, got
