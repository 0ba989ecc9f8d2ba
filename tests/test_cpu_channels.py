"""CPU tier of the per-channel refinement (driver option -b 1): the header of calculate_residuals and
dirac_b200_bfgsfit_channels against the reference's declaration and the library's exports, and the
link order that puts the channel loop's calls on this library."""
import json
import os
import subprocess

from test_cpu_abi import _c_declarations

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_channels_header_matches_the_reference_and_the_library():
    """include/dirac_b200_channels.h declares calculate_residuals with the reference's own parameter
    type list (stored from Dirac_radio.h:639, tests/golden/make_golden_channels_signatures.py) next to
    the library's own entry points, and the library exports all of them"""
    from sagecal_b200 import lib as blib
    ours = _c_declarations(os.path.join(ROOT, "include", "dirac_b200_channels.h"))
    with open(os.path.join(ROOT, "tests", "golden", "ref_signatures_channels.json")) as f:
        ref = json.load(f)
    assert sorted(ours) == sorted(blib.CHANNELS_EXPORTED), sorted(ours)
    assert sorted(n for n in ours if not n.startswith("dirac_b200")) == sorted(ref) == ["calculate_residuals"]
    for name in ref:
        assert len(ours[name]) == 1 and ours[name][0] in ref[name], (name, ours[name], ref[name])
    # the main header brings them in, and declares none of them itself
    main = _c_declarations(os.path.join(ROOT, "include", "dirac_b200.h"))
    assert not set(main) & set(ours)
    assert '#include "dirac_b200_channels.h"' in open(os.path.join(ROOT, "include", "dirac_b200.h")).read()
    if os.path.exists(blib.LIB_PATH):
        import ctypes as C
        L = C.CDLL(blib.LIB_PATH)
        for name in ours:
            assert hasattr(L, name), name


def test_link_order_puts_the_channel_loop_on_this_library(tmp_path):
    """INTEGRATION.md section 2: `-ldirac_b200` in front of the reference's library takes
    precalculate_coherencies, bfgsfit_visibilities(_gpu) and calculate_residuals and leaves
    read_solutions with the reference.  The reference's library is stood in for by one that, like it,
    defines all the reference's names."""
    ref_names = ["precalculate_coherencies", "bfgsfit_visibilities", "bfgsfit_visibilities_gpu",
                 "calculate_residuals", "read_solutions"]
    refdir = str(tmp_path)
    stub = os.path.join(refdir, "dirac_ref_standin.c")
    with open(stub, "w") as f:
        f.write("".join("void %s(void) {}\n" % s for s in ref_names))
    subprocess.check_call(["gcc", "-shared", "-fPIC", "-o", os.path.join(refdir, "libdirac_ref.so"), stub])
    exe = os.path.join(refdir, "link_order_channels")
    libdir = os.path.join(ROOT, "sagecal_b200")
    cmd = ["gcc", "-O1", "-Wall", "-o", exe,
           os.path.join(ROOT, "tests", "c_caller", "link_order_channels.c"),
           "-I", os.path.join(ROOT, "include"), "-L", libdir, "-ldirac_b200", "-L", refdir,
           "-ldirac_ref", "-ldl", "-lm", "-Wl,-rpath," + libdir, "-Wl,-rpath," + refdir,
           "-Wl,--allow-shlib-undefined"]
    subprocess.check_call(cmd)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, (out.stdout, out.stderr)
    got = dict(line.split() for line in out.stdout.strip().splitlines())
    want = {n: "libdirac_b200.so" for n in ref_names[:4] + ["dirac_b200_bfgsfit_channels"]}
    want["read_solutions"] = "libdirac_ref.so"
    assert got == want, got
