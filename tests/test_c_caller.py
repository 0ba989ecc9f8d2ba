"""The C-ABI library compiled into and LINKED against a plain C host (tests/c_caller/caller.c), as the
reference driver would be: `gcc caller.c -I include -L sagecal_b200 -ldirac_b200`.  On a CPU box the
host only calls the index helpers and takes the address of every entry point; on the GPU box it also
runs precalculate_coherencies + sagefit_visibilities."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build(tmp_path):
    exe = os.path.join(str(tmp_path), "caller")
    libdir = os.path.join(ROOT, "sagecal_b200")
    cmd = ["gcc", "-O1", "-Wall", "-Werror", "-o", exe, os.path.join(ROOT, "tests", "c_caller", "caller.c"),
           "-I", os.path.join(ROOT, "include"), "-L", libdir, "-ldirac_b200", "-lm",
           "-Wl,-rpath," + libdir]
    subprocess.check_call(cmd)
    return exe


def test_c_host_links_and_calls_host_helpers(tmp_path):
    exe = build(tmp_path)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "C_CALLER OK" in out.stdout, (out.returncode, out.stdout, out.stderr)


@pytest.mark.gpu
def test_c_host_runs_the_solver(tmp_path):
    exe = build(tmp_path)
    out = subprocess.run([exe, "gpu"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "C_CALLER OK" in out.stdout, (out.returncode, out.stdout, out.stderr)


# every name link_order.c looks up: the hot-path entry points and three reference-only helpers
LINK_ORDER_SYMBOLS = ["sagefit_visibilities", "sagefit_visibilities_dual_pt_flt", "bfgsfit_visibilities",
                      "bfgsfit_visibilities_gpu", "precalculate_coherencies",
                      "precalculate_coherencies_withbeam_gpu", "predict_visibilities_multifreq",
                      "calculate_residuals_multifreq", "sagefit_visibilities_admm",
                      "bfgsfit_minibatch_visibilities", "lbfgs_persist_init", "generate_baselines",
                      "preset_flags_and_data", "whiten_data", "my_dscal", "my_dnrm2", "update_w_and_nu"]


def test_link_order_puts_the_hot_path_on_this_library(tmp_path):
    """INTEGRATION.md section 2 on a CPU box: `-ldirac_b200` in front of the reference's library takes
    over the hot-path symbols and leaves the rest with the reference.  The reference's library is
    stood in for by one that, like it, defines every name link_order.c looks up."""
    refdir = str(tmp_path)
    stub = os.path.join(refdir, "dirac_ref_standin.c")
    with open(stub, "w") as f:
        f.write("".join("void %s(void) {}\n" % s for s in LINK_ORDER_SYMBOLS))
    subprocess.check_call(["gcc", "-shared", "-fPIC", "-o", os.path.join(refdir, "libdirac_ref.so"), stub])
    exe = os.path.join(refdir, "link_order")
    libdir = os.path.join(ROOT, "sagecal_b200")
    cmd = ["gcc", "-O1", "-Wall", "-o", exe, os.path.join(ROOT, "tests", "c_caller", "link_order.c"),
           "-I", os.path.join(ROOT, "include"), "-L", libdir, "-ldirac_b200", "-L", refdir,
           "-ldirac_ref", "-ldl", "-lm", "-Wl,-rpath," + libdir, "-Wl,-rpath," + refdir,
           "-Wl,--allow-shlib-undefined"]
    subprocess.check_call(cmd)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, (out.stdout, out.stderr)
    got = dict(line.split() for line in out.stdout.strip().splitlines())
    assert sorted(got) == sorted(LINK_ORDER_SYMBOLS), got
    ours = [s for s, lib in got.items() if lib == "libdirac_b200.so"]
    theirs = [s for s, lib in got.items() if lib == "libdirac_ref.so"]
    assert sorted(theirs) == ["my_dnrm2", "my_dscal", "update_w_and_nu"], got
    assert len(ours) == len(got) - 3 and "sagefit_visibilities" in ours and "whiten_data" in ours, got


def test_struct_layouts_equal_the_reference_headers(tmp_path):
    """baseline_t, clus_source_t, exinfo_*, elementcoeff, the prefix of persistent_data_t and the
    STYPE_ / DOBEAM_ / STAT_ / SM_ constants: same sizes, offsets and values as a caller compiled
    against the reference's Dirac.h / Dirac_radio.h sees (74 lines compared; the reference's side is
    stored, tests/golden/make_golden_headers.py)."""
    exe = os.path.join(str(tmp_path), "ours")
    subprocess.check_call(["gcc", "-w", "-o", exe, os.path.join(ROOT, "tests", "c_caller", "layout.c"),
                           "-I", os.path.join(ROOT, "include")])
    ours = subprocess.run([exe], capture_output=True, text=True, timeout=60).stdout
    with open(os.path.join(ROOT, "tests", "golden", "ref_layout.txt")) as f:
        ref = f.read()
    assert ours == ref and len(ref.splitlines()) > 70
