"""CPU tier of the stochastic interval calls with station beams (sagecal -N -M -w -B, and with -A):
include/dirac_b200_stochastic.h compiles on its own from a plain C99 host, which links and is refused
for the lunar element beam (doBeam = 7) before the library needs a device."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_plain_c_host_compiles_links_and_is_refused(tmp_path):
    exe = os.path.join(str(tmp_path), "stochastic_beam_caller")
    libdir = os.path.join(ROOT, "sagecal_b200")
    subprocess.check_call(["gcc", "-std=c99", "-O1", "-Wall", "-Wextra", "-Werror", "-o", exe,
                           os.path.join(ROOT, "tests", "c_caller", "stochastic_beam_caller.c"),
                           "-I", os.path.join(ROOT, "include"), "-L", libdir, "-ldirac_b200", "-lm",
                           "-Wl,-rpath," + libdir])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "STOCHASTIC_BEAM_CALLER OK" in out.stdout, (out.stdout, out.stderr)
    for fn in ("dirac_b200_stochastic_interval_withbeam",
               "dirac_b200_stochastic_consensus_interval_withbeam"):
        assert "%s: doBeam = 7 is not a beam mode" % fn in out.stderr, out.stderr
