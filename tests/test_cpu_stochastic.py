"""CPU tier of the stochastic interval: include/dirac_b200_stochastic.h compiles on its own from a plain
C99 host and links against the library, which exports everything it declares; the call refuses more
bands than channels before it needs a device."""
import os
import subprocess

from test_cpu_abi import _c_declarations

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_stochastic_header_declares_the_exports():
    from sagecal_b200 import lib as blib
    ours = _c_declarations(os.path.join(ROOT, "include", "dirac_b200_stochastic.h"))
    assert sorted(ours) == sorted(blib.STOCHASTIC_EXPORTED), sorted(ours)
    main = _c_declarations(os.path.join(ROOT, "include", "dirac_b200.h"))
    assert not set(main) & set(ours)
    assert '#include "dirac_b200_stochastic.h"' in open(os.path.join(ROOT, "include", "dirac_b200.h")).read()


def test_plain_c_host_compiles_links_and_is_refused(tmp_path):
    exe = os.path.join(str(tmp_path), "stochastic_caller")
    libdir = os.path.join(ROOT, "sagecal_b200")
    subprocess.check_call(["gcc", "-std=c99", "-O1", "-Wall", "-Wextra", "-Werror", "-o", exe,
                           os.path.join(ROOT, "tests", "c_caller", "stochastic_caller.c"),
                           "-I", os.path.join(ROOT, "include"), "-L", libdir, "-ldirac_b200", "-lm",
                           "-Wl,-rpath," + libdir])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "STOCHASTIC_CALLER OK" in out.stdout, (out.stdout, out.stderr)
    assert "nsolbw = 2 bands of Nchan = 1 channels" in out.stderr
