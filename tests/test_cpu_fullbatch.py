"""CPU tier of the full-batch tile call: include/dirac_b200_fullbatch.h compiles on its own from a plain
C99 host with -Wall -Werror and links against the library, which exports exactly what it declares; both
calls refuse a tile without channels before they need a device."""
import os
import subprocess

from test_cpu_abi import _c_declarations

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_fullbatch_header_declares_the_exports():
    from sagecal_b200 import lib as blib
    ours = _c_declarations(os.path.join(ROOT, "include", "dirac_b200_fullbatch.h"))
    assert sorted(ours) == sorted(blib.FULLBATCH_EXPORTED), sorted(ours)
    main = _c_declarations(os.path.join(ROOT, "include", "dirac_b200.h"))
    assert not set(main) & set(ours)
    assert '#include "dirac_b200_fullbatch.h"' in open(os.path.join(ROOT, "include", "dirac_b200.h")).read()
    # the beam arguments sit after uvmax in the order of the _withbeam stochastic interval call
    plain = ours["dirac_b200_fullbatch_tile"][0]
    beam = ours["dirac_b200_fullbatch_tile_withbeam"][0]
    stoch = _c_declarations(os.path.join(ROOT, "include", "dirac_b200_stochastic.h"))
    sbeam = stoch["dirac_b200_stochastic_interval_withbeam"][0]
    assert beam == plain[:18] + sbeam[17:32] + plain[18:]


def test_plain_c_host_compiles_links_and_is_refused(tmp_path):
    exe = os.path.join(str(tmp_path), "fullbatch_caller")
    libdir = os.path.join(ROOT, "sagecal_b200")
    subprocess.check_call(["gcc", "-std=c99", "-O1", "-Wall", "-Wextra", "-Werror", "-o", exe,
                           os.path.join(ROOT, "tests", "c_caller", "fullbatch_caller.c"),
                           "-I", os.path.join(ROOT, "include"), "-L", libdir, "-ldirac_b200", "-lm",
                           "-Wl,-rpath," + libdir])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "FULLBATCH_CALLER OK" in out.stdout, (out.stdout, out.stderr)
    assert out.stderr.count("Nchan = 0 channels") == 2
