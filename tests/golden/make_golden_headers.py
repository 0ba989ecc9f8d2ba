"""What the reference's own headers say about the C ABI this library shares with it, stored so that the
ABI tests run without the reference sources:
  ref_layout.txt      sizes, field offsets and constants a caller compiled against the reference's
                      Dirac.h / Dirac_radio.h sees (tests/c_caller/layout.c built with -DUSE_REF);
  ref_signatures.json the reference's parameter type lists of every entry point include/dirac_b200.h
                      declares under a reference name (test_cpu_abi._c_declarations).

    python tests/golden/make_golden_headers.py <reference repository root>
"""
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from test_cpu_abi import _c_declarations  # noqa: E402


def main(ref_root):
    lib = os.path.join(ref_root, "src", "lib")
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "layout")
        subprocess.check_call(["gcc", "-w", "-o", exe, os.path.join(ROOT, "tests", "c_caller", "layout.c"),
                               "-DUSE_REF", "-I", os.path.join(lib, "Dirac"), "-I", os.path.join(lib, "Radio")])
        layout = subprocess.run([exe], capture_output=True, text=True, check=True, timeout=60).stdout
    with open(os.path.join(HERE, "ref_layout.txt"), "w") as f:
        f.write(layout)
    ref = {}
    for h in ("Dirac/Dirac.h", "Dirac/Dirac_common.h", "Radio/Dirac_radio.h"):
        for k, v in _c_declarations(os.path.join(lib, h)).items():
            ref.setdefault(k, []).extend(v)
    ours = _c_declarations(os.path.join(ROOT, "include", "dirac_b200.h"))
    wanted = sorted({n[:-4] if n.endswith("_hbb") else n for n in ours if not n.startswith("dirac_b200")})
    with open(os.path.join(HERE, "ref_signatures.json"), "w") as f:
        json.dump({n: ref[n] for n in wanted if n in ref}, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main(sys.argv[1])
