"""The reference's parameter type lists of the entry points include/dirac_b200_withsol.h declares, stored
so that the ABI test of the simulation calls (tests/test_cpu_withsol.py) runs without the reference
sources:

    python tests/golden/make_golden_withsol_signatures.py <reference repository root>
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from test_cpu_abi import _c_declarations  # noqa: E402


def main(ref_root):
    ref = _c_declarations(os.path.join(ref_root, "src", "lib", "Radio", "Dirac_radio.h"))
    ours = _c_declarations(os.path.join(ROOT, "include", "dirac_b200_withsol.h"))
    with open(os.path.join(HERE, "ref_signatures_withsol.json"), "w") as f:
        json.dump({n: ref[n] for n in sorted(ours)}, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main(sys.argv[1])
