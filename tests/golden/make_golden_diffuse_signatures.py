"""The reference's parameter type list of recalculate_diffuse_coherencies, the reference entry point
include/dirac_b200_diffuse.h declares, stored so that tests/test_oracle_diffuse_math.py checks the
header without the reference sources:

    python tests/golden/make_golden_diffuse_signatures.py <reference repository root>
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
    with open(os.path.join(HERE, "ref_signatures_diffuse.json"), "w") as f:
        json.dump({"recalculate_diffuse_coherencies": ref["recalculate_diffuse_coherencies"]}, f,
                  indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main(sys.argv[1])
