import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def ref():
    """the compiled reference CPU path (oracle/_ref), test infrastructure only: its recorded answers
    (tests/golden/ref), or the live library recording them when DIRAC_REF_RECORD is set"""
    import refdirac
    return refdirac.recorded()


@pytest.fixture(scope="session")
def refser():
    """the compiled reference with the worker threads of its robust RTR / NSD solvers run
    synchronously (oracle/ref_shim_rtr_serial.c): deterministic pin of solver_mode 5 and 6"""
    import refdirac
    return refdirac.recorded(serial=True)


@pytest.fixture(scope="session")
def api():
    """the product library; GPU tests only"""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from sagecal_b200 import lib
    return lib.load()
