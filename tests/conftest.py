import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA GPU with sm_90a (H100)")


@pytest.fixture(scope="session")
def golden():
    import numpy as np

    return dict(np.load(os.path.join(ROOT, "tests", "golden", "nf4_golden.npz")))


@pytest.fixture(scope="session")
def c_oracle():
    """ctypes handle on the C restatement (oracle/nf4_oracle.c), built on demand."""
    import ctypes as ct
    import subprocess

    so = os.path.join(ROOT, "oracle", "_build", "libnf4_oracle.so")
    src = os.path.join(ROOT, "oracle", "nf4_oracle.c")
    if not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.run(["make", "-C", os.path.join(ROOT, "oracle")], check=True, capture_output=True)
    lib = ct.CDLL(so)
    lib.nf4o_lut.restype = ct.POINTER(ct.c_float)
    lib.nf4o_thresholds.restype = ct.POINTER(ct.c_float)
    return lib
