import ctypes
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    # the synthetic renderer works on tiny tensors: intra-op threading only adds (large) overhead
    import torch
    torch.set_num_threads(1)


@pytest.fixture(scope="session")
def oracle_lib():
    """The CPU oracle (test infrastructure). Built on demand with oracle/Makefile."""
    path = os.path.join(ROOT, "oracle", "liboracle.so")
    if not os.path.exists(path):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle")])
    return ctypes.CDLL(path)


@pytest.fixture(scope="session")
def product_lib():
    import khronos_b200
    return khronos_b200.lib()
