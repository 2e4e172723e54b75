import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    """The CPU oracle (oracle/bodo_oracle.c) — the checker, never the thing under test."""
    from oracle import oracle as O

    O.build()
    return O


@pytest.fixture(scope="session")
def gpu_lib():
    """libbodo_b200.so with a visible GPU; a missing library or device FAILS the test (no fallback)."""
    from bodo_b200 import _lib

    L = _lib.lib()
    assert L.b200_device_count() > 0, "gpu-marked test ran without a CUDA device"
    return L
