import os
import sys
from pathlib import Path

import pytest

REPO = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(REPO))

ORACLE_DIR = REPO / "oracle"
PORT_SO = ORACLE_DIR / "_ref" / "liboracle_port.so"


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def _have_gpu():
    try:
        import ctypes
        from handbrake_b200 import LIBHBCU
        lib = ctypes.CDLL(str(LIBHBCU))
        return lib.hbcu_device_count() > 0
    except OSError:
        return False


@pytest.fixture(scope="session")
def ref():
    """the reference's own filters, answered from their stored result digests (tests/golden_ref.py)"""
    from golden_ref import GoldenRef
    return GoldenRef()


@pytest.fixture(scope="session")
def cuda_filters():
    import handbrake_b200
    if not _have_gpu():
        pytest.fail("GPU test selected but no CUDA device is visible: there is no CPU fallback")
    return handbrake_b200.filters()
