import os
import shutil
import sys
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture
def ipc_dir():
    """A fresh directory with a short path for ipc:// sockets: a Unix socket path holds at most 107 bytes, which
    pytest's tmp_path under a long temporary directory can exceed."""
    d = tempfile.mkdtemp(prefix="dm", dir="/tmp")
    yield d
    shutil.rmtree(d, ignore_errors=True)
