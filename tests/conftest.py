import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


@pytest.fixture(scope="session", autouse=True)
def _built_libraries():
    """Build the oracle (CPU) and the CUDA library if they are stale; both builds work without a GPU."""
    import oracle
    so = os.path.join(ROOT, "oracle", "liboracle_tsdf.so")
    if not os.path.exists(so):
        oracle.build()
    from pyslam_b200 import build as b
    if os.path.exists("/usr/local/cuda/bin/nvcc") or __import__("shutil").which("nvcc"):
        b.build()
    yield


def has_gpu() -> bool:
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False
