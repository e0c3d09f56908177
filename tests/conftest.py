import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with `-m gpu`)")


@pytest.fixture(scope="session")
def cuda_lib():
    """Build (if needed) and load the CUDA library; GPU tests must never run on a fallback."""
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from magicpig_b200 import _native

    if not os.path.exists(_native.LIB_PATH):
        from magicpig_b200 import build
        build.build()
    return _native.load()
