"""pytest configuration: `-m gpu` tests need an H100, everything else runs on CPU."""
import importlib
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100, sm_90a)")
    config.addinivalue_line("markers", "slow: long-running CPU test")


@pytest.fixture(scope="session")
def b200():
    """The product package (directory name is not an identifier)."""
    return importlib.import_module("mini-sglang_b200")


@pytest.fixture(scope="session")
def native_lib(b200):
    """libb200attn.so, built on demand (nvcc cross-compiles without a GPU)."""
    b200.build_native()
    return b200._cabi.load()


@pytest.fixture(autouse=True)
def _reset_ctx(b200):
    b200.core.set_global_ctx(None)
    yield
    b200.core.set_global_ctx(None)
