import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
PKG = ROOT / "3dgsconverter_b200"
for p in (str(ROOT), str(PKG)):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")
    config.addinivalue_line("markers", "slow: takes more than a few seconds on CPU")


@pytest.fixture(scope="session")
def gsx_lib():
    """libgsx.so, built on demand (nvcc cross-compiles without a GPU)."""
    so = PKG / "lib" / "libgsx.so"
    if not so.exists():
        sys.path.insert(0, str(ROOT))
        import __graft_entry__ as g
        g.build()
    from gsx import _abi
    return _abi.lib


@pytest.fixture(scope="session")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")
