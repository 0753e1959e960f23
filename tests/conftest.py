import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")


@pytest.fixture
def emu(monkeypatch):
    """Host-logic tests: run the block composition on CPU with the torch emulation of the kernels."""
    import emu_kernels
    emu_kernels.install(monkeypatch)
    return emu_kernels
