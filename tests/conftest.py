import os
import sys

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
def cabi_double(monkeypatch):
    """Route the package's C-ABI calls to the torch test double (tests/cabi_double.py) for host-logic tests on CPU."""
    import torch

    from chatts_b200 import _cabi
    from tests.cabi_double import TorchDouble

    dbl = TorchDouble()
    monkeypatch.setattr(_cabi, "get_context", lambda device=None: dbl)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self, raising=False)
    return dbl
