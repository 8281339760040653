import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

GOLDEN = Path(__file__).resolve().parent / "golden"


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (select with `-m gpu`)")


@pytest.fixture(scope="session")
def golden():
    def load(name):
        return np.load(GOLDEN / f"{name}.npz")
    return load


@pytest.fixture
def assert_ary_isclose():
    # same helper (and tolerances) as the reference's tests/conftest.py:5-15
    def _assert(x, y, rtol=1e-5, atol=1e-8):
        x, y = np.asarray(x), np.asarray(y)
        assert x.shape == y.shape, f"shape mismatch {x.shape} vs {y.shape}"
        assert np.allclose(x, y, rtol=rtol, atol=atol), f"max abs diff {np.abs(x - y).max()}"
    return _assert


@pytest.fixture(scope="session")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from dance_b200 import _lib
    _lib.lib()  # fail loudly if the extension is missing on a GPU box
    return torch.device("cuda:0")


def _host(a):
    return a.detach().cpu().numpy() if hasattr(a, "detach") else a


def rel_err(a, b):
    a = np.asarray(_host(a), dtype=np.float64)
    b = np.asarray(_host(b), dtype=np.float64)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30)
