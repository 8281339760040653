"""The ops-boundary checks of tests/test_ops_boundary.py applied to dance_b200/leiden.py, without a GPU: its library calls go
through ``ops._call``, its pointers come from ``ops._arg``, and it refuses CPU tensors before any library call."""
import ast
from pathlib import Path

import pytest
import torch

from dance_b200 import leiden, ops
from dance_b200._lib import B2Error

TREE = ast.parse(Path(leiden.__file__).read_text())


def test_library_calls_go_through_call():
    direct = sorted({n.attr for n in ast.walk(TREE) if isinstance(n, ast.Attribute) and n.attr.startswith("b2_")
                     and not n.attr.endswith("_workspace_bytes")})
    assert direct == []
    called = {n.func.attr if isinstance(n.func, ast.Attribute) else getattr(n.func, "id", None) for n in ast.walk(TREE)
              if isinstance(n, ast.Call)}
    assert "check" not in called and "_call" in called
    assert any(isinstance(n, ast.Constant) and n.value == "b2_leiden_f32" for n in ast.walk(TREE))


def test_pointers_come_from_the_accessor():
    assert not any(isinstance(n, ast.Attribute) and n.attr == "data_ptr" for n in ast.walk(TREE))


class Recorder:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if name == "b2_last_error":
            return lambda: b"recorded"
        if name.endswith("_workspace_bytes"):
            return lambda *a: 1 << 10
        return lambda *a: self.calls.append(name) or 0


def _cpu_csr(vals=True):
    A = ops.CSR.__new__(ops.CSR)
    A.rowptr = torch.tensor([0, 1, 2], dtype=torch.int32)
    A.colidx = torch.tensor([1, 0], dtype=torch.int32)
    A.vals = torch.ones(2) if vals else None
    A.shape, A.ptrs, A._t = (2, 2), (1, 1, 1 if vals else None), None
    return A


@pytest.mark.parametrize("vals", [True, False])
def test_leiden_refuses_cpu_tensors(monkeypatch, vals):
    rec = Recorder()
    monkeypatch.setattr(ops, "_raw_lib", lambda: rec)
    with pytest.raises(B2Error, match="expected a CUDA tensor"):
        leiden.leiden(_cpu_csr(vals))
    assert rec.calls == []


def test_neighbor_graph_refuses_cpu_tensors(monkeypatch):
    rec = Recorder()
    monkeypatch.setattr(ops, "_raw_lib", lambda: rec)
    with pytest.raises(B2Error, match="expected a CUDA tensor"):
        leiden.neighbor_graph(torch.zeros(8, 4), 3)
    assert rec.calls == []
