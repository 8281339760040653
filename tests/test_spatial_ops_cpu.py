"""The coordinate sweeps of SpaGCN's spot graph without a GPU: the boundary of ``dance_b200.spatial_ops`` refuses bad input
before any launch, and the product kernel's code keeps its wgmmas asynchronous (see kernel_codegen.py)."""
import ast
import re
from pathlib import Path

import pytest
import torch

from dance_b200 import ops, spatial_ops
from dance_b200._lib import B2Error
from kernel_codegen import compiled, needs_cuobjdump, needs_nvcc

SRC = ast.parse(Path(spatial_ops.__file__).read_text())


class _Recorder:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if name.endswith("_workspace_bytes"):
            return lambda *a: 0
        return lambda *a: self.calls.append(name) or 0


@pytest.fixture
def recorder(monkeypatch):
    rec = _Recorder()
    monkeypatch.setattr(ops, "_raw_lib", lambda: rec)
    return rec


def f32(*shape):
    return torch.zeros(shape, dtype=torch.float32)


def test_pointers_and_calls_go_through_the_ops_accessors():
    assert not any(isinstance(n, ast.Attribute) and n.attr == "data_ptr" for n in ast.walk(SRC))
    direct = {n.attr for n in ast.walk(SRC) if isinstance(n, ast.Attribute) and n.attr.startswith("b2_")}
    assert direct == {"b2_spatial_exp_adj_mm_workspace_bytes"}


CASES = {
    "matmul": lambda rows, cols, l: spatial_ops.spatial_exp_adj_matmul(rows, cols, l, f32(cols.shape[0], 4)),
    "sum": lambda rows, cols, l: spatial_ops.spatial_exp_adj_sum(rows, cols, l),
    "nearest": lambda rows, cols, l: spatial_ops.spatial_nearest(rows, cols, 3),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_refuses_before_launching(recorder, name):
    fn = CASES[name]
    with pytest.raises(B2Error, match="expected a CUDA tensor"):
        fn(f32(6, 2), f32(6, 2), 1.0)
    with pytest.raises(B2Error, match="1 to 4"):
        fn(f32(6, 5), f32(6, 5), 1.0)
    with pytest.raises(B2Error, match="1 to 4"):
        fn(f32(6, 2), f32(6, 3), 1.0)
    with pytest.raises(B2Error, match="2-D"):
        fn(f32(6), f32(6, 2), 1.0)
    if name != "nearest":
        for l in (0.0, -1.0, float("inf"), float("nan")):
            with pytest.raises(B2Error, match="positive and finite"):
                fn(f32(6, 2), f32(6, 2), l)
    assert recorder.calls == []


def test_shape_checks(recorder):
    with pytest.raises(B2Error, match="do not fit"):
        spatial_ops.spatial_exp_adj_matmul(f32(6, 2), f32(6, 2), 1.0, f32(5, 4))
    with pytest.raises(B2Error, match="at least one column"):
        spatial_ops.spatial_exp_adj_matmul(f32(6, 2), f32(6, 2), 1.0, f32(6, 0))
    for m in (0, 9, 7):
        with pytest.raises(B2Error, match="outside"):
            spatial_ops.spatial_nearest(f32(6, 2), f32(6, 2), m)
    assert recorder.calls == []


def test_c_entry_points_validate_without_a_gpu():
    from dance_b200 import _lib
    lib = _lib.lib()
    assert lib.b2_spatial_exp_adj_sum_f32(None, 4, None, 4, 2, 1.0, None, None) == -1
    assert b"null pointer" in lib.b2_last_error()
    p = 16   # never dereferenced: validation fails first
    assert lib.b2_spatial_exp_adj_sum_f32(p, 4, p, 4, 5, 1.0, p, None) == -1
    assert b"d=5" in lib.b2_last_error()
    assert lib.b2_spatial_exp_adj_sum_f32(p, 4, p, 4, 2, 0.0, p, None) == -1
    assert lib.b2_spatial_nearest_f32(p, 4, p, 4, 2, 9, p, None) == -1
    assert lib.b2_spatial_exp_adj_mm_f32(p, 4, p, 4, 2, 1.0, p, 4, 4, p, 4, p, 0, None) == -1
    assert b"workspace" in lib.b2_last_error()
    assert lib.b2_spatial_exp_adj_mm_workspace_bytes(100, 50) == 4 * 2 * 64 * 128
    assert lib.b2_spatial_exp_adj_mm_workspace_bytes(33, 130) == 2 * 2 * 64 * 128
    assert lib.b2_spatial_exp_adj_mm_workspace_bytes(1, 3) == 2 * 8 * 128


@needs_nvcc
def test_product_kernel_keeps_its_wgmmas_async():
    c = compiled("spatial_adj.cu")
    names = c.kernels("spatial_exp_adj_mm_kernel")
    assert len(names) == 4                              # N = 8, 16, 32, 64
    for name in names:
        assert c.frame(name) == (0, 0, 0), name         # no stack frame, no spills
        assert c.serialised(name) == [], name


@needs_cuobjdump
def test_product_hgmmas_take_descriptors_from_uniform_registers():
    c = compiled("spatial_adj.cu")
    for name in c.kernels("spatial_exp_adj_mm_kernel"):
        hgmma = [l for l in c.sass(name).splitlines() if "HGMMA" in l]
        assert len(hgmma) >= 12, name                   # 4 k-steps x 3 products per tile
        assert all(re.search(r"gdesc\[UR\d+\]", l) for l in hgmma), name
