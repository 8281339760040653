"""Argument validation of b2_leiden_f32 (no GPU needed): every case is rejected before any CUDA call, so it runs on a machine
without a device and the stand-in pointers are never dereferenced."""
import math

import pytest

INVALID = -1
P = 1 << 20          # a 16-byte aligned stand-in address
N, NNZ = 100, 1000

ORDER = ["rowptr", "colidx", "vals", "n", "nnz", "resolution", "max_iterations", "labels", "n_comm", "quality", "info", "workspace",
         "workspace_bytes"]
DEFAULTS = dict(rowptr=P, colidx=P, vals=None, n=N, nnz=NNZ, resolution=1.0, max_iterations=-1, labels=P, n_comm=P, quality=P,
                info=None, workspace=P, workspace_bytes=None)
CASES = [
    *[{k: None} for k in ("rowptr", "colidx", "labels", "n_comm", "quality", "workspace")],
    {"n": 0}, {"n": -5}, {"nnz": -1},
    {"resolution": -0.1}, {"resolution": math.inf}, {"resolution": math.nan},
    {"max_iterations": 0}, {"max_iterations": -2},
    {"workspace_bytes": "short"},
]


@pytest.mark.parametrize("kw", CASES, ids=["-".join(f"{k}={v}" for k, v in c.items()) for c in CASES])
def test_leiden_entry_point_validation(kw):
    from dance_b200 import _lib
    lib = _lib.lib()
    a = dict(DEFAULTS, **kw)
    need = lib.b2_leiden_workspace_bytes(N, NNZ)
    a["workspace_bytes"] = need - 1 if a["workspace_bytes"] == "short" else need
    assert lib.b2_leiden_f32(*[a[k] for k in ORDER], None) == INVALID
    assert lib.b2_last_error().decode().startswith("b2_leiden_f32:")


def test_workspace_bound_depends_on_the_input_size_only():
    from dance_b200 import _lib
    lib = _lib.lib()
    assert lib.b2_leiden_workspace_bytes(0, 10) == 0 and lib.b2_leiden_workspace_bytes(10, -1) == 0
    assert lib.b2_leiden_workspace_bytes(10, 1 << 31) == 0
    small, large = lib.b2_leiden_workspace_bytes(1000, 10_000), lib.b2_leiden_workspace_bytes(1000, 20_000)
    assert 0 < small < large
