"""Bindings of the coordinate sweeps of SpaGCN's spot graph (``csrc/spatial_adj.cu``): the weighted product, the weight total and
the nearest spots between two spot coordinate sets, without the N × N matrices.  Every tensor crosses the boundary through
``ops._arg`` and every entry point is invoked through ``ops._call``, as in :mod:`dance_b200.ops`; shapes, ``d`` and ``l`` are
checked before that."""
from __future__ import annotations

from typing import Optional

import torch

from .ops import _F32, _F64, _I32, B2Error, _arg, _call, _stream, _workspace, lib


def _spot_coords(rows: torch.Tensor, cols: torch.Tensor, where: str):
    """(n_rows, n_cols, d) of two coordinate sets [n, d] with 1 <= d <= 4."""
    for name, P in (("rows", rows), ("cols", cols)):
        if not isinstance(P, torch.Tensor) or P.dim() != 2:
            raise B2Error(f"{where}: {name} must be a 2-D tensor of spot coordinates")
    d = rows.shape[1]
    if not 1 <= d <= 4 or cols.shape[1] != d:
        raise B2Error(f"{where}: rows and cols need the same number of coordinates, 1 to 4 (got {rows.shape[1]} and {cols.shape[1]})")
    return rows.shape[0], cols.shape[0], d


def _coord_ptrs(rows: torch.Tensor, cols: torch.Tensor, d: int):
    return _arg(rows, "rows", _F32, (None, d)), _arg(cols, "cols", _F32, (None, d))


def _check_l(l: float, where: str) -> float:
    l = float(l)
    if not (l > 0.0 and l < float("inf")):
        raise B2Error(f"{where}: l must be positive and finite, got {l}")
    return l


def spatial_exp_adj_matmul(rows: torch.Tensor, cols: torch.Tensor, l: float, X: torch.Tensor, out: Optional[torch.Tensor] = None):
    """``AX = W · X`` with ``W_rc = exp(-D_rc² / (2 l²))`` of the euclidean distance between ``rows[r]`` and ``cols[c]``, the
    weight ``exp_adj(pairwise_l2_dense(...))`` gives for the pair, never materialised.  X [n_cols, F] fp32; tf32x3 tensor
    cores, error ~2⁻²¹ of ``W · |X|``."""
    l = _check_l(l, "spatial_exp_adj_matmul")
    if not isinstance(X, torch.Tensor) or X.dim() != 2 or X.shape[1] < 1:
        raise B2Error("spatial_exp_adj_matmul: X must be a 2-D tensor with at least one column")
    nr, nc, d = _spot_coords(rows, cols, "spatial_exp_adj_matmul")
    if nr < 1 or nc < 1 or X.shape[0] != nc:
        raise B2Error(f"spatial_exp_adj_matmul: {nr} rows, {nc} cols and X {tuple(X.shape)} do not fit (X needs n_cols rows)")
    r, c = _coord_ptrs(rows, cols, d)
    F = X.shape[1]
    x, ldx = _arg(X, "X", _F32, (nc, F), ld=True)
    out = torch.empty((nr, F), dtype=_F32, device=X.device) if out is None else out
    o, ldo = _arg(out, "out", _F32, (nr, F), ld=True)
    ws = _workspace(lib().b2_spatial_exp_adj_mm_workspace_bytes(nc, F), X.device)
    _call("b2_spatial_exp_adj_mm_f32", r, nr, c, nc, d, l, x, ldx, F, o, ldo, *ws, _stream())
    return out


def spatial_exp_adj_sum(rows: torch.Tensor, cols: torch.Tensor, l: float) -> torch.Tensor:
    """``Σ_rc exp(-D_rc² / (2 l²))`` over the distances between two coordinate sets, fp64 [1] on the device."""
    l = _check_l(l, "spatial_exp_adj_sum")
    nr, nc, d = _spot_coords(rows, cols, "spatial_exp_adj_sum")
    r, c = _coord_ptrs(rows, cols, d)
    acc = torch.empty(1, dtype=_F64, device=rows.device)
    _call("b2_spatial_exp_adj_sum_f32", r, nr, c, nc, d, l, _arg(acc, "sum", _F64, 1), _stream())
    return acc


def spatial_nearest(rows: torch.Tensor, cols: torch.Tensor, m: int) -> torch.Tensor:
    """int32 [n_rows, m], 1 <= m <= 8: per row the m columns of smallest fp32 distance (``pairwise_l2_dense``'s entries), ties
    to the lower column index — ``torch.sort(D, stable=True).indices[:, :m]`` of the materialised matrix."""
    m = int(m)
    nr, nc, d = _spot_coords(rows, cols, "spatial_nearest")
    if not 1 <= m <= min(8, nc):
        raise B2Error(f"spatial_nearest: m={m} outside 1..min(8, n_cols={nc})")
    r, c = _coord_ptrs(rows, cols, d)
    idx = torch.empty((nr, m), dtype=_I32, device=rows.device)
    _call("b2_spatial_nearest_f32", r, nr, c, nc, d, m, _arg(idx, "idx", _I32, (nr, m)), _stream())
    return idx
