"""Bindings of GraphSCI's lean training schedule (``csrc/graphsci.cu``): the BatchNorm statistics without their apply, and the
three decoder heads fused with the ZINB / MSE loss, in training (gradient over the heads' buffers in place) and in evaluation
(row ranges).  Every tensor crosses the boundary through ``ops._arg`` and every entry point is invoked through ``ops._call``,
as in :mod:`dance_b200.ops`."""
from __future__ import annotations

from typing import Optional

import torch

from .ops import _F32, _F64, _U8, B2Error, _arg, _call, _stream, _workspace, lib


def batchnorm_stats(X, running_mean, running_var, training: bool, momentum: float = 0.1, eps: float = 1e-5, save_mean=None,
                    save_invstd=None, n: Optional[int] = None):
    """The statistics half of :func:`batchnorm_fwd`: returns (save_mean, save_invstd) [c] without applying them.  Training: from
    the rows of ``X`` (running statistics updated).  Eval: from the running statistics; ``X`` may then be None, with ``n`` rows."""
    c = running_mean.shape[0]
    if X is None:
        if training:
            raise B2Error("batchnorm_stats: training statistics need X")
        x, ldx, n = None, 0, int(n if n is not None else 1)
    else:
        x, ldx = _arg(X, "X", _F32, (None, c), ld=True)
        n = X.shape[0]
    dev = running_mean.device
    sm = torch.empty(c, dtype=_F32, device=dev) if save_mean is None else save_mean
    si = torch.empty(c, dtype=_F32, device=dev) if save_invstd is None else save_invstd
    ws = _workspace(lib().b2_batchnorm_workspace_bytes(c), dev)
    _call("b2_batchnorm_stats_f32", x, ldx, n, c, _arg(running_mean, "running_mean", _F32, c), _arg(running_var, "running_var", _F32, c),
          int(training), momentum, eps, _arg(sm, "save_mean", _F32, c), _arg(si, "save_invstd", _F32, c), *ws, _stream())
    return sm, si


def _heads_args(pre, gamma, beta, mean, invstd, Y, size_factors, mask, what):
    """Pointers of the fused GraphSCI heads' common operands: the three [n, g] pre-BatchNorm outputs (one leading dimension), the
    packed [3, g] BatchNorm vectors, Y, the size factors and the optional byte mask."""
    if len(pre) != 3:
        raise B2Error(f"{what}: expected the three heads' pre-BatchNorm outputs (pi, disp, mean)")
    a, ld = _arg(pre[0], f"{what}: pre_pi", _F32, (None, None), ld=True)
    n, g = pre[0].shape
    b, ldb = _arg(pre[1], f"{what}: pre_disp", _F32, (n, g), ld=True)
    c, ldc = _arg(pre[2], f"{what}: pre_mean", _F32, (n, g), ld=True)
    if ldb != ld or ldc != ld:
        raise B2Error(f"{what}: the three pre-BatchNorm outputs must share a leading dimension")
    if isinstance(mask, torch.Tensor) and mask.dtype == torch.bool:
        mask = mask.view(_U8)
    vecs = [_arg(t, f"{what}: {k}", _F32, (3, g)) for t, k in ((gamma, "gamma"), (beta, "beta"), (mean, "mean"), (invstd, "invstd"))]
    return n, g, (a, b, c, ld, *vecs, *_arg(Y, f"{what}: Y", _F32, (n, g), ld=True), _arg(size_factors, f"{what}: size_factors", _F32, n),
                  *_arg(mask, f"{what}: mask", _U8, (n, g), ld=True, optional=True), n, g)


def heads_train(pre, gamma, beta, mean, invstd, Y, size_factors, mask=None, le: float = 1.0, ke: float = 1.0,
                         dgamma=None, dbeta=None):
    """GraphSCI's three decoder heads (BatchNorm with the batch statistics ``mean`` / ``invstd`` + activations) fused with the
    ZINB / MSE loss and its gradient.  ``pre`` = (pre_pi, pre_disp, pre_mean) [n, g] is overwritten IN PLACE by the gradient of
    le·nll_mean + ke·(0.5/g)·mse_mean w.r.t. each head's pre-BatchNorm input; ``gamma`` … ``invstd`` are packed [3, g].
    Returns (acc3 fp64 {Σnll, Σmse, count}, dgamma [3, g], dbeta [3, g])."""
    n, g, args = _heads_args(pre, gamma, beta, mean, invstd, Y, size_factors, mask, "heads_train")
    dev = pre[0].device
    dgamma = torch.empty((3, g), dtype=_F32, device=dev) if dgamma is None else dgamma
    dbeta = torch.empty((3, g), dtype=_F32, device=dev) if dbeta is None else dbeta
    acc = torch.empty(3, dtype=_F64, device=dev)
    ws = _workspace(lib().b2_graphsci_heads_workspace_bytes(g), dev)
    _call("b2_graphsci_heads_train_f32", *args, float(le), float(ke), _arg(dgamma, "dgamma", _F32, (3, g)), _arg(dbeta, "dbeta", _F32, (3, g)),
          _arg(acc, "acc", _F64, 3), *ws, _stream())
    return acc, dgamma, dbeta


def heads_eval(pre, gamma, beta, mean, invstd, Y, size_factors, mask=None, acc=None, z_exp=None):
    """Eval-mode form of :func:`heads_train` over the rows of ``pre`` (read only): ``mean`` / ``invstd`` from the running
    statistics.  Adds {Σnll, Σmse, count} to ``acc`` (a new zeroed one when None) and writes mean·sf to ``z_exp`` when given
    (both may be row ranges of larger tensors).  Returns acc."""
    n, g, args = _heads_args(pre, gamma, beta, mean, invstd, Y, size_factors, mask, "heads_eval")
    accumulate = acc is not None
    acc = torch.empty(3, dtype=_F64, device=pre[0].device) if acc is None else acc
    _call("b2_graphsci_heads_eval_f32", *args, int(accumulate), _arg(acc, "acc", _F64, 3),
          *_arg(z_exp, "z_exp", _F32, (n, g), ld=True, optional=True), _stream())
    return acc
