"""float64 restatements of the bf16 GEMM mode, for the tests: every product rounds its two operands to bfloat16 the way the
kernel does (round-to-nearest-even, torch's ``.to(torch.bfloat16)``) and is then computed exactly in float64.

:func:`feature_ae_step_bf16` is ``oracle.scgnn_step_ref.feature_ae_step`` with each of its four products replaced by
:class:`Bf16MatMul`, whose backward rounds its operands as well: the engine's dX and dW GEMMs run in bf16 too.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from oracle.scgnn_step_ref import FEATURE_AE_PARAMS


def bf16(x: torch.Tensor) -> torch.Tensor:
    """``x`` rounded to bfloat16 (nearest even), as float64."""
    return x.to(torch.bfloat16).to(torch.float64)


class Bf16MatMul(torch.autograd.Function):
    """``a @ b`` with both operands rounded to bf16; the gradients ``g @ bᵀ`` and ``aᵀ @ g`` round theirs too."""

    @staticmethod
    def forward(ctx, a, b):
        ctx.save_for_backward(a, b)
        return bf16(a) @ bf16(b)

    @staticmethod
    def backward(ctx, g):
        a, b = ctx.saved_tensors
        return bf16(g) @ bf16(b).t(), bf16(a).t() @ bf16(g)


def feature_ae_step_bf16(x: torch.Tensor, params: Dict[str, torch.Tensor], regularizer_type: str = "LTMG",
                         regu_strength: float = 0.9, ltmg: Optional[torch.Tensor] = None) -> dict:
    """Forward, loss and backward of one Feature-AE mini-batch with bf16-rounded products; same arguments and result as
    ``feature_ae_step`` (all float64)."""
    p = {k: params[k].detach().to(torch.float64).clone().requires_grad_() for k in FEATURE_AE_PARAMS}
    x = x.to(torch.float64)
    mm = Bf16MatMul.apply
    h1 = torch.relu(mm(x, p["fc1.weight"].t()) + p["fc1.bias"])
    z = torch.relu(mm(h1, p["fc2.weight"].t()) + p["fc2.bias"])
    h3 = torch.relu(mm(z, p["fc3.weight"].t()) + p["fc3.bias"])
    recon = torch.relu(mm(h3, p["fc4.weight"].t()) + p["fc4.bias"])
    sq = (recon - x)**2
    if regularizer_type == "noregu":
        loss = sq.sum()
    elif regularizer_type == "LTMG":
        loss = (1 - regu_strength) * sq.sum()
        if ltmg is not None:
            loss = loss + regu_strength * (sq * ltmg.to(torch.float64)).sum()
    else:
        raise ValueError(f"unsupported regularizer_type {regularizer_type!r}")
    grads = torch.autograd.grad(loss, [p[k] for k in FEATURE_AE_PARAMS])
    return {"loss": loss.detach(), "z": z.detach(), "recon": recon.detach(), "grads": dict(zip(FEATURE_AE_PARAMS, grads))}
