"""Restatement of scGNN's GATLayer / Graph_AE.encode_gat in train() mode, with GATLayer's dropout given as explicit masks.

``oracle.port.gat_layer`` restates the layer with dropout 0; this module adds the three ``nn.Dropout`` sites of
GATLayer.forward (scgnn2.py:999-1031), each as a pre-drawn SCALED mask (0 or 1 / (1 - p)) that multiplies the tensor:

* ``input`` [N, FIN] on the layer input x; the projection AND the skip connection read the dropped x';
* ``proj`` [N, NH·F] on the projection x' Wᵀ; the scores and the messages read it, the skip projection does not;
* ``attn`` [E, NH] on the attention coefficients after the neighbourhood softmax, in ``edge_index`` order.

A missing site (or ``masks=None``) is no dropout, and then the result is ``oracle.port.gat_layer``'s bit for bit (every
operation is the same; a mask of ones multiplies exactly).  Plain torch, differentiable in any dtype.
"""
from __future__ import annotations

import torch
import torch.nn.functional as Fn


def scaled_mask(keep, p: float, dtype=torch.float64):
    """keep (bool / 0-1) → keep / (1 - p); p = 1 gives zeros."""
    keep = torch.as_tensor(keep).to(dtype)
    return keep * (1.0 / (1.0 - p)) if p < 1 else keep * 0


def gat_layer(x, edge_index, proj_w, skip_w, a_src, a_trg, bias, concat: bool, act=None, masks=None):
    """GATLayer.forward (scgnn2.py:989-1051, helpers :1057-1215) with the dropout masks ``masks`` = {site: scaled mask}."""
    masks = masks or {}
    nh, F_ = a_src.shape[1], a_src.shape[2]
    n = x.shape[0]
    src, trg = edge_index[0], edge_index[1]
    if "input" in masks:
        x = x * masks["input"]
    proj = (x @ proj_w.t()).view(-1, nh, F_)
    if "proj" in masks:
        proj = proj * masks["proj"].reshape(-1, nh, F_)
    s_src = (proj * a_src).sum(-1)
    s_trg = (proj * a_trg).sum(-1)
    scores = Fn.leaky_relu(s_src.index_select(0, src) + s_trg.index_select(0, trg), 0.2)
    ex = (scores - scores.max()).exp()
    denom = torch.zeros(n, nh, dtype=ex.dtype).index_add_(0, trg, ex)
    att = (ex / (denom.index_select(0, trg) + 1e-16)).unsqueeze(-1)
    if "attn" in masks:
        att = att * masks["attn"].reshape(-1, nh, 1)
    out = torch.zeros(n, nh, F_, dtype=x.dtype).index_add_(0, trg, proj.index_select(0, src) * att)
    if out.shape[-1] == x.shape[-1]:
        out = out + x.unsqueeze(1)          # identity skip: the raw (dropped) input on every head, skip_proj unused
    else:
        out = out + (x @ skip_w.t()).view(-1, nh, F_)
    out = out.view(-1, nh * F_) if concat else out.mean(dim=1)
    if bias is not None:
        out = out + bias
    return act(out) if act is not None else out


def graph_ae_gat_forward(x, edge_index, sd, masks=None):
    """Graph_AE.encode_gat (scgnn2.py:385-386) from a reference state_dict; ``masks`` = [layer-0 masks, layer-1 masks]."""
    h = x
    for l, (concat, act) in enumerate(((True, Fn.elu), (False, None))):
        pre = f"gat.gat_net.{l}."
        h = gat_layer(h, edge_index, sd[pre + "linear_proj.weight"], sd[pre + "skip_proj.weight"], sd[pre + "scoring_fn_source"],
                      sd[pre + "scoring_fn_target"], sd[pre + "bias"], concat, act, None if masks is None else masks[l])
    return h


def fixture_masks(gg, tag: str, dtype=torch.float64):
    """The scaled masks stored by make_golden_gat_dropout.py for configuration ``tag``: [{site: mask}] per layer."""
    p = float(gg[f"{tag}.p"])
    return [{site: scaled_mask(torch.from_numpy(gg[f"{tag}.mask.{l}.{site}"]), p, dtype) for site in ("input", "proj", "attn")}
            for l in range(2)]
