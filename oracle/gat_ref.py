"""fp64 restatement of the GAT kernels (dance_b200/csrc/gat.cu) on an explicit edge list, as test arbiter.

Edges are numbered as in the target-indexed CSR the kernels read: edge p goes from ``src[p]`` (CSR column) to
``trg[p]`` (CSR row), so an α of shape [nnz, nheads] lines up with the kernels' ``alpha``.  Everything is plain torch
and differentiable; backward references come from ``torch.autograd`` on these functions.

* global shift: the max over every (edge, head) score, as ``port.gat_layer`` (scgnn2.py:1076) — NOT detached unless
  ``detach_max``; its gradient only matters where Σ exp(score - max) is comparable to the 1e-16 of the denominator;
* per-target shift: the detached per-target max of ``pyg_lite.softmax`` (PyG).
"""
from __future__ import annotations

import torch
import torch.nn.functional as Fn

EPS = 1e-16


def csr_edges(rowptr, colidx):
    """(src, trg) int64 edge lists of a target-indexed CSR, in CSR order."""
    rowptr = torch.as_tensor(rowptr).long().cpu()
    deg = rowptr[1:] - rowptr[:-1]
    trg = torch.repeat_interleave(torch.arange(len(deg)), deg)
    return torch.as_tensor(colidx).long().cpu(), trg


def scores(H, a_src, a_trg, nheads):
    """s_src[n, h] = <H[n, h, :], a_src[h, :]>, s_trg likewise."""
    n = H.shape[0]
    Hv = H.reshape(n, nheads, -1)
    return (Hv * a_src.reshape(nheads, -1)).sum(-1), (Hv * a_trg.reshape(nheads, -1)).sum(-1)


def score_act(x, act, slope=0.2):
    return Fn.leaky_relu(x, slope) if act == "leakyrelu" else torch.sigmoid(x)


def edge_softmax(e, trg, n, shift, detach_max=False):
    """α [E, nh] of the edge scores e [E, nh] over the in-edges of each target."""
    if e.shape[0] == 0:
        return e.clone()
    idx = trg.to(e.device).view(-1, 1).expand_as(e)
    if shift == "global":
        c = e.max()
        ex = (e - (c.detach() if detach_max else c)).exp()
    else:
        m = torch.full((n, e.shape[1]), float("-inf"), dtype=e.dtype, device=e.device)
        m = m.scatter_reduce(0, idx, e.detach(), reduce="amax", include_self=True)
        ex = (e - m.gather(0, idx)).exp()
    den = torch.zeros((n, e.shape[1]), dtype=e.dtype, device=e.device).scatter_add(0, idx, ex)
    return ex / (den.gather(0, idx) + EPS)


def aggregate(H, s_src, s_trg, src, trg, nheads, act="leakyrelu", slope=0.2, shift="global", detach_max=False, H2=None):
    """(out [n, W], α [E, nh]) — and out2 = Σ α H2[u] when a tied second layer H2 is given (STAGATE's conv3)."""
    n = H.shape[0]
    src, trg = src.to(H.device), trg.to(H.device)
    e = score_act(s_src.index_select(0, src) + s_trg.index_select(0, trg), act, slope)
    alpha = edge_softmax(e, trg, n, shift, detach_max)

    def msg(X):
        lifted = X.reshape(n, nheads, -1).index_select(0, src) * alpha.unsqueeze(-1)
        return torch.zeros((n, ) + lifted.shape[1:], dtype=X.dtype, device=X.device).index_add(0, trg, lifted).reshape(n, -1)

    if H2 is None:
        return msg(H), alpha
    return msg(H), alpha, msg(H2)


def combine(agg, skip, bias, nheads, concat, act=None):
    """skip + concat | head-mean + bias + activation (port.gat_layer's tail, scgnn2.py:1189-1215)."""
    n = agg.shape[0]
    out = agg.reshape(n, nheads, -1)
    if skip is not None:
        out = out + skip.reshape(n, nheads, -1)
    out = out.reshape(n, -1) if concat else out.mean(dim=1)
    if bias is not None:
        out = out + bias
    return {None: lambda x: x, "none": lambda x: x, "relu": torch.relu, "elu": Fn.elu, "tanh": torch.tanh}[act](out)
