"""fp64 restatement of one ``GraphSCI.train`` call (dance_b200/modules/graphsci.py), as test arbiter.

Plain torch, no module or ``ops`` code; it runs on whatever device its inputs live on (CUDA in the GPU tests, the CPU
elsewhere) and casts everything to float64.  Gradients come from ``torch.autograd``.  Semantics are those of the reference
GraphSCI (graphsci.py:37-122 model, :286-337 train, :420-483 get_loss):

* GNN over the gene graph: four GraphConv(norm="both") with structural degrees, Ân = D_in^-1/2 Aᵀ D_out^-1/2 (dense, G × G),
  node features [G, N cells].  ``z_adj_log_std`` comes from ``dec_mean`` too; z = mu + exp(log_std)·ε.
* AE over cells: ReLU(X·(z Wfᵀ) + b), two (Linear, BatchNorm, ReLU) blocks, three (Linear, BatchNorm) heads with Sigmoid /
  clamp(softplus) / clamp(exp).
* get_loss, including the rule that a NaN negative-binomial term counts as +inf.
* The validation loss comes from an eval-mode forward that uses the running statistics the training forward has just
  updated, exactly as ``train`` calls ``evaluate`` before ``backward``.

Dropout is given as keep-masks already scaled by 1/(1 − p), one per site of :data:`SITES`, in the order the reference draws
them.  A site missing from ``masks`` is not dropped.  When neither ``h2_mean`` nor ``h2_log_std`` is dropped the two
dec_mean calls see the same input, and log_std is the same node as mean.

Every product the module computes with ``ops.gemm`` goes through ``mm`` (``torch.matmul``, or a bf16-rounding autograd
function), forward and backward alike; the graph aggregations are plain float64 products.
"""
from __future__ import annotations

from typing import Callable, Dict, Optional

import torch
import torch.nn.functional as F

H1 = H2 = 256
HEADS = ("dec_pi", "dec_disp", "dec_mean")
# dropout sites in the order the reference draws them: GNN (graphsci.py:118-121), then AE (:81, buildNetwork :40)
SITES = ("feat", "h1", "h2_mean", "h2_log_std", "X", "enc.1", "enc.5", "dec_pi", "dec_disp", "dec_mean")
BN_KEYS = ("enc.2", "enc.6", "dec_pi.2", "dec_disp.2", "dec_mean.2")
PARAMS = ("aemodel.mul_layer.bias", "aemodel.mul_layer.fc_layer.weight", "aemodel.enc.1.weight", "aemodel.enc.1.bias",
          "aemodel.enc.2.weight", "aemodel.enc.2.bias", "aemodel.enc.5.weight", "aemodel.enc.5.bias", "aemodel.enc.6.weight",
          "aemodel.enc.6.bias") + tuple(f"aemodel.{h}.{k}" for h in HEADS for k in ("1.weight", "1.bias", "2.weight", "2.bias")) + (
              "gnnmodel.conv1.weight", "gnnmodel.conv1.bias", "gnnmodel.conv2.weight", "gnnmodel.conv2.bias",
              "gnnmodel.dec_mean.weight", "gnnmodel.dec_mean.bias")
LOSSES = ("loss_adj", "loss_exp", "log_lik", "kl", "train_loss")
BN_MOMENTUM, BN_EPS = 0.1, 1e-5


class GeneGraph:
    """Dense float64 views of the gene graph (edges u → v): Ân for the GraphConvs, the unit adjacency adj[u, v] = 1 that is
    the cross-entropy target, its class weights and norm (graphsci.py:242-244, :473-475)."""

    def __init__(self, src, dst, num_genes: int, device):
        G = int(num_genes)
        u = torch.as_tensor(src, device=device).long()
        v = torch.as_tensor(dst, device=device).long()
        A = torch.zeros(G, G, dtype=torch.float64, device=device)
        A.index_put_((u, v), torch.ones(u.numel(), dtype=torch.float64, device=device), accumulate=True)
        outdeg = A.sum(1).clamp(min=1)
        indeg = A.sum(0).clamp(min=1)
        self.An = (indeg.pow(-0.5)[:, None] * A.t() * outdeg.pow(-0.5)[None, :]).contiguous()
        self.adj = (A > 0).to(torch.float64)
        rs = self.adj.sum(1)
        self.pos_weight = (G * G - rs) / rs
        self.norm_adj = G * G / float((G * G - float(self.adj.sum())) * 2)
        self.G = G


def _drop(x, masks, site):
    m = None if masks is None else masks.get(site)
    return x if m is None else x * m.to(x)


def gnn_forward(p, feat, graph: GeneGraph, eps, masks=None, mm: Callable = torch.matmul):
    """GNNModel.forward (graphsci.py:117-123) with ``torch.normal(mean, std)`` = mean + std·ε.  Returns (z, log_std, mean)."""
    An = graph.An.to(feat.dtype)
    h1 = torch.tanh(An @ mm(_drop(feat, masks, "feat"), p["gnnmodel.conv1.weight"]) + p["gnnmodel.conv1.bias"])
    h2 = torch.relu(mm(An @ _drop(h1, masks, "h1"), p["gnnmodel.conv2.weight"]) + p["gnnmodel.conv2.bias"])
    Wm, bm = p["gnnmodel.dec_mean.weight"], p["gnnmodel.dec_mean.bias"]
    mu = mm(An @ _drop(h2, masks, "h2_mean"), Wm) + bm
    if masks is not None and (masks.get("h2_mean") is not None or masks.get("h2_log_std") is not None):
        ls = mm(An @ _drop(h2, masks, "h2_log_std"), Wm) + bm
    else:
        ls = mu
    return mu + torch.exp(ls) * eps.to(mu), ls, mu


def ae_forward(p, X, z, running, training: bool, masks=None, mm: Callable = torch.matmul):
    """AEModel.forward (graphsci.py:79-104).  ``running`` maps each BatchNorm key to (running_mean, running_var); in training
    mode they are updated in place (momentum 0.1, unbiased variance), as nn.BatchNorm1d does.  Returns (pi, disp, mean)."""

    def bn(x, key):
        rm, rv = running[key]
        return F.batch_norm(x, rm, rv, p[f"aemodel.{key}.weight"], p[f"aemodel.{key}.bias"], training, BN_MOMENTUM, BN_EPS)

    zf = mm(z, p["aemodel.mul_layer.fc_layer.weight"].t())
    h = torch.relu(mm(_drop(X, masks, "X"), zf) + p["aemodel.mul_layer.bias"])
    for lin, key in (("enc.1", "enc.2"), ("enc.5", "enc.6")):
        h = torch.relu(bn(mm(_drop(h, masks, lin), p[f"aemodel.{lin}.weight"].t()) + p[f"aemodel.{lin}.bias"], key))
    pre = {hd: bn(mm(_drop(h, masks, hd), p[f"aemodel.{hd}.1.weight"].t()) + p[f"aemodel.{hd}.1.bias"], f"{hd}.2") for hd in HEADS}
    pi = torch.sigmoid(pre["dec_pi"])
    disp = torch.clamp(F.softplus(pre["dec_disp"]), 1e-4, 1e4)
    mean = torch.clamp(torch.exp(pre["dec_mean"]), 1e-5, 1e6)
    return pi, disp, mean


def get_loss(Xraw, graph: GeneGraph, z, ls, mu, mean, disp, pi, sf, mask, le, la, ke, ka):
    """GraphSCI.get_loss (graphsci.py:420-503).  ``mask`` is a boolean [N, G].  Returns the dict of :data:`LOSSES` plus the
    four weighted terms (``terms``) whose combination is the loss."""
    N, G = Xraw.shape
    # F.cross_entropy with class-probability targets and class weights, mean over the G rows
    ce = -(graph.adj.to(z) * graph.pos_weight.to(z) * torch.log_softmax(z, dim=1)).sum() / z.shape[0]
    loss_adj = la * graph.norm_adj * ce
    eps = 1e-10
    z_exp = mean * sf.reshape(-1, 1)
    m = z_exp
    disp = torch.clamp(disp, max=1e6)
    t1 = torch.lgamma(disp + eps) + torch.lgamma(Xraw + 1) - torch.lgamma(Xraw + disp + eps)
    t2 = (disp + Xraw) * torch.log(1.0 + (m / (disp + eps))) + (Xraw * (torch.log(disp + eps) - torch.log(m + eps)))
    nb = t1 + t2
    nb = torch.where(torch.isnan(nb), torch.full_like(nb, float("inf")), nb)
    zero_nb = torch.pow(disp / (disp + m + eps), disp)
    zero_case = -torch.log(pi + ((1 - pi) * zero_nb) + eps)
    loss_exp = le * torch.where(Xraw < 1e-8, zero_case, nb)[mask].mean()
    kl_adj = (0.5 / N) * torch.mean(torch.sum(1 + 2 * ls - torch.square(mu) - torch.square(torch.exp(ls)), 1))
    kl_exp = 0.5 / G * ((z_exp - Xraw)**2)[mask].mean()
    kl = ka * kl_adj - ke * kl_exp
    log_lik = loss_exp + loss_adj
    out = dict(loss_adj=loss_adj, loss_exp=loss_exp, log_lik=log_lik, kl=kl, train_loss=log_lik - kl)
    out["terms"] = dict(exp=loss_exp, adj=loss_adj, kl_adj=-ka * kl_adj, kl_exp=ke * kl_exp)
    return out


def evaluate(params, running, X, Xraw, sf, graph: GeneGraph, mask, le, la, ke, ka, eps, feat=None, mm: Callable = torch.matmul,
             dtype=torch.float64):
    """GraphSCI.evaluate (graphsci.py:339-381): eval-mode forward (no dropout, BatchNorm on ``running``) and the loss over
    ``mask``.  Returns (loss, z_exp)."""
    p = {k: v.detach().to(dtype) for k, v in params.items()}
    run = {k: (m.detach().to(dtype), v.detach().to(dtype)) for k, (m, v) in running.items()}
    X, Xraw, sf = X.to(dtype), Xraw.to(dtype), sf.to(dtype)
    feat = X.t() if feat is None else feat.to(dtype)
    with torch.no_grad():
        z, ls, mu = gnn_forward(p, feat, graph, eps, None, mm)
        pi, disp, mean = ae_forward(p, X, z, run, False, None, mm)
        loss = get_loss(Xraw, graph, z, ls, mu, mean, disp, pi, sf, mask.bool(), le, la, ke, ka)["train_loss"]
    return loss, mean * sf.reshape(-1, 1)


def train_step(params: Dict[str, torch.Tensor], running: Dict[str, tuple], X, Xraw, sf, graph: GeneGraph, train_mask, valid_mask,
               le, la, ke, ka, eps_train, eps_eval, masks: Optional[Dict[str, torch.Tensor]] = None, feat=None,
               mm: Callable = torch.matmul, term_grads: bool = False, dtype=torch.float64) -> dict:
    """Forward, loss, validation loss and backward of one ``GraphSCI.train`` call from the weights ``params`` (keys of
    :data:`PARAMS`, the module's layouts) and the BatchNorm running statistics ``running`` ({key: (mean, var)}, left untouched).
    ``X`` is the (masked) training matrix, ``feat`` the GNN's node features (default ``X.t()``).

    Returns {"losses": {name: float} for :data:`LOSSES` and "valid_loss", "grads": {name: ∂train_loss/∂param},
    "running": {key: (mean, var)} after the training forward, "z_exp": the eval forward's reconstruction}, all float64.
    With ``term_grads`` also "term_grads": {term: {name: gradient of that weighted term alone}}.  ``dtype`` float32 gives
    the same step in plain float32 torch, a yardstick for how far any float32 evaluation lands from float64."""
    p = {k: params[k].detach().to(dtype).clone().requires_grad_() for k in PARAMS}
    run = {k: (m.detach().to(dtype).clone(), v.detach().to(dtype).clone()) for k, (m, v) in running.items()}
    X, Xraw, sf = X.to(dtype), Xraw.to(dtype), sf.to(dtype)
    feat = X.t() if feat is None else feat.to(dtype)
    z, ls, mu = gnn_forward(p, feat, graph, eps_train, masks, mm)
    pi, disp, mean = ae_forward(p, X, z, run, True, masks, mm)
    L = get_loss(Xraw, graph, z, ls, mu, mean, disp, pi, sf, train_mask.bool(), le, la, ke, ka)
    valid_loss, z_exp = evaluate(p, run, X, Xraw, sf, graph, valid_mask, le, la, ke, ka, eps_eval, feat, mm, dtype)
    leaves = [p[k] for k in PARAMS]
    out = {"losses": {k: float(L[k].detach()) for k in LOSSES}, "running": run, "z_exp": z_exp}
    out["losses"]["valid_loss"] = float(valid_loss)
    if term_grads:
        out["term_grads"] = {}
        for t, v in L["terms"].items():
            gs = torch.autograd.grad(v, leaves, retain_graph=True, allow_unused=True)
            out["term_grads"][t] = {k: (g if g is not None else torch.zeros_like(p[k])) for k, g in zip(PARAMS, gs)}
    out["grads"] = dict(zip(PARAMS, torch.autograd.grad(L["train_loss"], leaves)))
    return out
