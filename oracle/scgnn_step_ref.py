"""fp64 restatement of one training step of each scGNN engine (dance_b200/engine.py), as test arbiter.

Plain torch, no engine or ``ops`` code; it runs on whatever device its inputs live on (CUDA in the GPU tests, the CPU
elsewhere) and casts everything to float64.  Gradients come from ``torch.autograd``.

* Feature-AE (Feature_AE + loss_function_graph, scgnn2.py:352-370, 1298-1315): fc1…fc4 with ReLU after every layer,
  loss ``noregu`` = Σ (r − x)², ``LTMG`` = (1 − s)·Σ (r − x)² + s·Σ (r − x)²·T, where ``ltmg=None`` stands for the all-zero
  T of the reference driver, i.e. the weight (1 − s).
* Graph-AE, GCN branch (Graph_AE + GraphConvolution + gae_loss_function, scgnn2.py:396-412, 499-501, 603-615):
  hidden1 = relu(Â x W1), mu = Â hidden1 W2, logvar = Â hidden1 W3, z = mu + eps·exp(logvar), loss = norm × mean over all
  n² logits z zᵀ of the pos-weighted BCE, plus the KLD term.  The n² decoder term is never materialised: its value and its
  gradient with respect to z come from the row-chunked closed form :func:`gae_reference_rows` and are injected into the
  autograd graph at z.
"""
from __future__ import annotations

from typing import Callable, Dict, Optional, Tuple

import torch
import torch.nn.functional as F

FEATURE_AE_PARAMS = ("fc1.weight", "fc1.bias", "fc2.weight", "fc2.bias", "fc3.weight", "fc3.bias", "fc4.weight", "fc4.bias")


def gae_reference_rows(z, rowptr, colidx, norm, pw, rows, chunk=512):
    """fp64 closed form of gae_loss_function (scgnn2.py:603-612) restricted to `rows` × all columns, evaluated on z's device
    with torch in row chunks: returns (Σ over those rows of the per-logit cost · norm / n², the gradient rows).  With labels y
    (pattern of the CSR, unit values) and pos_weight = y·pw:  cost = y·pw·softplus(−x) + (1−y)·softplus(x);  ∂/∂z_i = 2·Σ_j c_ij z_j
    with c = σ(x) off the pattern and −pw·σ(−x) on it (labels symmetric)."""
    zd = z.double()
    n = zd.shape[0]
    rp = rowptr.long()
    loss = 0.0
    out = torch.empty(len(rows), zd.shape[1], dtype=torch.float64, device=z.device)
    for a in range(0, len(rows), chunk):
        r = rows[a:a + chunk]
        x = zd[r] @ zd.t()
        c = torch.sigmoid(x)
        cost = F.softplus(x)
        # label pattern of these rows
        cnt = rp[r + 1] - rp[r]
        loc = torch.repeat_interleave(torch.arange(len(r), device=z.device), cnt)
        start = torch.repeat_interleave(rp[r], cnt)
        within = torch.arange(int(cnt.sum()), device=z.device) - torch.repeat_interleave(torch.cumsum(cnt, 0) - cnt, cnt)
        cols = colidx.long()[start + within]
        xe = x[loc, cols]
        cost[loc, cols] = pw * F.softplus(-xe)
        c[loc, cols] = -pw * torch.sigmoid(-xe)
        loss += float(cost.sum())
        out[a:a + chunk] = 2.0 * (c @ zd)
    return norm * loss / (float(n) * n), out * (norm / (float(n) * n))


def _leaves(params: Dict[str, torch.Tensor], names):
    return {k: params[k].detach().to(torch.float64).clone().requires_grad_() for k in names}


def feature_ae_step(x: torch.Tensor, params: Dict[str, torch.Tensor], regularizer_type: str = "LTMG", regu_strength: float = 0.9,
                    ltmg: Optional[torch.Tensor] = None) -> dict:
    """Forward, loss and backward of one Feature-AE mini-batch ``x`` [B, dim] from the weights ``params`` (keys fc1.weight …
    fc4.bias, nn.Linear layout).  Returns {"loss", "z", "recon", "grads": {name: ∂loss/∂param}}, all float64."""
    p = _leaves(params, FEATURE_AE_PARAMS)
    x = x.to(torch.float64)
    h1 = torch.relu(x @ p["fc1.weight"].t() + p["fc1.bias"])
    z = torch.relu(h1 @ p["fc2.weight"].t() + p["fc2.bias"])
    h3 = torch.relu(z @ p["fc3.weight"].t() + p["fc3.bias"])
    recon = torch.relu(h3 @ p["fc4.weight"].t() + p["fc4.bias"])
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


def graph_ae_step(x: torch.Tensor, adj_rowptr, adj_colidx, adj_vals, labels_rowptr, labels_colidx, norm: float, pos_weight: float,
                  weights: Dict[str, torch.Tensor], eps: Optional[torch.Tensor],
                  decoder: Optional[Callable[[torch.Tensor], Tuple[float, torch.Tensor]]] = None) -> dict:
    """Forward, loss and backward of one Graph-AE (GCN) epoch on the normalised adjacency Â (CSR, n × n) and the label pattern
    A + I (CSR, unit values), from ``weights`` gc1.weight [dim, 32], gc2.weight / gc3.weight [32, emb] (GraphConvolution layout).
    ``eps=None`` is eval mode (z = mu).  ``decoder(z)`` → (loss, dz), float64, replaces the unit-label closed form
    :func:`gae_reference_rows` (then the label arguments are not read): real-valued labels.  Returns {"loss", "z", "mu",
    "logvar", "dz", "dmu", "dlogvar", "grads": {name: …}}, all float64; dmu / dlogvar are the total loss gradients (decoder through
    z plus KLD)."""
    names = ("gc1.weight", "gc2.weight", "gc3.weight")
    w = _leaves(weights, names)
    n = x.shape[0]
    dev = x.device
    rp = adj_rowptr.long().to(dev)
    rows = torch.repeat_interleave(torch.arange(n, device=dev), rp[1:] - rp[:-1])
    A = torch.sparse_coo_tensor(torch.stack([rows, adj_colidx.long().to(dev)]), adj_vals.to(device=dev, dtype=torch.float64), (n, n),
                                check_invariants=True)
    x = x.to(torch.float64)
    hidden1 = torch.relu(torch.sparse.mm(A, x @ w["gc1.weight"]))
    mu = torch.sparse.mm(A, hidden1 @ w["gc2.weight"])
    logvar = torch.sparse.mm(A, hidden1 @ w["gc3.weight"])
    z = mu if eps is None else eps.to(torch.float64) * torch.exp(logvar) + mu
    kld = -0.5 / n * torch.mean(torch.sum(1 + 2 * logvar - mu.pow(2) - logvar.exp().pow(2), 1))
    for t in (mu, logvar, z):
        t.retain_grad()
    if decoder is None:
        dec, dz = gae_reference_rows(z.detach(), labels_rowptr.to(dev), labels_colidx.to(dev), norm, pos_weight,
                                     torch.arange(n, device=dev))
    else:
        dec, dz = decoder(z.detach())
        dz = torch.as_tensor(dz, dtype=torch.float64, device=dev)
    torch.autograd.backward([z, kld], [dz, torch.ones_like(kld)])
    return {"loss": dec + kld.item(), "z": z.detach(), "mu": mu.detach(), "logvar": logvar.detach(), "dz": dz, "dmu": mu.grad,
            "dlogvar": logvar.grad, "grads": {k: w[k].grad for k in names}}
