"""Generate ``tests/golden/graph_ae_gat_dropout.npz`` by running the REFERENCE's own Graph_AE(use_GAT=True) in train() mode
with GATLayer's dropout replaced by pre-drawn masks.  TEST INFRASTRUCTURE, like ``oracle/make_golden.py``: it needs the
reference sources (through ``oracle.ref_loader``) and is run by hand from the repository root:

    python tests/make_golden_gat_dropout.py

Each GATLayer owns one ``nn.Dropout`` that its forward calls three times (scgnn2.py:1005 input, :1010 projection, :1029
attention); ``_MaskDropout`` replaces it and multiplies by the next stored mask in that order.  Two configurations on the
``knn_graph.npz`` cells and edges (i → its k neighbours, as graph_AE_handler builds edge_index):

* ``proj``: Graph_AE(16, 16, 0.3, 2, 64) — both layers use skip_proj;
* ``ident``: Graph_AE(16, 32, 0.3, 2, 16) — FIN == FOUT in both layers, the identity skip (scgnn2.py:1167-1171).

Stored per configuration: the keep masks, the initial weights, the embedding, the plain-BCE loss, every parameter gradient
(none for an unused skip_proj) and the weights after one Adam step (lr 1e-2).
"""
from __future__ import annotations

import sys
import warnings
from pathlib import Path

import numpy as np
import scipy.sparse as sp
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from oracle import ref_loader  # noqa: E402

OUT = ROOT / "tests" / "golden"
P = 0.3
CONFIGS = (("proj", (16, 0.3, 2, 64), 21), ("ident", (32, 0.3, 2, 16), 22))


class _MaskDropout(torch.nn.Module):
    """Applies the given scaled masks in call order (input, projection, attention), one per call."""

    def __init__(self, masks):
        super().__init__()
        self.masks = list(masks)

    def forward(self, t):
        m = self.masks.pop(0)
        return t * m.reshape(t.shape).to(t.dtype)


def _config(ref, tag, args, seed, X, edge_index, labels, out):
    torch.manual_seed(seed)
    model = ref.Graph_AE(X.shape[1], *args)
    with torch.no_grad():
        for layer in model.gat.gat_net:
            layer.bias.normal_(0, 0.1)           # non-zero biases (the reference initialises them to zero)
    out[f"{tag}.p"] = np.float64(P)
    out.update({f"{tag}.init.{k}": v.detach().clone().numpy() for k, v in model.state_dict().items() if k.startswith("gat.")})
    rng = np.random.default_rng(seed)
    n, E = X.shape[0], edge_index.shape[1]
    for l, layer in enumerate(model.gat.gat_net):
        nh, F_ = layer.num_of_heads, layer.num_out_features
        shapes = {"input": (n, layer.linear_proj.in_features), "proj": (n, nh * F_), "attn": (E, nh)}
        keeps = {site: rng.random(shape) >= P for site, shape in shapes.items()}
        for site, keep in keeps.items():
            out[f"{tag}.mask.{l}.{site}"] = keep
        layer.dropout = _MaskDropout(torch.from_numpy(keeps[s].astype(np.float32)) * (1.0 / (1.0 - P)) for s in ("input", "proj", "attn"))
    model.train()
    opt = torch.optim.Adam(model.parameters(), lr=1e-2)
    opt.zero_grad()
    embed, _, recon = model(torch.from_numpy(X), edge_index, use_GAT=True)
    loss = ref.loss_function(preds=recon, labels=labels)
    loss.backward()
    assert all(not layer.dropout.masks for layer in model.gat.gat_net), "every mask is used exactly once"
    out[f"{tag}.z"] = embed.detach().numpy()
    out[f"{tag}.loss"] = np.float64(loss.item())
    for k, p in model.named_parameters():
        if k.startswith("gat.") and p.grad is not None:
            out[f"{tag}.grad.{k}"] = p.grad.numpy().copy()
    opt.step()
    out.update({f"{tag}.after.{k}": v.detach().numpy().copy() for k, v in model.state_dict().items() if k.startswith("gat.")})


def main():
    ref = ref_loader.scgnn2()
    g = np.load(OUT / "knn_graph.npz")
    X = g["X"]
    n, k = g["knn_idx"].shape
    edge_index = torch.from_numpy(np.stack([np.repeat(np.arange(n), k), g["knn_idx"].reshape(-1)]).astype(np.int64))
    adj = sp.csr_matrix((np.ones(len(g["adj_indices"])), g["adj_indices"], g["adj_indptr"]), shape=(n, n))
    labels = torch.from_numpy((adj + sp.eye(n)).toarray()).float()
    out = {}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for tag, args, seed in CONFIGS:
            _config(ref, tag, args, seed, X, edge_index, labels, out)
    np.savez_compressed(OUT / "graph_ae_gat_dropout.npz", **out)
    print("graph_ae_gat_dropout.npz", (OUT / "graph_ae_gat_dropout.npz").stat().st_size)


if __name__ == "__main__":
    main()
