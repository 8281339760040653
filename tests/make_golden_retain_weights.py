"""Generate ``tests/golden/scgnn_retain_weights.npz`` from the REFERENCE's own functions (through ``oracle.ref_loader``) for
``graph_AE_retain_weights``.  TEST INFRASTRUCTURE, like ``oracle/make_golden.py``: it needs the reference sources and is run by
hand from the repository root:

    python tests/make_golden_retain_weights.py

Two cases of 300 cells, prefixed ``k5.`` and ``k15.``.  The k = 5 embedding holds one pair of identical cells, so one row lists
itself among its ranks 1..k (the diagonal feature2adj drops) and one weight is 1e16.  Per case:

* the kNN lists of ``calculateKNNgraphDistanceMatrixStatsSingleThread`` (scgnn2.py:675-689) with their fp64 distances;
* feature2adj(retain_weights=True), lines 659-670, with the nodes inserted in cell order first: W (``adj``), Â of
  ``preprocess_graph`` (fp32), the labels adj_train + I (fp32), ΣW, pos_weight and norm;
* the reference's own ``feature2adj(X, k, True)`` output (``pi_adj``) and its node order π (first appearance in edgeList);
* k = 15 only: one training step of ``Graph_AE`` on each branch — GCN with ``gae_loss_function`` and recorded ε, GAT (dropout 0)
  with ``loss_function`` — initial weights, loss, gradients and the weights after one Adam step (lr 1e-2); and the Cluster-AE
  weights of ``graph_celltype_regu_handler(adj, labels)`` for fixed cluster labels.
"""
from __future__ import annotations

import sys
import warnings
from pathlib import Path

import networkx as nx
import numpy as np
import scipy.sparse as sp
import torch
from scipy.spatial import distance

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from oracle import port, ref_loader  # noqa: E402

OUT = ROOT / "tests" / "golden"


def _csr(out, key, m, dtype):
    m = sp.csr_matrix(m)
    m.sort_indices()
    out[key + ".indptr"], out[key + ".indices"], out[key + ".data"] = m.indptr.astype(np.int32), m.indices.astype(np.int32), m.data.astype(dtype)


def _case(ref, tag, X, k, out, train):
    n = X.shape[0]
    edge_list = ref.calculateKNNgraphDistanceMatrixStatsSingleThread(X, k=k)
    knn_idx = np.array([e[1] for e in edge_list], dtype=np.int32).reshape(n, k)
    knn_dist = np.empty((n, k))
    for i in range(n):          # the same cdist row the reference ranks (scgnn2.py:682-683)
        knn_dist[i] = distance.cdist(X[i].reshape(1, -1), X, "euclidean")[0, knn_idx[i]]
    assert np.array_equal(1 / (knn_dist.reshape(-1) + 1e-16), np.array([e[2] for e in edge_list]))
    out[f"{tag}.X"], out[f"{tag}.k"], out[f"{tag}.knn_idx"], out[f"{tag}.knn_dist"] = X, np.int64(k), knn_idx, knn_dist

    # feature2adj lines 659-670 with the nodes in cell order
    G = nx.DiGraph()
    G.add_nodes_from(range(n))
    G.add_weighted_edges_from(edge_list)
    adj = nx.adjacency_matrix(G).astype(np.float64)
    adj_train = adj - sp.dia_matrix((adj.diagonal()[np.newaxis, :], [0]), shape=adj.shape)
    adj_train.eliminate_zeros()
    an = ref.preprocess_graph(adj_train).coalesce()
    ahat = sp.csr_matrix((an.values().numpy(), an.indices().numpy()), shape=tuple(an.shape))
    labels = np.asarray((adj_train + sp.eye(n)).todense(), dtype=np.float32)     # adj_label → FloatTensor (scgnn2.py:557, 572)
    sum_w = adj_train.sum()
    pos_weight = float(n * n - sum_w) / sum_w
    norm = n * n / float((n * n - sum_w) * 2)
    _csr(out, f"{tag}.W", adj, np.float64)
    _csr(out, f"{tag}.ahat", ahat, np.float32)
    _csr(out, f"{tag}.labels", sp.csr_matrix(labels), np.float32)
    out[f"{tag}.sum_w"], out[f"{tag}.pos_weight"], out[f"{tag}.norm"] = np.float64(sum_w), np.float64(pos_weight), np.float64(norm)
    out[f"{tag}.n_self"] = np.int64(int(np.sum(knn_idx == np.arange(n)[:, None])))

    # the reference's own call: nodes in first-appearance order π
    pi_adj, _, _ = ref.feature2adj(X, k, True)
    Gp = nx.DiGraph()
    Gp.add_weighted_edges_from(edge_list)
    out[f"{tag}.pi"] = np.array(list(Gp.nodes()), dtype=np.int64)
    _csr(out, f"{tag}.pi_adj", pi_adj, np.float64)
    if not train:
        return

    # GCN branch, one step (scgnn2.py:555-595, 603-615)
    torch.manual_seed(3)
    model = ref.Graph_AE(X.shape[1], 16, 0, 2, 64)
    x = torch.from_numpy(X)
    w = {k_: v.detach().clone().numpy() for k_, v in model.state_dict().items() if k_.startswith("gc")}
    out.update({f"{tag}.gcn.w1": w["gc1.weight"], f"{tag}.gcn.w2": w["gc2.weight"], f"{tag}.gcn.w3": w["gc3.weight"]})
    model.train()
    opt = torch.optim.Adam(model.parameters(), lr=1e-2)
    torch.manual_seed(5)
    eps = torch.randn(n, 16)
    torch.manual_seed(5)            # reparameterize draws randn_like(std) first → the same ε
    opt.zero_grad()
    z, info, recon = model(x, an.float(), use_GAT=False)
    assert torch.allclose(z, eps * torch.exp(info[1]) + info[0])
    loss = ref.gae_loss_function(preds=recon, labels=torch.from_numpy(labels), mu=info[0], logvar=info[1], n_nodes=n, norm=norm,
                                 pos_weight=pos_weight)
    loss.backward()
    out.update({f"{tag}.gcn.eps": eps.numpy(), f"{tag}.gcn.z": z.detach().numpy(), f"{tag}.gcn.loss": np.float64(loss.item())})
    for i in (1, 2, 3):
        out[f"{tag}.gcn.g_w{i}"] = getattr(model, f"gc{i}").weight.grad.numpy().copy()
    opt.step()
    for i in (1, 2, 3):
        out[f"{tag}.gcn.w{i}_after"] = getattr(model, f"gc{i}").weight.detach().numpy().copy()

    # GAT branch, dropout 0, one step (scgnn2.py:560-563, 581, 618-619)
    torch.manual_seed(13)
    model = ref.Graph_AE(X.shape[1], 16, 0, 2, 64)
    with torch.no_grad():
        for layer in model.gat.gat_net:
            layer.bias.normal_(0, 0.1)           # non-zero biases (the reference initialises them to zero)
    out.update({f"{tag}.gat.init.{k_}": v.detach().clone().numpy() for k_, v in model.state_dict().items() if k_.startswith("gat.")})
    edge_index = torch.from_numpy(np.array(ref.edgeList2edgeIndex(edge_list)).T.astype(np.int64))
    model.train()
    opt = torch.optim.Adam(model.parameters(), lr=1e-2)
    opt.zero_grad()
    embed, _, recon = model(x, edge_index, use_GAT=True)
    loss = ref.loss_function(preds=recon, labels=torch.from_numpy(labels))
    loss.backward()
    out.update({f"{tag}.gat.z": embed.detach().numpy(), f"{tag}.gat.loss": np.float64(loss.item())})
    for k_, p in model.named_parameters():
        if k_.startswith("gat.") and p.grad is not None:
            out[f"{tag}.gat.grad.{k_}"] = p.grad.numpy().copy()
    opt.step()
    out.update({f"{tag}.gat.after.{k_}": v.detach().numpy().copy() for k_, v in model.state_dict().items() if k_.startswith("gat.")})

    # Cluster-AE weights of graph_celltype_regu_handler on the weighted adj (scgnn2.py:716-730, 844-846)
    lab = np.random.default_rng(7).integers(0, 5, n)
    adjdense, _ = ref.graph_celltype_regu_handler(sp.csr_matrix(adj), lab.tolist())   # networkx now returns a csr_array
    adjdense = np.asarray(adjdense)
    out[f"{tag}.regu.labels"] = lab.astype(np.int32)
    out[f"{tag}.regu.w"] = np.array([adjdense[lab == lab[j], j].sum() for j in range(n)])


def main():
    ref = ref_loader.scgnn2()
    out = {}
    X5 = port.synthetic_embedding(300, d=16, n_clusters=4, seed=31)
    X5[201] = X5[200]                    # one pair of identical cells: a self-listed neighbour and a zero distance
    X15 = port.synthetic_embedding(300, d=16, n_clusters=4, seed=32)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        _case(ref, "k5", X5, 5, out, train=False)
        _case(ref, "k15", X15, 15, out, train=True)
    assert out["k5.n_self"] >= 1 and out["k15.n_self"] == 0
    np.savez_compressed(OUT / "scgnn_retain_weights.npz", **out)
    print("scgnn_retain_weights.npz", (OUT / "scgnn_retain_weights.npz").stat().st_size)


if __name__ == "__main__":
    main()
