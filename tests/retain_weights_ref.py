"""numpy / torch restatement of scGNN's Graph-AE inputs and losses with ``graph_AE_retain_weights`` (test infrastructure).

* :func:`weighted_graph` — feature2adj(retain_weights=True) in cell order (scgnn2.py:659-670), preprocess_graph (:1191-1198), the
  label matrix and ΣW (:555-569), from the kNN lists: W[i, j] = 1/(d_ij + 1e-16), directed; adj_train = W without its diagonal;
  Â = ((adj_train + I)·Dm)ᵀ·Dm with Dm = diag(rowsum^-1/2), in fp64, then fp32.
* :func:`decoder_loss_grad` — the Graph-AE decoder loss and d loss / d z in fp64 for dense, real-valued labels: gae_loss_function
  (pos_weight = labels·pw, times norm) or loss_function (plain mean BCE).
* :func:`regu_weights` — the per-cell weights the Cluster-AE takes from graph_celltype_regu_handler(adj) (scgnn2.py:716-730):
  adjdense[i, j] = colsum_j / rowsum_i, summed over i in j's cluster; diagonal entries of adj are not counted.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp
import torch


def weighted_adj(knn_idx: np.ndarray, knn_dist: np.ndarray) -> sp.csr_matrix:
    """W in cell order, fp64, sorted columns, any diagonal kept (the ``adj`` graph_AE_handler returns)."""
    n, k = knn_idx.shape
    w = 1.0 / (knn_dist.reshape(-1).astype(np.float64) + 1e-16)
    W = sp.csr_matrix((w, (np.repeat(np.arange(n), k), knn_idx.reshape(-1).astype(np.int64))), shape=(n, n))
    W.sort_indices()
    return W


def weighted_graph(knn_idx: np.ndarray, knn_dist: np.ndarray):
    """Returns (W, adj_train, Â fp32 CSR, labels fp32 CSR = adj_train + I, ΣW)."""
    W = weighted_adj(knn_idx, knn_dist)
    n = W.shape[0]
    adj_train = (W - sp.diags(W.diagonal())).tocsr()
    adj_train.eliminate_zeros()
    adj_train.sort_indices()
    plus_i = (adj_train + sp.eye(n)).tocsr()
    rowsum = np.asarray(plus_i.sum(1)).ravel()
    dm = sp.diags(np.power(rowsum, -0.5))
    ahat = plus_i.dot(dm).transpose().dot(dm).tocsr()
    ahat.sort_indices()
    ahat = sp.csr_matrix((ahat.data.astype(np.float32), ahat.indices, ahat.indptr), shape=ahat.shape)
    labels = sp.csr_matrix((plus_i.data.astype(np.float32), plus_i.indices, plus_i.indptr), shape=plus_i.shape)
    labels.sort_indices()
    return W, adj_train, ahat, labels, float(adj_train.sum())


def gae_constants(sum_w: float, n: int):
    """(pos_weight, norm) of graph_AE_handler (scgnn2.py:567-569) from ΣW."""
    return float(n * n - sum_w) / sum_w, n * n / float((n * n - sum_w) * 2)


def decoder_loss_grad(z, labels_dense, norm: float, pw: float, use_pos_weight: bool = True):
    """fp64 loss and dz of the matrix-free decoder with real-valued labels y (rows × all columns when z_rows is given)."""
    z = torch.as_tensor(z).double().detach().requires_grad_()
    y = torch.as_tensor(labels_dense).double()
    x = z @ z.t()
    if use_pos_weight:
        loss = norm * torch.nn.functional.binary_cross_entropy_with_logits(x, y, pos_weight=y * pw)
    else:
        loss = torch.nn.functional.binary_cross_entropy_with_logits(x, y)
    loss.backward()
    return loss.item(), z.grad.cpu().numpy()


def regu_weights(W: sp.spmatrix, cluster_labels) -> np.ndarray:
    lab = np.asarray(cluster_labels)
    A = (W - sp.diags(W.diagonal())).tocsr()
    rowsum = np.asarray(A.sum(1)).ravel()
    colsum = np.asarray(A.sum(0)).ravel()
    inv = np.where(rowsum != 0, 1.0 / np.where(rowsum != 0, rowsum, 1.0), 0.0)
    per_cluster = np.bincount(lab, weights=inv, minlength=lab.max() + 1)
    return (colsum * per_cluster[lab]).astype(np.float32)
