"""Leiden community detection on the device (``csrc/leiden.cu``) and the neighbour graph it runs on: scanpy's
``pp.neighbors(method="umap")`` followed by ``tl.leiden``, which SpaGCN's ``init="louvain"`` calls (spagcn.py:481-492).

Label parity with leidenalg is unpinned: leidenalg's refinement draws its merges at random (θ = 0.01), this one takes the best
merge, and leidenalg / igraph are not available to compare against.  What is pinned is the quality both optimise."""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple

import torch

from . import ops


class LeidenResult(NamedTuple):
    labels: torch.Tensor      # int32 [n] on the device, 0..K-1 by decreasing community size (ties: smallest member)
    n_communities: int
    quality: float            # Q / W = networkx modularity(resolution=γ) of the labels
    iterations: int
    levels: int               # most aggregation levels in one iteration


def neighbor_graph(X: torch.Tensor, n_neighbors: int) -> ops.CSR:
    """The UMAP fuzzy connectivities of the exact euclidean kNN graph of the rows of ``X`` (``scanpy.pp.neighbors(method="umap",
    metric="euclidean")``; the cell itself counts among its ``n_neighbors``): a symmetric device CSR."""
    idx, dist = ops.knn(X, int(n_neighbors), include_rank0=True)
    return ops.umap_connectivities(idx, dist.float())


def leiden(A: ops.CSR, resolution: float = 1.0, max_iterations: int = -1) -> LeidenResult:
    """Leiden on the symmetric CSR ``A`` (both directions stored, values None = unit weights) with the quality of
    ``leidenalg.RBConfigurationVertexPartition`` at ``resolution_parameter = resolution``.  ``max_iterations = -1`` iterates until
    an iteration changes nothing (scanpy's ``n_iterations=-1``).  Synchronises the stream."""
    n, nnz = A.shape[0], A.nnz
    rp = ops._arg(A.rowptr, "rowptr", torch.int32, (n + 1, ))
    ci = ops._arg(A.colidx, "colidx", torch.int32, (nnz, ), empty=rp)
    vals = ops._arg(A.vals, "vals", torch.float32, (nnz, ), optional=True, empty=rp)
    labels = torch.empty(n, dtype=torch.int32, device=A.rowptr.device)
    nbytes = ops.lib().b2_leiden_workspace_bytes(n, nnz)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=A.rowptr.device)
    n_comm, quality, info = C.c_int32(), C.c_double(), (C.c_int32 * 2)()
    ops._call("b2_leiden_f32", rp, ci, vals, n, nnz, float(resolution), int(max_iterations), ops._arg(labels, "labels", torch.int32, n),
              C.byref(n_comm), C.byref(quality), info, ops._arg(ws, "workspace", torch.uint8, nbytes), nbytes, ops._stream())
    return LeidenResult(labels, n_comm.value, quality.value, info[0], info[1])
