"""Float64 sequential restatement of Leiden (Traag, Waltman & van Eck 2019) with the quality of leidenalg's
RBConfigurationVertexPartition, the reference csrc/leiden.cu is tested against.

For a symmetric weighted graph A (both directions stored), W = Σᵢⱼ Aᵢⱼ, kᵢ = Σⱼ Aᵢⱼ, K_c = Σ_{i∈c} kᵢ:
    Q = Σ_c (e_c − γ·K_c²/W),  e_c = Σ_{i,j∈c} Aᵢⱼ,  reported as Q / W.
Local moving visits vertices in index order and moves each to the community (a neighbouring one or an empty one) with the
largest positive gain, until a pass moves nothing; refinement merges well-connected singletons greedily, in index order, into
the well-connected sub-community of their community with the largest non-negative gain; aggregation collapses the refined
communities and starts from the unrefined ones; iterations repeat until one changes nothing."""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

EPS = 1e-13


def quality(A, labels, gamma: float) -> float:
    """Q / W of ``labels`` on the symmetric CSR ``A``."""
    A = sp.csr_matrix(A, dtype=np.float64)
    labels = np.asarray(labels)
    W = A.sum()
    if W == 0:
        return 0.0
    coo = A.tocoo()
    e_in = coo.data[labels[coo.row] == labels[coo.col]].sum()
    K = np.bincount(labels, weights=np.asarray(A.sum(axis=1)).ravel())
    return float(e_in / W - gamma * (K * K).sum() / (W * W))


def canonical(labels) -> np.ndarray:
    """0..K-1 by decreasing community size, ties by the smallest member."""
    labels = np.asarray(labels)
    uniq, inv, cnt = np.unique(labels, return_inverse=True, return_counts=True)
    first = np.full(len(uniq), len(labels))
    np.minimum.at(first, inv, np.arange(len(labels)))
    order = np.lexsort((first, -cnt))
    rank = np.empty(len(uniq), dtype=np.int64)
    rank[order] = np.arange(len(uniq))
    return rank[inv]


def _rows(A):
    return [(A.indices[A.indptr[v]:A.indptr[v + 1]], A.data[A.indptr[v]:A.indptr[v + 1]]) for v in range(A.shape[0])]


def _move_nodes(rows, k, comm, g, W):
    n = len(rows)
    K = np.bincount(comm, weights=k, minlength=n)
    size = np.bincount(comm, minlength=n)
    moved_any = True
    while moved_any:
        moved_any = False
        for v in range(n):
            a = comm[v]
            wc = {}
            for u, w in zip(*rows[v]):
                if u != v:
                    wc[comm[u]] = wc.get(comm[u], 0.0) + w
            own = wc.get(a, 0.0)
            Ka = K[a] - k[v]
            best, best_c = EPS * W, -1
            for c in sorted(wc):
                if c == a:
                    continue
                gain = wc[c] - own - g * k[v] * (K[c] - Ka)
                if gain > best:
                    best, best_c = gain, c
            if size[a] > 1:
                gain = -own + g * k[v] * Ka
                if gain > best:
                    best, best_c = gain, int(np.flatnonzero(size == 0)[0])
            if best_c >= 0:
                K[a] -= k[v]
                size[a] -= 1
                K[best_c] += k[v]
                size[best_c] += 1
                comm[v] = best_c
                moved_any = True
    return comm


def _refine(rows, k, comm, g):
    n = len(rows)
    K = np.bincount(comm, weights=k, minlength=n)
    ref = np.arange(n)
    Kt = k.copy()
    size = np.ones(n, dtype=np.int64)
    wout = np.zeros(n)       # w(T, S∖T) of each sub-community T
    wS = np.zeros(n)
    for v in range(n):
        for u, w in zip(*rows[v]):
            if u != v and comm[u] == comm[v]:
                wout[v] += w
                wS[v] += w
    for v in range(n):
        if size[ref[v]] != 1 or wS[v] < g * k[v] * (K[comm[v]] - k[v]):
            continue
        wt = {}
        for u, w in zip(*rows[v]):
            if u != v and comm[u] == comm[v]:
                wt[ref[u]] = wt.get(ref[u], 0.0) + w
        KS = K[comm[v]]
        best, best_t = -1.0, -1
        for t in sorted(wt):
            if wout[t] < g * Kt[t] * (KS - Kt[t]):
                continue
            gain = wt[t] - g * k[v] * Kt[t]
            if gain >= 0 and gain > best:
                best, best_t = gain, t
        if best_t < 0:
            continue
        # v joins best_t: the edges between them become internal
        wout[best_t] += wout[v] - 2 * wt[best_t]
        Kt[best_t] += k[v]
        size[best_t] += 1
        size[v] = 0
        ref[v] = best_t
    return ref


def leiden_ref(A, gamma: float, max_iterations: int = -1, max_cap: int = 100):
    """Canonical labels of Leiden on the symmetric CSR ``A``, and the number of iterations run."""
    A0 = sp.csr_matrix(A, dtype=np.float64)
    A0.sort_indices()
    n0 = A0.shape[0]
    W = A0.sum()
    labels = np.arange(n0)
    if W == 0:
        return labels, 0
    g = gamma / W
    cap = max_iterations if max_iterations > 0 else max_cap
    it = 0
    for it in range(1, cap + 1):
        A, comm, node = A0, labels.copy(), np.arange(n0)
        while True:
            rows = _rows(A)
            k = np.asarray(A.sum(axis=1)).ravel()
            comm = _move_nodes(rows, k, comm, g, W)
            ref = _refine(rows, k, comm, g)
            _, rid = np.unique(ref, return_inverse=True)
            n2 = rid.max() + 1
            if n2 >= A.shape[0]:
                break
            _, cid = np.unique(comm, return_inverse=True)
            nxt = np.zeros(n2, dtype=np.int64)
            nxt[rid] = cid
            P = sp.csr_matrix((np.ones(A.shape[0]), (np.arange(A.shape[0]), rid)), shape=(A.shape[0], n2))
            A = sp.csr_matrix(P.T @ A @ P)
            A.sort_indices()
            node = rid[node]
            comm = nxt
        new = canonical(comm[node])
        if np.array_equal(new, labels):
            break
        labels = new
    return labels, it
