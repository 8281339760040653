"""Exact kNN beyond the candidate-list path (k + r0 + 8 > 64: batched tf32x3 estimate, radix select, fp64 refine), UMAP
connectivities at k > 64, and Leiden on the k = 300 graph: indices and fp64 distances bit-exact against a host fp64 brute force
(scipy cdist, stable argsort: ties by the smaller index)."""
import numpy as np
import pytest
import torch
from scipy.spatial.distance import cdist

pytestmark = pytest.mark.gpu


def _ref(X, k, include_rank0=False, rows=None):
    r0 = 0 if include_rank0 else 1
    rows = np.arange(X.shape[0]) if rows is None else np.asarray(rows)
    idx, dist = [], []
    for i0 in range(0, len(rows), 512):
        d = cdist(X[rows[i0:i0 + 512]], X, "euclidean")
        o = np.argsort(d, axis=1, kind="stable")[:, r0:r0 + k]
        idx.append(o)
        dist.append(np.take_along_axis(d, o, 1))
    return np.concatenate(idx), np.concatenate(dist)


def _check(X, k, include_rank0=False, q_begin=0, q_end=None, rows=None):
    from dance_b200 import ops
    n = X.shape[0]
    q_end = n if q_end is None else q_end
    idx, dist = ops.knn(torch.from_numpy(X).cuda(), k, include_rank0=include_rank0, q_begin=q_begin, q_end=q_end)
    idx, dist = idx.cpu().numpy(), dist.cpu().numpy()
    rows = np.arange(q_begin, q_end) if rows is None else np.asarray(rows)
    ref_idx, ref_dist = _ref(X, k, include_rank0, rows)
    assert np.array_equal(idx[rows - q_begin].astype(np.int64), ref_idx)
    assert np.array_equal(dist[rows - q_begin], ref_dist)
    return idx, dist


def _mixture(n, d, seed, clusters=6, sort=False):
    rng = np.random.default_rng(seed)
    lab = rng.integers(0, clusters, n)
    if sort:
        lab = np.sort(lab)                              # neighbours contiguous in index
    X = rng.normal(0, 3, (clusters, d))[lab] + rng.normal(size=(n, d))
    return X.astype(np.float32), lab


@pytest.mark.parametrize("include_rank0", [False, True])
@pytest.mark.parametrize("n,d,k", [(3000, 50, 57), (5000, 300, 300), (2500, 17, 1024), (301, 8, 300)])
def test_large_k_bit_exact(cuda, n, d, k, include_rank0):
    if k + (0 if include_rank0 else 1) > n:
        pytest.skip("k + r0 > n")
    X, _ = _mixture(n, d, seed=n + d)
    _check(X, k, include_rank0)


def test_large_k_query_range_sorted_clusters_odd_d(cuda):
    X, _ = _mixture(2000, 33, seed=3, sort=True)
    full, _ = _check(X, 100)
    part, _ = _check(X, 100, q_begin=150, q_end=1700)
    assert np.array_equal(part, full[150:1700])


@pytest.mark.parametrize("include_rank0", [False, True])
def test_large_k_identical_rows(cuda, include_rank0):
    """400 identical rows at k = 300: every query of the block ties with 399 others at distance 0, so the index breaks the ties
    and the collected candidates outnumber k."""
    rng = np.random.default_rng(7)
    X = rng.normal(size=(1000, 12)).astype(np.float32)
    same = rng.choice(1000, 400, replace=False)
    X[same] = X[same[0]]
    idx, dist = _check(X, 300, include_rank0)
    r0 = 0 if include_rank0 else 1
    block = np.sort(same)
    assert np.array_equal(idx[block[5]], block[r0:r0 + 300]) and not dist[block[5]].any()


def test_large_k_common_offset(cuda):
    """|x| ≈ 10³ with a spread of 10⁻²: the estimate's error bound exceeds every distance, so every reference is collected and
    each batch's candidates are sorted in several parts."""
    rng = np.random.default_rng(11)
    d = 50
    X = (1e3 / np.sqrt(d) + 1e-2 * rng.normal(size=(3000, d))).astype(np.float32)
    _check(X, 57)
    _check(X, 80, include_rank0=True, q_begin=1000, q_end=1400)


def test_large_k_split_batches(cuda):
    """24 000 references: the [bq, n] estimate block holds 22 369 query rows (2 GiB), so the queries run in two batches."""
    X, _ = _mixture(24000, 8, seed=13)
    rows = np.r_[0:100, 22300:22450, 23900:24000]
    _check(X, 60, rows=rows)


def test_workspace_covers_both_paths(cuda):
    from dance_b200 import ops
    lib = ops.lib()
    assert lib.b2_knn_workspace_bytes(5000, 300, 300, 5000) > 4 * 5000 * 5000
    assert lib.b2_knn_workspace_bytes(5000, 300, 56, 5000) >= lib.b2_knn_workspace_bytes(5000, 300, 55, 5000)


def _knn_host32(X, k):
    idx, dist = _ref(X, k, include_rank0=True)
    return idx.astype(np.int32), dist.astype(np.float32)


@pytest.mark.parametrize("n,d,k", [(500, 20, 65), (400, 30, 300)])
def test_umap_connectivities_large_k(cuda, n, d, k):
    """The warp-per-cell smooth_knn_dist against oracle/port.py's restatement, with test_gpu_neighbor_graph.py's tolerances."""
    from dance_b200 import ops
    from oracle import port
    X, _ = _mixture(n, d, seed=n + k, clusters=3)
    X[7] = X[3]
    idx, dist = _knn_host32(X, k)
    ref = port.umap_connectivities(idx, dist)
    out = ops.umap_connectivities(torch.from_numpy(idx).cuda(), torch.from_numpy(dist).cuda())
    assert np.array_equal(out.rowptr.cpu().numpy(), ref.indptr) and np.array_equal(out.colidx.cpu().numpy(), ref.indices)
    assert np.allclose(out.vals.cpu().numpy(), ref.data, rtol=2e-5, atol=1e-7)


def test_leiden_on_300nn_graph(cuda):
    """Leiden on the k = 300 UMAP graph of a separated 300-d mixture: its quality is the host fp64 recomputation and the planted
    clusters come back."""
    import scipy.sparse as sp
    from sklearn.metrics import adjusted_rand_score

    from dance_b200.leiden import leiden, neighbor_graph
    from leiden_ref import quality
    rng = np.random.default_rng(21)
    lab = np.repeat(np.arange(4), 500)
    X = (rng.normal(0, 4, (4, 300))[lab] + rng.normal(size=(2000, 300))).astype(np.float32)
    A = neighbor_graph(torch.from_numpy(X).cuda(), 300)
    res = leiden(A)
    labels = res.labels.cpu().numpy()
    q = quality(sp.csr_matrix(A.to_scipy(), dtype=np.float64), labels, 1.0)
    assert abs(res.quality - q) <= 1e-9 * abs(q)
    assert adjusted_rand_score(lab, labels) == 1.0
