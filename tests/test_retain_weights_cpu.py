"""graph_AE_retain_weights without a GPU: the fixture against the reference's own node order, the numpy restatement against the
fixture, and argument validation of the weighted graph builder and regulariser (rejected before any CUDA call, so stand-in pointers
are never dereferenced)."""
import numpy as np
import pytest
import scipy.sparse as sp

from retain_weights_ref import regu_weights, weighted_graph

INVALID = -1
P = 1 << 20          # a 16-byte aligned stand-in address
N = 1000


def _csr(g, key, dtype=None):
    data = g[key + ".data"]
    n = len(g[key + ".indptr"]) - 1
    return sp.csr_matrix((data if dtype is None else data.astype(dtype), g[key + ".indices"], g[key + ".indptr"]), shape=(n, n))


@pytest.mark.parametrize("tag", ["k5", "k15"])
def test_reference_node_order_is_one_relabelling(golden, tag):
    """The reference's own feature2adj(X, k, True) orders nodes by first appearance in edgeList (π): its adj is exactly the
    cell-order W relabelled by π, and nothing else."""
    g = golden("scgnn_retain_weights")
    W, pi_adj, pi = _csr(g, f"{tag}.W"), _csr(g, f"{tag}.pi_adj"), g[f"{tag}.pi"]
    assert sorted(pi.tolist()) == list(range(W.shape[0]))
    relabelled = W[pi][:, pi].tocsr()
    relabelled.sort_indices()
    assert np.array_equal(relabelled.indptr, pi_adj.indptr) and np.array_equal(relabelled.indices, pi_adj.indices)
    assert np.array_equal(relabelled.data, pi_adj.data)


@pytest.mark.parametrize("tag", ["k5", "k15"])
def test_restatement_reproduces_fixture(golden, tag):
    g = golden("scgnn_retain_weights")
    W, adj_train, ahat, labels, sum_w = weighted_graph(g[f"{tag}.knn_idx"], g[f"{tag}.knn_dist"])
    for mine, key in ((W, "W"), (ahat, "ahat"), (labels, "labels")):
        ref = _csr(g, f"{tag}.{key}")
        assert np.array_equal(mine.indptr, ref.indptr) and np.array_equal(mine.indices, ref.indices), key
        assert np.array_equal(mine.data, ref.data), key
    assert sum_w == float(g[f"{tag}.sum_w"])
    if tag == "k5":                                   # the self-listed slot is dropped from adj_train and comes back as + I
        assert int(g["k5.n_self"]) >= 1 and W.diagonal().max() == 1e16 and adj_train.diagonal().max() == 0


def test_regulariser_restatement_matches_reference(golden):
    g = golden("scgnn_retain_weights")
    w = regu_weights(_csr(g, "k15.W"), g["k15.regu.labels"])
    ref = g["k15.regu.w"]
    assert (ref == 0).any() and (ref > 0).any()          # cells nobody lists have colsum 0
    assert np.all(np.abs(w - ref) <= 1e-6 * np.abs(ref))


# ---- argument validation -------------------------------------------------------------------------------------------
def _build_args(**kw):
    import ctypes
    from dance_b200 import _lib
    nnz = ctypes.c_int64(0)
    a = dict(idx=P, dist=P, n=N, k=5, rowptr=P, colidx=P, y=P, norm_t=P, t_rowptr=P, t_colidx=P, t_y=P, norm=P, sum_w=P,
             cap=N * 6, nnz=ctypes.byref(nnz), ws=P, ws_bytes=_lib.lib().b2_knn_graph_weighted_workspace_bytes(N, 5))
    a.update(kw)
    return list(a.values()) + [None]


@pytest.mark.parametrize("kw", [{"idx": None}, {"dist": None}, {"y": None}, {"norm_t": None}, {"t_rowptr": None}, {"norm": None},
                                {"sum_w": None}, {"n": 0}, {"k": 0}, {"cap": N * 6 - 1}, {"ws": None}, {"ws_bytes": 1024}],
                         ids=lambda kw: "-".join(f"{k}={v}" for k, v in kw.items()))
def test_weighted_builder_validation(kw):
    from dance_b200 import _lib
    lib = _lib.lib()
    assert lib.b2_knn_graph_weighted_build(*_build_args(**kw)) == INVALID
    assert lib.b2_last_error().decode().startswith("b2_knn_graph_weighted_build:")


@pytest.mark.parametrize("arg", [0, 1, 2, 3, 6, 7])
def test_weighted_regu_validation(arg):
    from dance_b200 import _lib
    lib = _lib.lib()
    args = [P, P, P, P, N, 4, P, P, None]
    args[arg] = None
    assert lib.b2_graph_regu_weights_weighted_f32(*args) == INVALID
    assert lib.b2_graph_regu_weights_weighted_f32(P, P, P, P, N, 0, P, P, None) == INVALID
