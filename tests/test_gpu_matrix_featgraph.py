"""utils.matrix.normalize (a20) and FeatureFeatureGraph (a15) on the device against the reference's own normalize()
(loaded through oracle.ref_loader when generating; here: the numpy restatement pinned by the reference's
tests/utils/test_matrix.py vectors in tests/test_oracle.py) and the numpy/dgl restatement of the graph builder."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mode", ["normalize", "standardize", "minmax", "l2"])
@pytest.mark.parametrize("axis", [0, 1])
@pytest.mark.parametrize("eps", [-1.0, 0.5])
def test_matrix_normalize_matches_reference_formula(cuda, mode, axis, eps):
    from dance_b200 import matrix
    from oracle import port
    rng = np.random.default_rng(3)
    X = rng.normal(size=(301, 77)).astype(np.float32) * 3 + 1
    X[:, 5] = 0          # zero column: sum / std / range / l2 all zero → denominator rule
    X[17, :] = 2.5       # constant row
    X[40, :] = 0
    ref = port.matrix_normalize(X, mode=mode, axis=axis, eps=eps)
    out = matrix.normalize(X, mode=mode, axis=axis, eps=eps)
    assert out.dtype == np.float32 and out.shape == X.shape
    assert np.allclose(out, ref, rtol=2e-5, atol=2e-6)
    out_t = matrix.normalize(torch.from_numpy(X).to(cuda), mode=mode, axis=axis, eps=eps)
    assert out_t.is_cuda and np.array_equal(out_t.cpu().numpy(), out)


def test_matrix_normalize_reference_known_answers(cuda):
    """The golden vectors of the reference's tests/utils/test_matrix.py:10-29."""
    from dance_b200 import matrix
    mat = np.array([[1, 1], [4, 4]], dtype=np.float32)
    f32 = lambda v: np.array(v, dtype=np.float32)       # the reference's vectors, rounded to the fp32 the kernels work in
    assert np.array_equal(matrix.normalize(mat, mode="normalize", axis=0), f32([[0.2, 0.2], [0.8, 0.8]]))
    assert np.array_equal(matrix.normalize(mat, mode="normalize", axis=1), f32([[0.5, 0.5], [0.5, 0.5]]))
    assert np.array_equal(matrix.normalize(mat, mode="standardize", axis=0), f32([[-1, -1], [1, 1]]))
    assert np.array_equal(matrix.normalize(mat, mode="standardize", axis=1), f32([[0, 0], [0, 0]]))
    assert np.array_equal(matrix.normalize(mat, mode="minmax", axis=0), f32([[0, 0], [1, 1]]))
    assert np.array_equal(matrix.normalize(mat, mode="minmax", axis=1), f32([[0, 0], [0, 0]]))
    assert np.allclose(matrix.normalize(mat, mode="l2", axis=0), mat / np.sqrt(17.0), rtol=1e-6)
    with pytest.raises(ValueError):
        matrix.normalize(mat, mode="normalize", eps=0.0)
    with pytest.raises(TypeError):
        matrix.normalize([[1.0]])


@pytest.mark.parametrize("positive_only,normalize_edges", [(False, True), (True, True), (False, False)])
def test_feature_feature_graph_matches_oracle(cuda, positive_only, normalize_edges):
    from dance_b200.data import AnnDataLite, Data
    from dance_b200.transforms import FeatureFeatureGraph
    from oracle import port
    rng = np.random.default_rng(9)
    n, g = 700, 150
    lat = rng.normal(size=(n, 6))
    X = (lat @ rng.normal(size=(6, g)) + rng.normal(size=(n, g)) * 2).astype(np.float32)
    X[:, 11] = 3.0       # zero-variance gene: NaN row/column, kept as edges by the reference
    src_r, dst_r, w_r, adj_r = port.feature_feature_graph(X, 0.3, positive_only, normalize_edges)
    data = Data(AnnDataLite(X))
    FeatureFeatureGraph(threshold=0.3, positive_only=positive_only, normalize_edges=normalize_edges)(data)
    gph = data.data.uns["FeatureFeatureGraph"]
    src, dst = gph.edges()
    assert np.array_equal(src.numpy(), src_r) and np.array_equal(dst.numpy(), dst_r)          # structure and edge order: bit-exact
    assert np.allclose(gph.edata["weight"].numpy(), w_r, rtol=1e-6, equal_nan=True)
    assert np.array_equal(gph.ndata["feat"].numpy(), X.T)
    assert gph.num_nodes() == g and len(src_r) > g


def test_pearson_corr_split_k_and_values(cuda):
    """Tall input (split over the cell axis with fp64 atomics) and a g that is not a multiple of the tile."""
    from dance_b200 import ops
    rng = np.random.default_rng(1)
    X = (rng.normal(size=(20000, 70)) + rng.normal(size=(20000, 1))).astype(np.float32)
    ref = np.corrcoef(X.T).astype(np.float32)
    out = ops.pearson_corr(torch.from_numpy(X).to(cuda)).cpu().numpy()
    assert np.abs(out - ref).max() <= 6e-8                 # at most one fp32 ulp of a value in [-1, 1]
    assert (out != ref).mean() < 1e-3
    assert np.array_equal(out, out.T)
    assert repr(__import__("dance_b200").transforms.FeatureFeatureGraph()) == \
        "FeatureFeatureGraph(threshold=0.3, positive_only=False, normalize_edges=True, score_func='pearson', score_func_kwargs={})"


@pytest.mark.parametrize("score_func,kw", [("spearman", None), ("rbf", {"scale_mode": "med_dist"}), ("rbf", {"scale_mode": "ind_med_dist", "denom_scale": 2.0})])
def test_feature_feature_graph_spearman_and_rbf(cuda, score_func, kw):
    from dance_b200.data import AnnDataLite, Data
    from dance_b200.transforms import FeatureFeatureGraph
    from oracle import port
    rng = np.random.default_rng(13)
    n, g = 600, 90
    lat = rng.gamma(2.0, 1.0, size=(n, 4))
    X = rng.poisson(lat @ rng.gamma(1.0, 0.7, size=(4, g))).astype(np.float32)
    thr = 0.3 if score_func == "spearman" else 0.5
    src_r, dst_r, w_r, adj_r = port.feature_feature_graph(X, thr, False, True, score_func=score_func, score_func_kwargs=kw)
    data = Data(AnnDataLite(X))
    FeatureFeatureGraph(threshold=thr, score_func=score_func, score_func_kwargs=kw)(data)
    gph = data.data.uns["FeatureFeatureGraph"]
    src, dst = gph.edges()
    if score_func == "spearman":      # fp64 correlations on both sides → the thresholded structure is exact
        assert np.array_equal(src.numpy(), src_r) and np.array_equal(dst.numpy(), dst_r)
        assert np.allclose(gph.edata["weight"].numpy(), w_r, rtol=1e-6)
    else:                             # fp32 Gram on both sides (BLAS vs tensor-core tf32x3): entries within round-off of the threshold may flip
        mine = set(zip(src.numpy().tolist(), dst.numpy().tolist()))
        ref = set(zip(src_r.tolist(), dst_r.tolist()))
        assert len(mine ^ ref) <= max(2, len(ref) // 500)
