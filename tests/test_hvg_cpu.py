"""highly_variable_genes(flavor="cell_ranger"): the float64 restatement (tests/hvg_ref.py) on a matrix worked out by hand, the
library's host half (transforms.pp.cell_ranger_hvg, from Σx and Σx²) against it, and the arguments that are not built."""
import numpy as np
import pytest

import hvg_ref

C = 0.6744897501960817


def _hand_matrix():
    """Two cells, 40 genes: gene j (1-based) reads j − 1 and j + 1, so mean = j, var (ddof 1) = 2 and dispersion = 2 / j."""
    j = np.arange(1, 41, dtype=np.float64)
    return np.stack([j - 1, j + 1]).astype(np.float32)


def test_restatement_by_hand():
    df = hvg_ref.cell_ranger(_hand_matrix(), n_top_genes=3)
    assert np.allclose(df["means"], np.arange(1, 41)) and np.allclose(df["dispersions"], 2 / np.arange(1, 41))
    # percentile 10 of 1..40 is 1 + 0.1·39 = 4.9: the first bin holds means 1..4, dispersions 2, 1, 2/3, 1/2;
    # median 5/6, |d − 5/6| = 7/6, 1/6, 1/6, 1/3 → MAD = (1/6 + 1/3)/2 / C = 1/(4C)
    dn = df["dispersions_norm"].to_numpy()
    assert np.allclose(dn[:4], (np.array([2, 1, 2 / 3, 1 / 2]) - 5 / 6) * 4 * C, rtol=1e-12)
    # percentile 15 is 1 + 0.15·39 = 6.85: the bin (4.9, 6.85] holds means 5 and 6, whose normalised dispersions are ±C
    assert np.allclose(dn[4:6], [C, -C], rtol=1e-12)
    # the largest is gene 1 (7/6·4C = 3.148…); the cut is the third largest, a +C of a two-gene bin (equal to C up to rounding)
    hv = df["highly_variable"].to_numpy()
    assert dn.max() == dn[0] and np.isclose(np.sort(dn[~np.isnan(dn)])[::-1][2], C)
    assert hv[0] and hv.sum() == 3 and np.array_equal(hv, dn >= np.sort(dn[~np.isnan(dn)])[::-1][2])


def test_host_half_matches_restatement():
    from dance_b200.transforms.pp import cell_ranger_hvg
    rng = np.random.default_rng(0)
    X = np.log1p(rng.poisson(rng.gamma(0.5, 2.0, 500), size=(300, 500))).astype(np.float32)
    X = X[:, X.sum(0) > 0]
    ref = hvg_ref.cell_ranger(X, 100)
    X64 = X.astype(np.float64)
    out = cell_ranger_hvg(X64.sum(0), (X64 * X64).sum(0), X.shape[0], 100)
    assert np.array_equal(out["highly_variable"], ref["highly_variable"].to_numpy())
    for key in ("means", "dispersions", "dispersions_norm"):
        assert np.allclose(out[key], ref[key].to_numpy(), rtol=1e-12, atol=0, equal_nan=True), key
    assert out["highly_variable"].sum() == 100


def test_duplicate_bin_edges_raise():
    from dance_b200.transforms.pp import cell_ranger_hvg
    with pytest.raises(ValueError, match="unique"):
        cell_ranger_hvg(np.ones(30), np.ones(30) * 2, 4, 5)


@pytest.mark.parametrize("kw", [dict(flavor="seurat", n_top_genes=5), dict(flavor="seurat_v3", n_top_genes=5),
                                dict(flavor="cell_ranger"), dict(flavor="cell_ranger", n_top_genes=5, batch_key="b"),
                                dict(flavor="cell_ranger", n_top_genes=5, layer="counts"),
                                dict(flavor="cell_ranger", n_top_genes=5, inplace=False)])
def test_unsupported_arguments_raise(kw):
    from dance_b200.data import AnnDataLite
    from dance_b200.transforms import AnnDataTransform
    from dance_b200.transforms.pp import highly_variable_genes
    with pytest.raises(NotImplementedError):
        highly_variable_genes(AnnDataLite(np.ones((4, 3), np.float32)), **kw)
    assert AnnDataTransform("scanpy.pp.highly_variable_genes").func is highly_variable_genes
