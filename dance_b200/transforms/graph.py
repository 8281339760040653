"""Graph-building transforms on the GPU kernels.

``CellFeatureGraph`` keeps the reference's constructor, ``out`` channel (``uns["CellFeatureGraph"]``), node
ordering (genes first), edge order, weights and node data names (reference
dance/transforms/graph/cell_feature_graph.py:12-79, incl. the ``cell_id``/``feat_id`` naming quirk :56-59).
``SpaGCNGraph`` / ``SpaGCNGraph2D`` (dance/transforms/graph/spatial_graph.py:13-76) produce the dense spot-to-spot
euclidean distance matrices with the pairwise-distance kernel (``utils/matrix.py:164-180`` in the reference)."""
from __future__ import annotations

from typing import Optional

import numpy as np
import scipy.sparse as sp
import torch

from .. import ops
from ..graph import GraphLite
from .base import BaseTransform
from .cell_feature import WeightedFeaturePCA


class CellFeatureGraph(BaseTransform):

    def __init__(self, cell_feature_channel: str, gene_feature_channel: Optional[str] = None, *, mod: Optional[str] = None,
                 normalize_edges: bool = True, **kwargs):
        super().__init__(**kwargs)
        self.cell_feature_channel = cell_feature_channel
        self.gene_feature_channel = gene_feature_channel or cell_feature_channel
        self.mod = mod
        self.normalize_edges = normalize_edges

    def __call__(self, data):
        feat = data.get_feature(return_type="default", mod=self.mod)
        if sp.issparse(feat):
            feat = feat.toarray()
        num_cells, num_feats = feat.shape
        X = torch.as_tensor(np.ascontiguousarray(feat, dtype=np.float32)).cuda()
        src, dst, w, nnz = ops.cellgene_graph(X, self.normalize_edges)
        self.logger.info(f"Number of nonzero entries: {nnz:,}")
        self.logger.info(f"Nonzero rate = {nnz / num_cells / num_feats:.1%}")
        g = GraphLite(src.cpu(), dst.cpu(), num_cells + num_feats)      # stored on the host: the dataset cache pickles it
        g.edata["weight"] = w.cpu()
        g.ndata["cell_id"] = torch.concat((torch.arange(num_feats, dtype=torch.int32), -torch.ones(num_cells, dtype=torch.int32)))
        g.ndata["feat_id"] = torch.concat((-torch.ones(num_feats, dtype=torch.int32), torch.arange(num_cells, dtype=torch.int32)))
        gene_feature = data.get_feature(return_type="torch", channel=self.gene_feature_channel, mod=self.mod, channel_type="varm")
        cell_feature = data.get_feature(return_type="torch", channel=self.cell_feature_channel, mod=self.mod, channel_type="obsm")
        g.ndata["features"] = torch.vstack((gene_feature, cell_feature))
        data.data.uns[self.out] = g
        return data


class PCACellFeatureGraph(BaseTransform):
    """WeightedFeaturePCA followed by CellFeatureGraph (cell_feature_graph.py:83-112)."""

    _DISPLAY_ATTRS = ("n_components", "split_name")

    def __init__(self, n_components: int = 400, split_name: Optional[str] = None, *, normalize_edges: bool = True,
                 feat_norm_mode: Optional[str] = None, feat_norm_axis: int = 0, mod: Optional[str] = None, log_level="WARNING"):
        super().__init__(log_level=log_level)
        self.n_components, self.split_name, self.normalize_edges = n_components, split_name, normalize_edges
        self.feat_norm_mode, self.feat_norm_axis, self.mod = feat_norm_mode, feat_norm_axis, mod

    def __call__(self, data):
        WeightedFeaturePCA(self.n_components, self.split_name, feat_norm_mode=self.feat_norm_mode, feat_norm_axis=self.feat_norm_axis,
                           log_level=self.log_level)(data)
        CellFeatureGraph(cell_feature_channel="WeightedFeaturePCA", mod=self.mod, normalize_edges=self.normalize_edges,
                         log_level=self.log_level)(data)
        return data


def _pairwise_distance_host(x: np.ndarray) -> np.ndarray:
    """``pairwise_distance(x.astype(float32), dist_func_id=0)`` on the device, returned as the fp32 host matrix the
    reference stores in ``obsp``."""
    X = torch.as_tensor(np.ascontiguousarray(x, dtype=np.float32)).cuda()
    return ops.pairwise_l2_dense(X).cpu().numpy()


class SpaGCNGraph(BaseTransform):
    """Distance over (x, y, z) where z is the histology colour summary of each spot's pixel window
    (spatial_graph.py:13-62 ≡ spagcn.py:81-116).  The window means are a few thousand small uint8 slices of a host
    image and stay on the host, as in the reference; the N×N distance matrix is the device kernel."""

    _DISPLAY_ATTRS = ("alpha", "beta")

    def __init__(self, alpha, beta, *, channels=("spatial", "spatial_pixel", "image"), channel_types=("obsm", "obsm", "uns"), **kwargs):
        super().__init__(**kwargs)
        self.alpha, self.beta = alpha, beta
        self.channels, self.channel_types = channels, channel_types

    def __call__(self, data):
        xy = data.get_feature(return_type="numpy", channel=self.channels[0], channel_type=self.channel_types[0])
        xy_pixel = data.get_feature(return_type="numpy", channel=self.channels[1], channel_type=self.channel_types[1])
        img = data.get_feature(return_type="numpy", channel=self.channels[2], channel_type=self.channel_types[2])
        # window means of the three colour channels around every spot through a summed-area table (one pass over the image
        # instead of one slice per spot); integer images sum exactly, so the means equal np.mean over the clipped window
        half = round(self.beta / 2)
        img = np.asarray(img)
        if img.ndim == 2:
            img = img[:, :, None]
        H, Wd = img.shape[:2]
        sat = np.zeros((H + 1, Wd + 1, img.shape[2]), dtype=np.float64)
        np.cumsum(np.cumsum(img, axis=0, dtype=np.float64), axis=1, out=sat[1:, 1:])
        px = np.asarray(xy_pixel)
        r0, c0 = np.clip(px[:, 0] - half, 0, None).astype(np.int64), np.clip(px[:, 1] - half, 0, None).astype(np.int64)
        r1, c1 = np.minimum(H, px[:, 0] + half + 1).astype(np.int64), np.minimum(Wd, px[:, 1] + half + 1).astype(np.int64)
        area = ((r1 - r0) * (c1 - c0)).astype(np.float64)[:, None]
        colour = (sat[r1, c1] - sat[r0, c1] - sat[r1, c0] + sat[r0, c0]) / area
        colour_var = colour.var(axis=0)
        self.logger.info(f"colour-channel variances: {colour_var}")
        # third coordinate: variance-weighted grey value, standardised, scaled to alpha × the larger spatial spread
        depth = colour @ (colour_var / colour_var.sum())
        depth = (depth - depth.mean()) / depth.std() * (xy.std(axis=0).max() * self.alpha)
        xyz = np.column_stack([xy, depth]).astype(np.float32)
        self.logger.info(f"coordinate variances (x, y, z): {xyz.var(axis=0)}")
        data.data.obsp[self.out] = _pairwise_distance_host(xyz)
        return data


class SpaGCNGraph2D(BaseTransform):
    """Distance over the pixel coordinates only (spatial_graph.py:66-76)."""

    def __init__(self, *, channel: str = "spatial_pixel", **kwargs):
        super().__init__(**kwargs)
        self.channel = channel

    def __call__(self, data):
        x = data.get_feature(channel=self.channel, channel_type="obsm", return_type="numpy")
        data.data.obsp[self.out] = _pairwise_distance_host(x.astype(np.float32))
        return data


class StagateGraph(BaseTransform):
    """STAGATE spatial graph (spatial_graph.py:113-151): ``radius`` → all spot pairs within ``radius`` (self included,
    sklearn ``radius_neighbors_graph``), ``knn`` → the ``n_neighbors`` nearest spots of every spot, the spot itself being
    the first of them (sklearn ``kneighbors_graph`` on its own training data).  Unit weights, scipy CSR in ``obsp``.
    Exact ties at the k-th distance are broken by the lower spot index (sklearn's tree order is unspecified there)."""

    _MODELS = ("radius", "knn")
    _DISPLAY_ATTRS = ("model_name", "radius", "n_neighbors")

    def __init__(self, model_name: str = "radius", *, radius: float = 1, n_neighbors: int = 5, channel: str = "spatial_pixel",
                 channel_type: str = "obsm", **kwargs):
        super().__init__(**kwargs)
        if not isinstance(model_name, str) or (model_name.lower() not in self._MODELS):
            raise ValueError(f"Unknown model {model_name!r}, available options are {self._MODELS}")
        self.model_name, self.radius, self.n_neighbors = model_name, radius, n_neighbors
        self.channel, self.channel_type = channel, channel_type

    def __call__(self, data):
        xy = np.asarray(data.get_feature(return_type="numpy", channel=self.channel, channel_type=self.channel_type))
        n = xy.shape[0]
        if self.model_name.lower() == "radius":
            A = ops.radius_graph(torch.as_tensor(np.ascontiguousarray(xy, dtype=np.float64)).cuda(), float(self.radius))
            indptr, indices = A.rowptr.cpu().numpy(), A.colidx.cpu().numpy()
        else:
            k = int(self.n_neighbors)
            idx, _ = ops.knn(torch.as_tensor(np.ascontiguousarray(xy, dtype=np.float32)).cuda(), k, include_rank0=True, return_dist=False)
            indices = np.sort(idx.cpu().numpy(), axis=1).reshape(-1)
            indptr = np.arange(0, n * k + 1, k, dtype=np.int32)
        adj = sp.csr_matrix((np.ones(len(indices), dtype=np.float64), indices, indptr), shape=(n, n))
        data.data.obsp[self.out] = adj
        return data


def _average_ranks(X: torch.Tensor, chunk: int = 64) -> torch.Tensor:
    """Column-wise ranks with ties averaged (scipy.stats.rankdata(method="average") along axis 0, as used by
    ``scipy.stats.spearmanr``): a value whose equals occupy sorted positions lb … ub-1 gets rank (lb + ub + 1) / 2.
    Sort / searchsorted are library plumbing (like the CUB sorts elsewhere); ranks ≤ 2²⁴ are exact in fp32."""
    n, g = X.shape
    out = torch.empty((n, g), dtype=torch.float32, device=X.device)
    for c0 in range(0, g, chunk):
        xt = X[:, c0:c0 + chunk].t().contiguous()
        sv = torch.sort(xt, dim=1).values
        lb = torch.searchsorted(sv, xt, right=False)
        ub = torch.searchsorted(sv, xt, right=True)
        out[:, c0:c0 + chunk] = ((lb + ub + 1).to(torch.float32) * 0.5).t()
    return out


def _median_np(v: torch.Tensor, dim=None):
    """numpy.median semantics (mean of the two middle order statistics for an even count)."""
    if dim is None:
        sv = torch.sort(v.flatten()).values
        m = sv.numel()
        return (sv[(m - 1) // 2] + sv[m // 2]) * 0.5
    sv = torch.sort(v, dim=dim).values
    m = v.shape[dim]
    return (sv.select(dim, (m - 1) // 2) + sv.select(dim, m // 2)).unsqueeze(dim) * 0.5


def _rbf_from_gram(gram: torch.Tensor, denom_scale: float = 1.0, scale_mode: str = "med_dist") -> torch.Tensor:
    """feature_feature_graph.py:53-57 + utils/matrix.py:70-97 from the Gram matrix ``featᵀ·feat``: euclidean distances between
    gene columns (negative round-off clipped), then ``exp(-d / denom)`` with the reference's three scaling modes."""
    nv = torch.diagonal(gram).unsqueeze(0)
    dist = torch.sqrt(torch.clamp(nv + nv.t() - 2 * gram, min=0))
    if scale_mode == "med_dist":
        denom = _median_np(dist) * denom_scale
    elif scale_mode == "ind_med_dist":
        denom = _median_np(dist, dim=1) * denom_scale
    elif scale_mode == "scale":
        denom = denom_scale
    else:
        raise ValueError(f"Uknwon rbf scaling mode {scale_mode}")
    return torch.exp(-dist / denom)


class FeatureFeatureGraph(BaseTransform):
    """Gene–gene similarity graph (feature_feature_graph.py:14-87): similarity of the gene columns — ``pearson`` (np.corrcoef),
    ``spearman`` (Pearson of the tie-averaged ranks, scipy.stats.spearmanr) or ``rbf`` (Gaussian kernel of the euclidean
    distance, utils/matrix.py:70-97) — entries with |score| below ``threshold`` dropped, edges in row-major order, unit weights
    optionally normalised like ``dgl.nn.EdgeWeightNorm("both")``.  Result: ``uns[out]`` = graph with ``ndata["feat"] = Xᵀ`` and
    ``edata["weight"]``.  The correlations run through the fp64 Gram kernel; the rbf Gram through the tensor-core GEMM (the
    reference uses an fp32 BLAS product there, so entries within round-off of the threshold may differ)."""

    _DISPLAY_ATTRS = ("threshold", "positive_only", "normalize_edges", "score_func", "score_func_kwargs")

    def __init__(self, threshold: float = 0.3, *, positive_only: bool = False, normalize_edges: bool = True, score_func="pearson",
                 score_func_kwargs=None, **kwargs):
        super().__init__(**kwargs)
        self.threshold, self.positive_only, self.normalize_edges = threshold, positive_only, normalize_edges
        self.score_func, self.score_func_kwargs = score_func, score_func_kwargs or {}

    def __call__(self, data):
        feat = data.get_feature(return_type="numpy")
        if self.score_func not in ("pearson", "spearman", "rbf"):
            raise ValueError(f"Unknown similarity score function {self.score_func!r}, supported options are: 'pearson', 'spearman', 'rbf'")
        X = torch.as_tensor(np.ascontiguousarray(feat, dtype=np.float32)).cuda()
        if self.score_func == "pearson":
            adj = ops.pearson_corr(X)
        elif self.score_func == "spearman":
            adj = ops.pearson_corr(_average_ranks(X))
        else:
            adj = _rbf_from_gram(ops.gemm(X, X, transA=True), **self.score_func_kwargs).contiguous()
        src, dst, w, _ = ops.threshold_graph(adj, self.threshold, self.positive_only, self.normalize_edges)
        g = GraphLite(src.cpu(), dst.cpu(), adj.shape[0])
        g.ndata["feat"] = torch.from_numpy(np.ascontiguousarray(feat.astype(np.float32).T))
        g.edata["weight"] = w.cpu()
        data.data.uns[self.out] = g
        return data


class NeighborGraph(BaseTransform):
    """kNN connectivity graph of the cells (neighbor_graph.py:9-57): ``scanpy.pp.neighbors(use_rep=channel, n_neighbors,
    method="umap", metric="euclidean")`` → ``obsp[out]`` = the symmetric fuzzy-simplicial-set connectivities (scipy CSR,
    fp32).  The neighbour search is the exact device kNN at every size (scanpy switches to approximate pynndescent above
    4096 cells; the exact graph is what that approximates)."""

    _DISPLAY_ATTRS = ("n_neighbors", "n_pcs", "knn", "random_state", "method", "metric")

    def __init__(self, n_neighbors: int = 15, *, n_pcs: Optional[int] = None, knn: bool = True, random_state: int = 0,
                 method: Optional[str] = "umap", metric: str = "euclidean", channel: Optional[str] = "CellPCA", **kwargs):
        super().__init__(**kwargs)
        self.n_neighbors, self.n_pcs, self.knn, self.random_state = n_neighbors, n_pcs, knn, random_state
        self.method, self.metric, self.channel = method, metric, channel

    def __call__(self, data):
        if self.method != "umap" or self.metric != "euclidean" or not self.knn:
            raise NotImplementedError("only method='umap', metric='euclidean', knn=True (the defaults) are built")
        rep = data.get_feature(return_type="numpy", channel=self.channel, channel_type="obsm" if self.channel else "X")
        if self.n_pcs is not None:
            rep = rep[:, :self.n_pcs]
        X = torch.as_tensor(np.ascontiguousarray(rep, dtype=np.float32)).cuda()
        idx, dist = ops.knn(X, int(self.n_neighbors), include_rank0=True)
        Cn = ops.umap_connectivities(idx, dist.float())
        n = X.shape[0]
        adj = sp.csr_matrix((Cn.vals.cpu().numpy(), Cn.colidx.cpu().numpy(), Cn.rowptr.cpu().numpy()), shape=(n, n))
        data.data.obsp[self.out] = adj
        return data
