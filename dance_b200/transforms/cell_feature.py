"""PCA feature transforms on the GPU (``ops.pca``: tensor-core GEMM for the Gram / covariance matrix + Jacobi
eigensolver).  Same constructors, output channels and ``repr`` as the reference
(dance/transforms/cell_feature.py: ``WeightedFeaturePCA`` :19-75, ``CellPCA`` :146-194; reprs pinned by the
reference's tests/transforms/test_basics.py:5-22).

sklearn's PCA picks a randomised solver for these shapes (seeded from the global numpy RNG, SURVEY App. A);
this implementation is the exact decomposition, so results agree with sklearn on explained variance and on
the leading subspace rather than entry by entry.
"""
from __future__ import annotations

from typing import Optional, Union

import numpy as np
import torch

from .. import ops
from .base import BaseTransform


def _to_cuda(a) -> torch.Tensor:
    if not torch.cuda.is_available():
        raise RuntimeError("dance_b200 needs a CUDA device (there is no CPU fallback)")
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32)).cuda()


class CellPCA(BaseTransform):
    _DISPLAY_ATTRS = ("n_components", )

    def __init__(self, n_components: Union[float, int] = 400, *, channel: Optional[str] = None, mod: Optional[str] = None,
                 save_info: bool = False, svd_solver: str = "auto", **kwargs):
        super().__init__(**kwargs)
        self.n_components, self.channel, self.save_info, self.svd_solver = n_components, channel, save_info, svd_solver

    def __call__(self, data):
        feat = data.get_feature(return_type="numpy", channel=self.channel)
        if self.n_components > min(feat.shape):
            self.logger.warning(f"n_components={self.n_components} must be between 0 and min(n_samples, n_features)={min(feat.shape)}")
            self.n_components = min(feat.shape)
        fitted = data.data.uns.get("pca") if hasattr(data.data, "uns") else None
        if fitted is not None:
            # a pre-fitted decomposition in uns["pca"] is applied, not re-fitted (reference cell_feature.py:176-178: pca.transform):
            # any object / mapping with `mean_` and `components_` (sklearn's PCA attributes) is accepted
            get = (lambda k: fitted[k]) if isinstance(fitted, dict) else (lambda k: getattr(fitted, k))
            mean = torch.as_tensor(np.asarray(get("mean_"), dtype=np.float32)).cuda()
            comp = torch.as_tensor(np.ascontiguousarray(get("components_"), dtype=np.float32)).cuda()
            centred = (_to_cuda(feat) - mean).contiguous()
            data.data.obsm[self.out] = ops.gemm(centred, comp, transB=True).cpu().numpy()
            return data
        res = ops.pca(_to_cuda(feat), _resolve_components(self.n_components, feat, self.logger))
        data.data.obsm[self.out] = res["scores"].cpu().numpy()
        if self.save_info:
            ev = res["explained_variance"].cpu().numpy()
            total_var = float(np.var(np.asarray(feat, dtype=np.float64), axis=0, ddof=1).sum())
            data.data.uns["pca_components"] = res["components"].cpu().numpy()
            data.data.uns["pca_mean"] = res["mean"].cpu().numpy()
            data.data.uns["pca_explained_variance"] = ev
            data.data.uns["pca_explained_variance_ratio"] = ev / total_var
        return data


def _resolve_components(n_components, feat, logger) -> int:
    """sklearn's ``PCA(n_components)`` rule: an int is the number of components; a float in (0, 1) the smallest number of
    components whose cumulative explained-variance ratio exceeds it (full decomposition, then truncated)."""
    if isinstance(n_components, (int, np.integer)) or float(n_components) >= 1:
        return int(n_components)
    frac = float(n_components)
    if not 0.0 < frac < 1.0:
        raise ValueError(f"n_components={n_components!r} must be a positive int or a float in (0, 1)")
    kmax = min(feat.shape)
    res = ops.pca(_to_cuda(feat), kmax)
    ev = res["explained_variance"].double().cpu().numpy()
    total = float(np.var(np.asarray(feat, dtype=np.float64), axis=0, ddof=1).sum())
    k = int(np.searchsorted(np.cumsum(ev) / total, frac, side="right") + 1)
    logger.info(f"n_components={frac} → {k} components")
    return min(k, kmax)


class WeightedFeaturePCA(BaseTransform):
    _DISPLAY_ATTRS = ("n_components", "split_name", "feat_norm_mode", "feat_norm_axis")

    def __init__(self, n_components: Union[float, int] = 400, split_name: Optional[str] = None, feat_norm_mode: Optional[str] = None,
                 feat_norm_axis: int = 0, save_info=False, **kwargs):
        super().__init__(**kwargs)
        self.n_components, self.split_name = n_components, split_name
        self.feat_norm_mode, self.feat_norm_axis, self.save_info = feat_norm_mode, feat_norm_axis, save_info

    def __call__(self, data):
        feat = data.get_x(self.split_name)                      # cells × genes
        feat_dev = None
        if self.feat_norm_mode is not None:      # normalize(feat, mode, axis) before the decomposition (cell_feature.py:51-54)
            feat_dev = ops.matrix_normalize(_to_cuda(feat), self.feat_norm_mode, self.feat_norm_axis % 2)
        if self.n_components > min(feat.shape):
            self.logger.warning(f"n_components={self.n_components} must be between 0 and min(n_samples, n_features)={min(feat.shape)}")
            self.n_components = min(feat.shape)
        k = _resolve_components(self.n_components, np.asarray(feat).T, self.logger)
        # genes × cells: genes are the PCA samples (cell_feature.py:61)
        Xt = _to_cuda(np.asarray(feat).T) if feat_dev is None else feat_dev.t().contiguous()
        res = ops.pca(Xt, k)
        gene_feat = res["scores"]                               # genes × components
        x = _to_cuda(data.get_x())
        # normalize(x, mode="normalize", axis=1) @ gene_feat   (cell_feature.py:66-67); zero row sums → divide by 1
        rs = x.sum(1, keepdim=True)
        rs[rs == 0] = 1
        cell_feat = ops.gemm((x / rs).contiguous(), gene_feat.contiguous())
        data.data.obsm[self.out] = cell_feat.cpu().numpy().astype(np.float32)
        data.data.varm[self.out] = gene_feat.cpu().numpy().astype(np.float32)
        if self.save_info:
            ev = res["explained_variance"].cpu().numpy()
            total_var = float(Xt.double().var(dim=0, unbiased=True).sum().item())
            data.data.uns["pca_components"] = res["components"].cpu().numpy()
            data.data.uns["pca_mean"] = res["mean"].cpu().numpy()
            data.data.uns["pca_explained_variance"] = ev
            data.data.uns["pca_explained_variance_ratio"] = ev / total_var
        return data
