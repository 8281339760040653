"""GPU counterparts of the ``scanpy.pp`` functions the pipelines call through ``AnnDataTransform`` (reference
examples/single_modality/imputation/scgnn2.py:190, examples/spatial/spatial_domain/spagcn.py pipeline,
transforms/normalize.py:563,618-620, graph-sc's preprocessing_pipeline graphsc.py:109-153).
Same call signature for the arguments the reference uses; they mutate ``adata.X`` in place.

The matrix makes one round trip host → HBM → host per call (the AnnData contract keeps X on the host);
``NormalizeTotalLog1P`` fuses both steps into a single kernel pass.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import scipy.sparse as sp
import torch

from .. import ops


def _to_device(adata):
    """Device copy of ``adata.X``: the stand-in AnnData keeps it resident between operators (data.AnnDataLite.device_X); a foreign
    AnnData is uploaded for this call."""
    if hasattr(adata, "device_X"):
        return adata.device_X()
    X = adata.X
    if sp.issparse(X):
        X = X.toarray()
    if not torch.cuda.is_available():
        raise RuntimeError("dance_b200 needs a CUDA device (there is no CPU fallback)")
    return torch.as_tensor(np.ascontiguousarray(X, dtype=np.float32)).cuda()


def _store(adata, Xd):
    if hasattr(adata, "set_device_X"):
        adata.set_device_X(Xd)          # stays in HBM; the host array is rebuilt on the next `.X` read
    else:
        adata.X = Xd.cpu().numpy()


def normalize_total(adata, target_sum: Optional[float] = None, exclude_highly_expressed: bool = False, max_fraction: float = 0.05,
                    key_added: Optional[str] = None, layer=None, layers=None, layer_norm=None, inplace: bool = True, copy: bool = False,
                    _log1p: bool = False, _base: Optional[float] = None):
    if layer is not None or layers is not None or layer_norm is not None or copy or not inplace:
        raise NotImplementedError("only in-place normalisation of adata.X is built")
    Xd = _to_device(adata)
    ops.normalize_total_log1p_(Xd, target_sum=target_sum, max_fraction=max_fraction if exclude_highly_expressed else 1.0,
                               normalize=True, log1p=_log1p, base=_base)
    _store(adata, Xd)


def log1p(adata, base: Optional[float] = None, copy: bool = False, chunked=None, chunk_size=None, layer=None, obsm=None):
    if copy or layer is not None or obsm is not None:
        raise NotImplementedError("only in-place log1p of adata.X is built")
    Xd = _to_device(adata)
    ops.normalize_total_log1p_(Xd, normalize=False, log1p=True, base=base)
    _store(adata, Xd)


def filter_genes(data, min_counts=None, min_cells=None, max_counts=None, max_cells=None, inplace: bool = True, copy: bool = False):
    """``scanpy.pp.filter_genes``: keep genes by total counts or by the number of cells expressing them (exactly one criterion per
    call, like scanpy).  ``inplace=False`` returns ``(gene_subset, number_per_gene)`` as numpy arrays."""
    return _filter(data, "genes", min_counts, min_cells, max_counts, max_cells, inplace, copy)


def filter_cells(data, min_counts=None, min_genes=None, max_counts=None, max_genes=None, inplace: bool = True, copy: bool = False):
    """``scanpy.pp.filter_cells``."""
    return _filter(data, "cells", min_counts, min_genes, max_counts, max_genes, inplace, copy)


def _filter(data, target, min_counts, min_other, max_counts, max_other, inplace, copy):
    if copy:
        raise NotImplementedError("copy=True is not built")
    given = [o is not None for o in (min_counts, min_other, max_counts, max_other)]
    if sum(given) != 1:
        other = "cells" if target == "genes" else "genes"
        raise ValueError(f"Only provide one of the optional parameters `min_counts`, `min_{other}`, `max_counts`, `max_{other}` per call.")
    is_adata = hasattr(data, "X") and not isinstance(data, (np.ndarray, torch.Tensor))
    if is_adata:
        Xd = _to_device(data)
    elif isinstance(data, torch.Tensor):
        Xd = data
    else:
        Xd = torch.as_tensor(np.ascontiguousarray(data.toarray() if sp.issparse(data) else data, dtype=np.float32)).cuda()
    if target == "genes":
        s, _, k = ops.gene_stats(Xd, want_sumsq=False)
    else:
        s, k = ops.cell_stats(Xd)
    use_counts = min_counts is not None or max_counts is not None
    number = s if use_counts else k
    lo = min_counts if min_counts is not None else min_other
    hi = max_counts if max_counts is not None else max_other
    subset = number >= lo if lo is not None else number <= hi
    subset_np = subset.cpu().numpy()
    number_np = number.cpu().numpy()
    number_np = number_np if use_counts else number_np.astype(np.int64)
    if not inplace or not is_adata:
        return subset_np, number_np
    label = "n_counts" if use_counts else ("n_cells" if target == "genes" else "n_genes")
    if target == "genes":
        data.var[label] = number_np
        data._inplace_subset_var(subset_np)
    else:
        data.obs[label] = number_np
        data._inplace_subset_obs(subset_np)


_MAD_SCALE = 0.6744897501960817     # Φ⁻¹(3/4): statsmodels.robust.mad's normalising constant


def highly_variable_genes(adata, layer=None, n_top_genes: Optional[int] = None, min_disp: float = 0.5, max_disp: float = np.inf,
                          min_mean: float = 0.0125, max_mean: float = 3, span: float = 0.3, n_bins: int = 20, flavor: str = "seurat",
                          subset: bool = False, inplace: bool = True, batch_key=None, check_values: bool = True):
    """``scanpy.pp.highly_variable_genes(flavor="cell_ranger", n_top_genes=…)``, restated from scanpy 1.10.1.

    One device pass (:func:`ops.gene_stats`) gives each gene's fp64 Σx and Σx² over ``adata.X``; the rest is over G values on the
    host in float64.  Writes ``var`` columns ``highly_variable``, ``means``, ``dispersions`` and ``dispersions_norm`` (float32,
    as scanpy casts it) and ``uns["hvg"]``; ``subset=True`` keeps the selected genes (on the device when X is resident there).
    As in scanpy, ``n_top_genes`` makes the mean / dispersion cut-offs irrelevant.  Other flavours, ``batch_key``,
    ``n_top_genes=None``, ``layer`` and ``inplace=False`` raise NotImplementedError."""
    if flavor != "cell_ranger" or batch_key is not None or n_top_genes is None or layer is not None or not inplace:
        raise NotImplementedError("only highly_variable_genes(flavor='cell_ranger', n_top_genes=…) in place on adata.X is built")
    Xd = _to_device(adata)
    n = Xd.shape[0]
    s, q, _ = ops.gene_stats(Xd, want_nnz=False)
    df = cell_ranger_hvg(s.cpu().numpy(), q.cpu().numpy(), n, n_top_genes)
    adata.uns["hvg"] = {"flavor": flavor}
    for key in ("highly_variable", "means", "dispersions"):
        adata.var[key] = df[key]
    adata.var["dispersions_norm"] = df["dispersions_norm"].astype(np.float32)
    if subset:
        adata._inplace_subset_var(df["highly_variable"])


def cell_ranger_hvg(gene_sum: np.ndarray, gene_sumsq: np.ndarray, n_obs: int, n_top_genes: int) -> dict:
    """The cell_ranger selection (float64 columns) from each gene's Σx and Σx² over ``n_obs`` cells (scanpy 1.10.1
    ``_highly_variable_genes_single_batch`` / ``_subset_genes``):

    1. ``mean``; ``var`` with ddof = 1 as ``(mean(x²) − mean²)·n/(n − 1)``; ``mean[mean == 0] = 1e-12``; ``disp = var / mean``.
    2. Bins with edges ``[-inf, percentile(mean, 10, 15, …, 100), inf]``, right-closed like ``pd.cut``; duplicate edges raise
       ValueError as ``pd.cut`` does.
    3. Per bin ``median(disp)`` and ``MAD = median(|disp − median| / 0.6744897501960817)``; ``disp_norm = (disp − median) / MAD``.
       Choice of this restatement: a bin holding one gene has MAD = 0 and its gene gets NaN (0 / 0), as NumPy gives it; a bin whose
       genes share one dispersion likewise gets NaN.  NaN genes are never selected.
    4. ``n = min(n_top_genes, G)``, lowered to the number of non-NaN ``disp_norm`` if that is smaller; the cut is the n-th largest
       non-NaN ``disp_norm``, and a gene is selected when ``nan_to_num(disp_norm, nan=-inf) >= cut``."""
    gene_sum = np.asarray(gene_sum, np.float64)
    mean = gene_sum / n_obs
    var = (np.asarray(gene_sumsq, np.float64) / n_obs - mean**2) * (n_obs / (n_obs - 1))
    mean[mean == 0] = 1e-12
    disp = var / mean
    edges = np.r_[-np.inf, np.percentile(mean, np.arange(10, 105, 5)), np.inf]
    if np.any(np.diff(edges) == 0):
        raise ValueError(f"Bin edges must be unique: {edges!r}.")
    bins = np.searchsorted(edges, mean, side="left") - 1          # (edges[b], edges[b + 1]]
    avg = np.full(len(edges) - 1, np.nan)
    dev = np.full(len(edges) - 1, np.nan)
    for b in np.unique(bins):
        d = disp[bins == b]
        avg[b] = np.median(d)
        dev[b] = np.median(np.abs(d - avg[b]) / _MAD_SCALE)
    with np.errstate(divide="ignore", invalid="ignore"):
        disp_norm = (disp - avg[bins]) / dev[bins]
    finite = disp_norm[~np.isnan(disp_norm)]
    n = min(int(n_top_genes), disp_norm.size, finite.size)
    if n == 0:
        hv = np.zeros(disp_norm.size, bool)
    else:
        cut = np.sort(finite)[::-1][n - 1]
        hv = np.nan_to_num(disp_norm, nan=-np.inf) >= cut
    return {"highly_variable": hv, "means": mean, "dispersions": disp, "dispersions_norm": disp_norm}
