"""graph-sc on the H100-native kernels — mirror of ``dance/modules/single_modality/clustering/graphsc.py`` (GraphSC :34-270,
GCNAE :290-380, InnerProductDecoder :386-411, WeightedGraphConv :414-484).

Training is :class:`dance_b200.engine.GraphSCEngine`: full-neighbour blocks over the cell–gene graph on the device, two train-mode
forwards per batch (the first one's embedding is recorded, the second one's logits give the loss), Adam once per batch.
Reference behaviour kept on purpose:

* the decoder's dropout (p = 0.1) is on whatever ``dropout`` is (``F.dropout`` defaults to training=True);
* with ``hidden_bn`` both forwards update the running statistics, and a one-row batch raises as BatchNorm1d does;
* ``eval_epoch`` chooses the epoch by ARI against the cell indices (``fit`` sets "label" to ``feat_id``);
* ``activation="prelu"`` raises TypeError on the first forward (F.prelu is handed no weight).
"""
from __future__ import annotations

import logging
from typing import Any, Literal, Optional

import numpy as np
import torch

from ..engine import GraphSCEngine, prepare_graph
from .scgnn2 import kmeans_fit_predict

_ACTIVATIONS = ("relu", "leaky_relu", "gelu")
logger = logging.getLogger(__name__)


class GraphSC:
    """GraphSC(agg, activation, in_feats, n_hidden, hidden_dim, hidden_1, hidden_2, dropout, n_layers, hidden_relu, hidden_bn,
    n_clusters, cluster_method, num_workers, device) — the reference's constructor (graphsc.py:69-107)."""

    def __init__(self, agg: str = "sum", activation: str = "relu", in_feats: int = 50, n_hidden: int = 1, hidden_dim: int = 200,
                 hidden_1: int = 300, hidden_2: int = 0, dropout: float = 0.1, n_layers: int = 1, hidden_relu: bool = False,
                 hidden_bn: bool = False, n_clusters: int = 10, cluster_method: Literal["kmeans", "leiden"] = "kmeans",
                 num_workers: int = 1, device: str = "auto", precision: Optional[str] = None, drop_seed: int = 0):
        self.n_layers, self.n_clusters, self.cluster_method, self.num_workers = n_layers, n_clusters, cluster_method, num_workers
        self.device = torch.device("cuda" if device in ("auto", "cpu") else device)
        if self.device.type != "cuda":
            raise RuntimeError("dance_b200 runs on CUDA devices only")
        self.activation = activation
        self.model = GraphSCEngine(agg=agg, activation=activation if activation in _ACTIVATIONS else "relu", in_feats=in_feats,
                                   n_hidden=n_hidden, hidden_dim=hidden_dim, hidden_1=hidden_1, hidden_2=hidden_2, dropout=dropout,
                                   n_layers=n_layers, hidden_relu=hidden_relu, hidden_bn=hidden_bn, device=self.device,
                                   drop_seed=drop_seed, precision=precision)
        self.z: Optional[np.ndarray] = None

    @staticmethod
    def preprocessing_pipeline(n_top_genes: int = 3000, normalize_weights: str = "log_per_cell", n_components: int = 50,
                               normalize_edges: bool = False, log_level="INFO"):
        """graphsc.py:109-153.  The scanpy steps run through AnnDataTransform, each dispatched to its device counterpart in
        :mod:`dance_b200.transforms.pp`; the cell–gene graph is PCACellFeatureGraph on the device."""
        from ..transforms import AnnDataTransform, Compose, SetConfig
        from ..transforms.graph import PCACellFeatureGraph
        transforms = [
            AnnDataTransform("scanpy.pp.filter_genes", min_counts=3),
            AnnDataTransform("scanpy.pp.filter_cells", min_counts=1),
            AnnDataTransform("scanpy.pp.normalize_total"),
            AnnDataTransform("scanpy.pp.log1p"),
            AnnDataTransform("scanpy.pp.highly_variable_genes", min_mean=0.0125, max_mean=4, flavor="cell_ranger", min_disp=0.5,
                             n_top_genes=n_top_genes, subset=True),
        ]
        if normalize_weights == "log_per_cell":
            transforms += [AnnDataTransform("scanpy.pp.log1p"), AnnDataTransform("scanpy.pp.normalize_total", target_sum=1)]
        elif normalize_weights == "per_cell":
            transforms.append(AnnDataTransform("scanpy.pp.normalize_total", target_sum=1))
        elif normalize_weights != "none":
            raise ValueError(f"Unknown normalization option {normalize_weights!r}."
                             "Available options are: 'none', 'log_per_cell', 'per_cell'")
        transforms += [
            PCACellFeatureGraph(n_components=n_components, normalize_edges=normalize_edges, feat_norm_mode="standardize"),
            SetConfig({"feature_channel": "CellFeatureGraph", "feature_channel_type": "uns", "label_channel": "Group"}),
        ]
        return Compose(*transforms, log_level=log_level)

    def fit(self, g, y: Optional[Any] = None, *, epochs: int = 100, lr: float = 1e-5, batch_size: int = 128,
            show_epoch_ari: bool = False, eval_epoch: bool = False):
        """graphsc.py:155-245.  ``g``: the CellFeatureGraph (GraphLite with ndata "features" / "feat_id", edata "weight")."""
        if self.activation not in _ACTIVATIONS:
            # GCNAE keeps an unknown name as a string, and "prelu" is F.prelu without its weight: both fail on the first call
            raise TypeError(f"activation {self.activation!r} cannot be called on a tensor alone (graphsc.py:324-331)")
        graph = prepare_graph(g, self.device)
        labels = np.arange(graph["n_cells"])                  # "label" := feat_id, the cell index (graphsc.py:179)
        aris, Z = [], {}
        for epoch in range(epochs):
            self.model.train_epoch(graph, graph["train_ids"], batch_size, lr)
            if eval_epoch or epoch == epochs - 1:
                self.z = self.model.z.cpu().numpy()
            if eval_epoch:
                score = self.score(None, labels)
                aris.append(score)
                if show_epoch_ari:
                    logger.info(f"epoch {epoch:4d}, ARI {score:.4f}")
                Z[epoch] = self.z
        if eval_epoch:
            self.z = Z[int(np.argmax(aris))]
        return self

    def predict(self, x: Optional[Any] = None):
        """KMeans(n_clusters, init="k-means++", random_state=5, n_init=10) on the device (graphsc.py:259-260), or Leiden on the
        embedding's 300-NN graph (:func:`run_leiden`)."""
        if self.cluster_method == "kmeans":
            return kmeans_fit_predict(self.z, self.n_clusters, self.device, seed=5, n_init=10).cpu().numpy().astype(np.int64)
        if self.cluster_method == "leiden":
            return run_leiden(self.z, self.device)
        raise ValueError(f"Unknown clustering {self.cluster_method}, available options are: 'kmeans', 'leiden'")

    def get_latent(self):
        return self.z

    def score(self, x, y, score_func=None) -> float:
        """Adjusted Rand index by default (``BaseClusteringMethod._DEFAULT_METRIC = "ari"``, modules/base.py)."""
        pred = self.predict(x)
        if score_func is None:
            from sklearn.metrics import adjusted_rand_score as score_func
        return float(score_func(np.asarray(y), pred))

    def fit_predict(self, x, y=None, **fit_kwargs):
        self.fit(x, y, **fit_kwargs)
        return self.predict(x)

    def fit_score(self, x, y, score_func=None, **fit_kwargs) -> float:
        self.fit(x, y, **fit_kwargs)
        return self.score(x, y, score_func)


def run_leiden(data, device=None):
    """graphsc.py:568-587, ``sc.pp.neighbors(AnnData(z), use_rep="X", n_neighbors=300, n_pcs=0); sc.tl.leiden(adata)``, on the
    device: the UMAP connectivities of the exact 300-NN graph of the rows of ``data`` (scanpy 1.10.1 ``compute_neighbors`` takes
    ``1 + int(0.5 · n_obs)`` neighbours when 300 > n_obs), then Leiden at ``tl.leiden``'s resolution = 1 until nothing moves.
    Returns the labels as a list of Python ints.  Label parity with leidenalg is unpinned (see :mod:`dance_b200.leiden`)."""
    from ..leiden import leiden, neighbor_graph
    X = torch.as_tensor(np.ascontiguousarray(data, dtype=np.float32), device=device or "cuda")
    n_obs = X.shape[0]
    n_neighbors = 300 if 300 <= n_obs else 1 + int(0.5 * n_obs)
    res = leiden(neighbor_graph(X, n_neighbors), resolution=1.0, max_iterations=-1)
    return [int(x) for x in res.labels.cpu().tolist()]
