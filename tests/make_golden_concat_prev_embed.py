"""Generate ``tests/golden/scgnn_concat_prev_embed.npz`` from the REFERENCE's own ``feature_AE_handler`` and ``graph_AE_handler``
(through ``oracle.ref_loader``) with ``feature_AE_concat_prev_embed`` / ``graph_AE_concat_prev_embed``.  TEST INFRASTRUCTURE, like
``oracle/make_golden.py``: it needs the reference sources and is run by hand from the repository root:

    python tests/make_golden_concat_prev_embed.py

200 cells × 64 genes, a 16-d previous graph embedding and a 128-d previous feature embedding, 1-epoch schedules.  The reference's
``ExpressionDataset``, ``Feature_AE``, ``Graph_AE``, ``feature2adj`` and ``Feature_AE.load_state_dict`` are wrapped to record, per
call:

* ``fae.{graph,feature}.e{0,1,2}``: the matrix the Feature-AE trains on (``.X``), its ``dim``, which checkpoint entry was loaded
  (``.loaded``: "none" | "model" | "model_concat") and the returned checkpoint's keys (``.keys``); epochs chain their checkpoints;
* ``gae.{gcn,gat}.e{0,1}``: the matrix feature2adj sees (``.X``), its kNN lists (``.knn``, [N, k]) and the Graph_AE input ``dim``.
"""
from __future__ import annotations

import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from oracle import ref_loader  # noqa: E402

OUT = ROOT / "tests" / "golden" / "scgnn_concat_prev_embed.npz"
N, G = 200, 64


def _inputs():
    rng = np.random.default_rng(2024)
    X = np.where(rng.random((N, G)) < 0.7, 0.0, rng.gamma(2.0, 1.5, size=(N, G))).astype(np.float32)
    X = np.log1p(X).astype(np.float32)
    graph_embed = rng.standard_normal((N, 16)).astype(np.float32)
    feature_embed = np.maximum(rng.standard_normal((N, 128)), 0).astype(np.float32)
    x_embed = np.maximum(rng.standard_normal((N, 128)) * 2.0, 0).astype(np.float32)
    return X, graph_embed, feature_embed, x_embed


def _args(**kw):
    a = dict(feature_AE_batch_size=64, feature_AE_epoch=[1, 1], feature_AE_learning_rate=1e-3, feature_AE_regu_strength=0.9,
             feature_AE_dropout_prob=0.0, feature_AE_concat_prev_embed=None, graph_AE_use_GAT=False, graph_AE_learning_rate=1e-2,
             graph_AE_epoch=1, graph_AE_embedding_size=16, graph_AE_concat_prev_embed=False, graph_AE_normalize_embed=None,
             graph_AE_GAT_dropout=0.0, graph_AE_neighborhood_factor=0.05, graph_AE_retain_weights=False, gat_multi_heads=2,
             gat_hid_embed=64)
    a.update(kw)
    return SimpleNamespace(**a)


def main():
    ref = ref_loader.scgnn2()
    X, graph_embed, feature_embed, x_embed = _inputs()
    out = {"X": X, "graph_embed": graph_embed, "feature_embed": feature_embed, "x_embed": x_embed}
    rec = {}

    orig_ds, orig_fae, orig_gae, orig_f2a = ref.ExpressionDataset, ref.Feature_AE, ref.Graph_AE, ref.feature2adj
    orig_load = orig_fae.load_state_dict

    def dataset(Xw, *a, **k):
        rec["X"] = np.array(Xw, dtype=np.float32)
        return orig_ds(Xw, *a, **k)

    def feature_ae(dim, *a, **k):
        rec["dim"] = dim
        return orig_fae(dim, *a, **k)

    def graph_ae(dim, *a, **k):
        rec["dim"] = dim
        return orig_gae(dim, *a, **k)

    def f2a(X_embed, neighborhood_factor, retain_weights):
        rec["X"] = np.array(X_embed, dtype=np.float32)
        adj, adj_train, edge_list = orig_f2a(X_embed, neighborhood_factor, retain_weights)
        rec["knn"] = np.array([e[1] for e in edge_list], dtype=np.int32).reshape(X_embed.shape[0], -1)
        return adj, adj_train, edge_list

    def load(self, sd, *a, **k):
        rec["loaded_sd"] = sd
        return orig_load(self, sd, *a, **k)

    ref.ExpressionDataset, ref.Feature_AE, ref.Graph_AE, ref.feature2adj = dataset, feature_ae, graph_ae, f2a
    orig_fae.load_state_dict = load
    try:
        trs = np.zeros((N, G), dtype=np.float32)
        for mode in ("graph", "feature"):
            state = None
            for e in (0, 1, 2):
                torch.manual_seed(e)
                rec.clear()
                param = {"device": "cpu", "epoch_num": e, "total_epoch": 2, "dataloader_kwargs": {}, "n_feature_orig": G,
                         "x_dropout": X, "graph_embed": graph_embed, "feature_embed": feature_embed,
                         "impute_regu": (np.zeros((N, N), np.float32), np.zeros((N, N), np.float32))}
                _, recon, ckpt = ref.feature_AE_handler(X, trs, _args(feature_AE_concat_prev_embed=mode), param, state)
                sd = rec.get("loaded_sd")
                loaded = "none" if sd is None else ("model_concat" if state is not None and sd is state.get("model_concat") else "model")
                key = f"fae.{mode}.e{e}"
                out[key + ".X"], out[key + ".dim"] = rec["X"], np.int64(rec["dim"])
                out[key + ".loaded"], out[key + ".keys"] = np.array(loaded), np.array(sorted(ckpt))
                assert recon.shape == (N, G)
                state = ckpt
        for branch, gat in (("gcn", False), ("gat", True)):
            for e in (0, 1):
                torch.manual_seed(e)
                rec.clear()
                param = {"device": "cpu", "epoch_num": e, "graph_embed": graph_embed}
                ref.graph_AE_handler(x_embed, None, _args(graph_AE_use_GAT=gat, graph_AE_concat_prev_embed=True), param)
                key = f"gae.{branch}.e{e}"
                out[key + ".X"], out[key + ".knn"], out[key + ".dim"] = rec["X"], rec["knn"], np.int64(rec["dim"])
    finally:
        ref.ExpressionDataset, ref.Feature_AE, ref.Graph_AE, ref.feature2adj = orig_ds, orig_fae, orig_gae, orig_f2a
        orig_fae.load_state_dict = orig_load
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT} ({OUT.stat().st_size} bytes)")


if __name__ == "__main__":
    main()
