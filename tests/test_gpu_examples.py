"""The reference's example flows against the drop-in namespace (dance_b200/dropin.py + dance_b200/shims): the command-line
surface of the reference's example scripts restated in `_EXAMPLE_FLOWS` below (same imports, same calls, taken line by line from
examples/single_modality/imputation/scgnn2.py:178-237 and examples/single_modality/cell_type_annotation/scdeepsort.py:40-77)."""
import sys
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture
def synth_env(tmp_path, monkeypatch):
    # density 0.5: at the default 10 % the five synthetic types are barely separable on 400 genes (logistic regression: 34 %)
    monkeypatch.setenv("DANCE_B200_SYNTH", "cells=1200,genes=400,types=5,density=0.5")
    monkeypatch.chdir(tmp_path)
    from dance_b200 import dropin
    assert set(dropin.install()) == {"dance", "scanpy"}
    yield tmp_path
    for k in [k for k in sys.modules if k == "dance" or k.startswith("dance.") or k == "scanpy" or k.startswith("scanpy.")]:
        del sys.modules[k]


def _script(rel: str, flow: str, tmp_path: Path) -> Path:
    q = tmp_path / Path(rel).name
    q.write_text(flow)
    return q


_SCGNN2_FLOW = '''
import argparse
from pprint import pformat
import numpy as np
import scanpy as sc
import torch
from dance import logger
from dance.datasets.singlemodality import ImputationDataset
from dance.modules.single_modality.imputation.scgnn2 import ScGNN2
from dance.transforms import AnnDataTransform, CellwiseMaskData, Compose, FilterCellsScanpy, FilterGenesScanpy, FilterGenesTopK
from dance.transforms.misc import SetConfig
from dance.utils import set_seed
if __name__ == "__main__":
    parser = argparse.ArgumentParser()
    parser.add_argument("--total_epoch", type=int, default=31)
    parser.add_argument("--feature_AE_epoch", nargs=2, type=int, default=[500, 300])
    parser.add_argument("--feature_AE_batch_size", type=int, default=12800)
    parser.add_argument("--feature_AE_learning_rate", type=float, default=1e-3)
    parser.add_argument("--feature_AE_regu_strength", type=float, default=0.9)
    parser.add_argument("--feature_AE_dropout_prob", type=float, default=0)
    parser.add_argument("--feature_AE_concat_prev_embed", type=str, default=None)
    parser.add_argument("--graph_AE_epoch", type=int, default=200)
    parser.add_argument("--graph_AE_use_GAT", action="store_true", default=False)
    parser.add_argument("--graph_AE_GAT_dropout", type=float, default=0)
    parser.add_argument("--graph_AE_learning_rate", type=float, default=1e-2)
    parser.add_argument("--graph_AE_embedding_size", type=int, default=16)
    parser.add_argument("--graph_AE_concat_prev_embed", action="store_true", default=False)
    parser.add_argument("--graph_AE_normalize_embed", type=str, default=None)
    parser.add_argument("--graph_AE_graph_construction", type=str, default="v2")
    parser.add_argument("--graph_AE_neighborhood_factor", type=float, default=0.05)
    parser.add_argument("--graph_AE_retain_weights", action="store_true", default=False)
    parser.add_argument("--gat_multi_heads", type=int, default=2)
    parser.add_argument("--gat_hid_embed", type=int, default=64)
    parser.add_argument("--clustering_louvain_only", action="store_true", default=False)
    parser.add_argument("--clustering_use_flexible_k", action="store_true", default=False)
    parser.add_argument("--clustering_embed", type=str, default="graph")
    parser.add_argument("--clustering_method", type=str, default="KMeans")
    parser.add_argument("--cluster_AE_epoch", type=int, default=200)
    parser.add_argument("--cluster_AE_batch_size", type=int, default=12800)
    parser.add_argument("--cluster_AE_learning_rate", type=float, default=1e-3)
    parser.add_argument("--cluster_AE_regu_strength", type=float, default=0.9)
    parser.add_argument("--cluster_AE_dropout_prob", type=float, default=0)
    parser.add_argument("--data_dir", type=str, default="data")
    parser.add_argument("--dataset", default="mouse_brain_data", type=str)
    parser.add_argument("--train_size", type=float, default=0.9)
    parser.add_argument("--seed", type=int, default=0)
    parser.add_argument("--num_runs", type=int, default=1)
    args = parser.parse_args()
    rmses, mres = [], []
    for seed in range(args.seed, args.seed + args.num_runs):
        set_seed(seed)
        logger.info(pformat(vars(args)))
        preprocessing_pipeline = Compose(
            FilterGenesScanpy(min_cells=0.01),
            FilterCellsScanpy(min_genes=0.01),
            FilterGenesTopK(num_genes=2000, mode="var"),
            CellwiseMaskData(add_test_mask=True),
            AnnDataTransform(sc.pp.log1p),
            SetConfig({"feature_channel": ["train_mask", "valid_mask", "test_mask"], "feature_channel_type": ["layers", "layers", "layers"]}),
            log_level="INFO",
        )
        dataloader = ImputationDataset(data_dir=args.data_dir, dataset=args.dataset, train_size=args.train_size)
        data = dataloader.load_data(transform=preprocessing_pipeline)
        train_mask, valid_mask, test_mask = data.get_x(return_type="default")
        if not isinstance(data.data.X, np.ndarray):
            x_train = data.data.X.A * train_mask
            X = data.data.X.A
        else:
            x_train = data.data.X * train_mask
            X = data.data.X
        model = ScGNN2(args)
        model.fit(x_train)
        imputed_data = model.predict()
        X = torch.from_numpy(X)
        imputed_data = torch.from_numpy(imputed_data)
        train_RMSE = model.score(X, imputed_data.clone(), ~train_mask, "RMSE", log1p=False)
        val_pcc = model.score(X, imputed_data.clone(), ~valid_mask, "PCC", log1p=False)
        test_RMSE = model.score(X, imputed_data.clone(), ~test_mask, "RMSE", log1p=False)
        test_mre = model.score(X, imputed_data.clone(), ~test_mask, metric="MRE", log1p=False)
        rmses.append(test_RMSE)
        mres.append(test_mre)
    print(f"rmses: {rmses}")
    print(f"mres: {mres}")
'''

_SCDEEPSORT_FLOW = '''
import argparse
import pprint
from typing import get_args
import numpy as np
import torch
from dance import logger
from dance.datasets.singlemodality import CellTypeAnnotationDataset
from dance.modules.single_modality.cell_type_annotation.scdeepsort import ScDeepSort
from dance.typing import LogLevel
from dance.utils import set_seed
if __name__ == "__main__":
    parser = argparse.ArgumentParser()
    parser.add_argument("--batch_size", type=int, default=500)
    parser.add_argument("--cache", action="store_true")
    parser.add_argument("--dense_dim", type=int, default=400)
    parser.add_argument("--device", type=str, default="cpu")
    parser.add_argument("--dropout", type=float, default=0.1)
    parser.add_argument("--hidden_dim", type=int, default=200)
    parser.add_argument("--log_level", type=str, default="INFO", choices=get_args(LogLevel))
    parser.add_argument("--lr", type=float, default=1e-3)
    parser.add_argument("--n_epochs", type=int, default=300)
    parser.add_argument("--n_layers", type=int, default=1)
    parser.add_argument("--species", default="mouse", type=str)
    parser.add_argument("--test_dataset", nargs="+", type=int, default=[1759])
    parser.add_argument("--test_rate", type=float, default=0.2)
    parser.add_argument("--tissue", default="Spleen", type=str)
    parser.add_argument("--train_dataset", nargs="+", type=int, default=[1970])
    parser.add_argument("--weight_decay", type=float, default=5e-4)
    parser.add_argument("--seed", type=int, default=42)
    parser.add_argument("--num_runs", type=int, default=1)
    parser.add_argument("--val_size", type=float, default=0.0)
    args = parser.parse_args()
    logger.setLevel(args.log_level)
    scores = []
    for seed in range(args.seed, args.seed + args.num_runs):
        set_seed(seed)
        model = ScDeepSort(args.dense_dim, args.hidden_dim, args.n_layers, args.species, args.tissue, dropout=args.dropout,
                           batch_size=args.batch_size, device=args.device)
        preprocessing_pipeline = model.preprocessing_pipeline(n_components=args.dense_dim)
        dataloader = CellTypeAnnotationDataset(species=args.species, tissue=args.tissue, test_dataset=args.test_dataset,
                                               train_dataset=args.train_dataset, data_dir="./", val_size=args.val_size)
        data = dataloader.load_data(transform=preprocessing_pipeline, cache=args.cache)
        y_train = data.get_y(split_name="train", return_type="torch").argmax(1)
        y_test = data.get_y(split_name="test", return_type="torch")
        num_labels = y_test.shape[1]
        g = data.data.uns["CellFeatureGraph"]
        num_genes = data.shape[1]
        gene_ids = torch.arange(num_genes)
        train_cell_ids = torch.LongTensor(data.train_idx) + num_genes
        test_cell_ids = torch.LongTensor(data.test_idx) + num_genes
        g_train = g.subgraph(torch.concat((gene_ids, train_cell_ids)))
        g_test = g.subgraph(torch.concat((gene_ids, test_cell_ids)))
        model.fit(g_train, y_train, epochs=args.n_epochs, lr=args.lr, weight_decay=args.weight_decay, val_ratio=args.test_rate)
        score = model.score(g_test, y_test)
        scores.append(score.item())
        print(f"{score=:.4f}")
    print(f"{scores}")
'''


def test_scgnn2_example_script_runs_unchanged(cuda, synth_env, capsys):
    """examples/single_modality/imputation/scgnn2.py with its own documented reduced schedule
    (``--feature_AE_epoch 20 10 --cluster_AE_epoch 20 --total_epoch 2``, script docstring) plus a short Graph-AE."""
    from dance_b200 import dropin
    script = _script("single_modality/imputation/scgnn2.py", _SCGNN2_FLOW, synth_env)
    ns = dropin.run_example(script, ["--total_epoch", "2", "--feature_AE_epoch", "20", "10", "--cluster_AE_epoch", "20", "--graph_AE_epoch", "20",
                                     "--graph_AE_neighborhood_factor", "10"])
    out = capsys.readouterr().out
    assert "rmses:" in out and "mres:" in out
    rm = ns["rmses"]
    assert len(rm) == 1 and np.isfinite(rm[0]) and rm[0] > 0
    assert ns["imputed_data"].shape == ns["X"].shape


def test_scdeepsort_example_script_runs_unchanged(cuda, synth_env, capsys):
    """examples/single_modality/cell_type_annotation/scdeepsort.py (BASELINE config 0 at reduced size) — only CLI arguments differ
    from the defaults (``--device cuda``: this framework has no CPU path)."""
    from dance_b200 import dropin
    script = _script("single_modality/cell_type_annotation/scdeepsort.py", _SCDEEPSORT_FLOW, synth_env)
    ns = dropin.run_example(script, ["--device", "cuda", "--dense_dim", "64", "--hidden_dim", "32", "--n_epochs", "20", "--lr", "1e-2", "--batch_size", "200",
                                     "--weight_decay", "0", "--cache"])
    assert "score=" in capsys.readouterr().out
    assert ns["scores"][0] > 0.6, ns["scores"]
    # the processed Data object was cached as a pickle (datasets/base.py:117-149) and is served from it on the second load
    cached = list((synth_env / "cache").glob("*.pkl"))
    assert len(cached) == 1
    again = ns["dataloader"].load_data(transform=ns["preprocessing_pipeline"], cache=True)
    assert again.shape == ns["data"].shape and again.data.uns["CellFeatureGraph"].num_edges() == ns["g"].num_edges()
