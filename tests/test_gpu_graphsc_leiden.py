"""graph-sc with cluster_method="leiden" on the device (GraphSC.predict → modules.graphsc.run_leiden: the 300-NN UMAP graph of
the embedding, then Leiden), the device highly_variable_genes(flavor="cell_ranger") of its preprocessing pipeline, and the
reference's example script examples/single_modality/clustering/graphsc.py restated line by line (`_GRAPHSC_FLOW`)."""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import graphsc_ref as R
import hvg_ref

pytestmark = pytest.mark.gpu


def _graph():
    from dance_b200.graph import GraphLite
    gd = R.fixture_graph()
    g = GraphLite(torch.from_numpy(gd["src"]).long(), torch.from_numpy(gd["dst"]).long(), gd["n_nodes"])
    g.edata["weight"] = torch.from_numpy(gd["weight"]).float()
    G = gd["n_genes"]
    g.ndata["features"] = torch.from_numpy(gd["features"]).float()
    g.ndata["feat_id"] = torch.cat([-torch.ones(G, dtype=torch.int32), torch.arange(gd["n_nodes"] - G, dtype=torch.int32)])
    return g


def _by_hand(z, n_neighbors):
    from dance_b200.leiden import leiden, neighbor_graph
    res = leiden(neighbor_graph(torch.from_numpy(np.ascontiguousarray(z, np.float32)).cuda(), n_neighbors), resolution=1.0,
                 max_iterations=-1)
    return res.labels.cpu().numpy().tolist()


def test_predict_leiden_is_neighbor_graph_then_leiden(cuda):
    from dance_b200.modules.graphsc import GraphSC
    m = GraphSC(cluster_method="leiden", device=cuda)
    m.fit(_graph(), epochs=2, lr=1e-3)
    assert m.z.shape[1] == 300 and m.z.shape[0] >= 300
    pred = m.predict()
    assert isinstance(pred, list) and all(type(x) is int for x in pred)
    assert pred == _by_hand(m.z, 300)


def test_small_n_clamp(cuda):
    """scanpy's compute_neighbors: 300 > n_obs → 1 + int(0.5 · n_obs) neighbours."""
    from dance_b200.modules.graphsc import run_leiden
    rng = np.random.default_rng(3)
    z = (rng.normal(0, 5, (3, 300))[np.repeat(np.arange(3), 67)] + rng.normal(size=(201, 300))).astype(np.float32)
    assert run_leiden(z, cuda) == _by_hand(z, 101)


def test_fit_eval_epoch_with_leiden(cuda):
    from dance_b200.modules.graphsc import GraphSC
    m = GraphSC(cluster_method="leiden", device=cuda)
    m.fit(_graph(), epochs=2, lr=1e-3, eval_epoch=True)
    assert np.isfinite(m.score(None, np.arange(m.z.shape[0])))


def test_device_hvg_matches_restatement(cuda):
    from dance_b200.data import AnnDataLite
    from dance_b200.transforms import AnnDataTransform
    from dance_b200.transforms.pp import cell_ranger_hvg
    from dance_b200 import ops
    rng = np.random.default_rng(1)
    X = np.log1p(rng.poisson(rng.gamma(0.5, 2.0, 800), size=(1500, 800))).astype(np.float32)
    X = np.ascontiguousarray(X[:, X.sum(0) > 0])
    ref = hvg_ref.cell_ranger(X, 300)
    s, q, _ = ops.gene_stats(torch.from_numpy(X).cuda(), want_nnz=False)
    out = cell_ranger_hvg(s.cpu().numpy(), q.cpu().numpy(), X.shape[0], 300)
    assert np.array_equal(out["highly_variable"], ref["highly_variable"].to_numpy())
    # the sums differ only in order; var = mean(x²) − mean² loses digits to cancellation, so the dispersions get a wider rtol
    assert np.allclose(out["means"], ref["means"].to_numpy(), rtol=1e-12, atol=0)
    for key in ("dispersions", "dispersions_norm"):
        assert np.allclose(out[key], ref[key].to_numpy(), rtol=1e-9, atol=1e-12, equal_nan=True), key
    ad = AnnDataLite(X.copy())
    AnnDataTransform("scanpy.pp.highly_variable_genes", min_mean=0.0125, max_mean=4, flavor="cell_ranger", min_disp=0.5,
                     n_top_genes=300, subset=True)(type("D", (), {"data": ad})())
    keep = ref["highly_variable"].to_numpy()
    assert ad.shape == (X.shape[0], 300) and np.array_equal(ad.X, X[:, keep])
    assert np.array_equal(ad.var["names"], np.flatnonzero(keep).astype(str))
    assert np.allclose(ad.var["means"], ref["means"].to_numpy()[keep], rtol=1e-12, atol=0)
    assert ad.var["dispersions_norm"].dtype == np.float32 and ad.uns["hvg"] == {"flavor": "cell_ranger"}


@pytest.fixture
def synth_env(tmp_path, monkeypatch):
    monkeypatch.setenv("DANCE_B200_SYNTH", "cells=1200,genes=400,types=5,density=0.5")
    monkeypatch.chdir(tmp_path)
    from dance_b200 import dropin
    assert set(dropin.install()) == {"dance", "scanpy"}
    yield tmp_path
    for k in [k for k in sys.modules if k == "dance" or k.startswith("dance.") or k == "scanpy" or k.startswith("scanpy.")]:
        del sys.modules[k]


_GRAPHSC_FLOW = '''
import argparse
import numpy as np
from dance.datasets.singlemodality import ClusteringDataset
from dance.modules.single_modality.clustering.graphsc import GraphSC
from dance.utils import set_seed
if __name__ == "__main__":
    parser = argparse.ArgumentParser()
    parser.add_argument("-e", "--epochs", default=100, type=int)
    parser.add_argument("-dv", "--device", default="auto")
    parser.add_argument("-if", "--in_feats", default=50, type=int)
    parser.add_argument("-bs", "--batch_size", default=128, type=int)
    parser.add_argument("-nw", "--normalize_weights", default="log_per_cell", choices=["log_per_cell", "per_cell"])
    parser.add_argument("-ac", "--activation", default="relu", choices=["leaky_relu", "relu", "prelu", "gelu"])
    parser.add_argument("-drop", "--dropout", default=0.1, type=float)
    parser.add_argument("-nf", "--node_features", default="scale", choices=["scale_by_cell", "scale", "none"])
    parser.add_argument("-sev", "--same_edge_values", default=False, action="store_true")
    parser.add_argument("-en", "--edge_norm", default=True, action="store_true")
    parser.add_argument("-hr", "--hidden_relu", default=False, action="store_true")
    parser.add_argument("-hbn", "--hidden_bn", default=False, action="store_true")
    parser.add_argument("-lr", "--learning_rate", type=float, default=1e-5)
    parser.add_argument("-nl", "--n_layers", type=int, default=1, choices=[1, 2])
    parser.add_argument("-agg", "--agg", default="sum", choices=["sum", "mean"])
    parser.add_argument("-hd", "--hidden_dim", type=int, default=200)
    parser.add_argument("-nh", "--n_hidden", type=int, default=1, choices=[0, 1, 2])
    parser.add_argument("-h1", "--hidden_1", type=int, default=300)
    parser.add_argument("-h2", "--hidden_2", type=int, default=0)
    parser.add_argument("-ng", "--nb_genes", type=int, default=3000)
    parser.add_argument("-nr", "--num_run", type=int, default=1)
    parser.add_argument("-nbw", "--num_workers", type=int, default=1)
    parser.add_argument("-eve", "--eval_epoch", action="store_true")
    parser.add_argument("-show", "--show_epoch_ari", action="store_true")
    parser.add_argument("-plot", "--plot", default=False, action="store_true")
    parser.add_argument("-dd", "--data_dir", default="./data", type=str)
    parser.add_argument("-data", "--dataset", default="10X_PBMC",
                        choices=["10X_PBMC", "mouse_bladder_cell", "mouse_ES_cell", "worm_neuron_cell"])
    parser.add_argument("--seed", type=int, default=0, help="Initial seed random, offset for each repeatition")
    parser.add_argument("--num_runs", type=int, default=5, help="Number of repetitions")
    parser.add_argument("--cache", action="store_true", help="Cache processed data.")
    args = parser.parse_args()
    aris = []
    for seed in range(args.seed, args.seed + args.num_runs):
        set_seed(seed)
        dataloader = ClusteringDataset(args.data_dir, args.dataset)
        preprocessing_pipeline = GraphSC.preprocessing_pipeline(
            n_top_genes=args.nb_genes,
            normalize_weights=args.normalize_weights,
            n_components=args.in_feats,
            normalize_edges=args.edge_norm,
        )
        data = dataloader.load_data(transform=preprocessing_pipeline, cache=args.cache)
        graph, y = data.get_train_data()
        n_clusters = len(np.unique(y))
        model = GraphSC(agg=args.agg, activation=args.activation, in_feats=args.in_feats, n_hidden=args.n_hidden,
                        hidden_dim=args.hidden_dim, hidden_1=args.hidden_1, hidden_2=args.hidden_2,
                        dropout=args.dropout, n_layers=args.n_layers, hidden_relu=args.hidden_relu,
                        hidden_bn=args.hidden_bn, n_clusters=n_clusters, cluster_method="leiden",
                        num_workers=args.num_workers, device=args.device)
        model.fit(graph, epochs=args.epochs, lr=args.learning_rate, show_epoch_ari=args.show_epoch_ari,
                  eval_epoch=args.eval_epoch)
        score = model.score(None, y)
        print(f"{score=:.4f}")
        aris.append(score)
    print('graphsc')
    print(args.dataset)
    print(f'aris: {aris}')
    print(f'aris: {np.mean(aris)} +/- {np.std(aris)}')
'''


@pytest.mark.parametrize("extra", [[], ["--eval_epoch"]])
def test_graphsc_example_script_runs_unchanged(cuda, synth_env, capsys, extra):
    """examples/single_modality/clustering/graphsc.py (cluster_method="leiden") at a reduced size: only CLI arguments differ."""
    from dance_b200 import dropin
    script = synth_env / "graphsc.py"
    script.write_text(_GRAPHSC_FLOW)
    ns = dropin.run_example(script, ["-dv", "cuda", "--epochs", "5", "--num_runs", "1", "--nb_genes", "300", *extra])
    out = capsys.readouterr().out
    assert "score=" in out and "aris:" in out
    assert len(ns["aris"]) == 1 and np.isfinite(ns["aris"][0])
    assert ns["data"].shape[1] == 300
