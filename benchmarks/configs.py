"""Throughput of the other BASELINE.json configurations through the public model API (one JSON line each; the headline —
config 4, scGNN 1 M × 2 000 — is bench.py).  Device-event timed on synthetic data from dance_b200.synth; not a bench.py line.

  config 1  scDeepSort, 10 k cells × 2 k genes: PCACellFeatureGraph pipeline + ScDeepSort.fit (cells/s per training epoch incl. the
            per-epoch train / validation evaluation the reference performs)
  config 2  scGNN 100 k × 2 k, k = 15: `python bench.py --cells 100000` (same step as the headline)
  config 3  GraphSCI, N cells × 3 000 genes (default N = 500 000): one training epoch of GraphSCI.train (AE + gene-graph GNN, ZINB
            loss).  The GEMMs run in single-pass TF32 (`precision="tf32"`, at least bf16's 8-bit mantissa), the aggregate has the
            bf16-operand kernel available; there is no bf16 GEMM mode — dtype is reported as what ran
  config 5  SpaGCN: the reference model multiplies a DENSE N × N adjacency (spagcn.py:357-363); 200 k spots would need a 160 GB
            matrix, so the line is measured at --spots (default 20 000) on one GPU and says so

    python benchmarks/configs.py --only 1,3 [--cells3 500000]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def _ev():
    return torch.cuda.Event(enable_timing=True)


def config1(args):
    os.environ["DANCE_B200_SYNTH"] = "cells=10000,genes=2000,types=10"
    from dance_b200.datasets import CellTypeAnnotationDataset
    from dance_b200.modules.scdeepsort import ScDeepSort
    model = ScDeepSort(400, 200, 1, "synthetic", "tissue", dropout=0.1, batch_size=500, device="cuda", seed=0)
    t0 = time.perf_counter()
    data = CellTypeAnnotationDataset(species="synthetic", tissue="tissue", data_dir="/tmp/b2_cfg1").load_data(
        transform=model.preprocessing_pipeline(n_components=400))
    torch.cuda.synchronize()
    prep_s = time.perf_counter() - t0
    y = data.get_y(split_name="train", return_type="torch").argmax(1)
    g = data.data.uns["CellFeatureGraph"]
    G = data.shape[1]
    g_train = g.subgraph(torch.concat((torch.arange(G), torch.LongTensor(data.train_idx) + G)))
    model.fit(g_train, y, epochs=2, lr=1e-3, weight_decay=5e-4, val_ratio=0.2)          # warm-up
    torch.cuda.synchronize()
    s, e = _ev(), _ev()
    epochs = 10
    s.record()
    model.fit(g_train, y, epochs=epochs, lr=1e-3, weight_decay=5e-4, val_ratio=0.2)
    e.record()
    torch.cuda.synchronize()
    ms = s.elapsed_time(e) / epochs
    n_train = len(data.train_idx)
    return {"config": 1, "workload": "scDeepSort 10k cells × 2k genes, dense_dim 400, hidden 200, batch 500 (ScDeepSort.fit epoch = train + per-epoch evaluation)",
            "metric": "cells/sec per training epoch", "value": n_train / (ms / 1e3), "unit": "cells/s", "ms_per_epoch": ms,
            "preprocessing_s": prep_s, "edges": int(g.num_edges()), "dtype": "f32 (tf32x3 GEMMs)", "n_gpus": 1, "data": "synthetic"}


def config3(args):
    from dance_b200 import ops, synth
    from dance_b200.modules.graphsci import GraphSCI
    from dance_b200.transforms import FeatureFeatureGraph
    from dance_b200.data import AnnDataLite, Data
    N, G = args.cells3, 3000
    dev = torch.device("cuda:0")
    Xraw = synth.expression_counts(N, G, seed=1, density=0.10, device=dev)
    X = Xraw.clone()
    ops.normalize_total_log1p_(X, normalize=False, log1p=True)
    # gene-gene graph from a 20 k-cell sample (the graph has G nodes; building it is outside the epoch)
    sample = Data(AnnDataLite(X[:20000].cpu().numpy()))
    FeatureFeatureGraph(threshold=0.05, normalize_edges=True)(sample)
    graph = sample.data.uns["FeatureFeatureGraph"]
    graph.ndata["feat"] = X.t().contiguous()       # node features of the gene graph = (log-)expression of ALL cells ([G, N], graphsci.py:126)
    del sample
    model = GraphSCI(num_cells=N, num_genes=G, dataset="synthetic", dropout=0.1, gpu=0, seed=0, precision="tf32")
    model._bind_graph(graph)
    n_counts = Xraw.sum(1)
    model.size_factors = (n_counts / torch.median(n_counts)).contiguous()      # what fit() sets up (graphsci.py:270-276)
    model.lr, model.weight_decay = 1e-3, 1e-5
    tm = torch.ones(N, G, dtype=torch.uint8, device=dev)
    for _ in range(2):
        model.train(X, Xraw, graph, tm, tm, le=1, la=1e-9, ke=1e2, ka=1)
    torch.cuda.synchronize()
    s, e = _ev(), _ev()
    epochs = 3
    s.record()
    for _ in range(epochs):
        model.train(X, Xraw, graph, tm, tm, le=1, la=1e-9, ke=1e2, ka=1)
    e.record()
    torch.cuda.synchronize()
    ms = s.elapsed_time(e) / epochs
    return {"config": 3, "workload": f"GraphSCI {N} cells × {G} genes: one training epoch (AE + gene-graph GNN, ZINB + adjacency losses)",
            "metric": "cells/sec per training epoch", "value": N / (ms / 1e3), "unit": "cells/s", "ms_per_epoch": ms,
            "dtype": "tf32 single-pass GEMMs (no bf16 GEMM mode is built; the aggregate's bf16-operand kernel is available)", "n_gpus": 1,
            "data": "synthetic", "gene_graph_edges": int(graph.num_edges())}


def config5(args):
    from dance_b200 import ops, synth
    from dance_b200.modules.spagcn import SimpleGCDEC
    n, G = args.spots, 5000
    dev = torch.device("cuda:0")
    X = synth.expression_counts(n, G, seed=2, density=0.10, device=dev)
    ops.normalize_total_log1p_(X, target_sum=1e4, max_fraction=1.0)
    pcs = ops.pca(X, 50)["scores"].contiguous()
    xy = synth.spatial_coordinates(n, seed=2, device=dev).contiguous()
    D = ops.pairwise_l2_dense(xy)
    adj = torch.exp(-(D * D) / (2 * 150.0**2))
    model = SimpleGCDEC(50, 50, device=dev)
    init = torch.randint(0, 7, (n, ), generator=torch.Generator().manual_seed(0)).numpy()
    t0 = time.perf_counter()
    model.bind(pcs, adj)                          # AX = adj · X once (tensor-core GEMM); every epoch is then AX·W + b
    torch.cuda.synchronize()
    bind_s = time.perf_counter() - t0
    model.fit(pcs, adj, lr=0.005, epochs=5, opt="admin", init_labels=init, tol=0)
    torch.cuda.synchronize()
    s, e = _ev(), _ev()
    epochs = 50
    s.record()
    model.fit(pcs, adj, lr=0.005, epochs=epochs, opt="admin", init_labels=init, tol=0)
    e.record()
    torch.cuda.synchronize()
    ms = s.elapsed_time(e) / epochs
    return {"config": 5, "workload": f"SpaGCN SimpleGCDEC {n} spots × {G} genes → 50 PCs, dense {n}×{n} spatial adjacency (reference semantics); "
                                     "BASELINE names 200k spots on 4 GPUs — the dense adjacency alone would be 160 GB",
            "metric": "spots/sec per training epoch", "value": n / (ms / 1e3), "unit": "spots/s", "ms_per_epoch": ms, "adj_x_once_s": bind_s,
            "dtype": "f32 (tf32x3 GEMMs)", "n_gpus": 1, "data": "synthetic"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", type=str, default="1,3,5")
    ap.add_argument("--cells3", type=int, default=500_000)
    ap.add_argument("--spots", type=int, default=20_000)
    args = ap.parse_args()
    fns = {"1": config1, "3": config3, "5": config5}
    for k in args.only.split(","):
        try:
            print(json.dumps(fns[k.strip()](args)), flush=True)
        except Exception as ex:     # one failing configuration must not hide the others
            print(json.dumps({"config": int(k), "error": f"{type(ex).__name__}: {ex}"}), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
