"""Throughput of the other BASELINE.json configurations through the public model API (one JSON line each; the headline —
config 4, scGNN 1 M × 2 000 — is bench.py).  Device-event timed on synthetic data from dance_b200.synth; not a bench.py line.

  config 1  scDeepSort, 10 k cells × 2 k genes: PCACellFeatureGraph pipeline + ScDeepSort.fit (cells/s per training epoch incl. the
            per-epoch train / validation evaluation the reference performs)
  config 2  scGNN 100 k × 2 k, k = 15: `python bench.py --cells 100000` (same step as the headline)
  config 3  GraphSCI, N cells × 3 000 genes (default N = 500 000): one training epoch of GraphSCI.train (AE + gene-graph GNN, ZINB
            loss), with the training schedule GraphSCI chose for the size and the peak of torch.cuda.max_memory_allocated()
            over the whole run (inputs included).  The GEMMs run in the precision BASELINE names, bf16 (`--precision3 bf16`, the default: operands rounded to
            bfloat16 in the kernel, fp32 accumulate and fp32 tensors); `--precision3 tf32` gives the earlier single-pass TF32
            line, `tf32x3` the fp32-accurate one.  dtype is reported as what ran
  config 5  SpaGCN: the reference model multiplies a DENSE N × N adjacency (spagcn.py:357-363); 200 k spots would need a 160 GB
            matrix, so the dense line (`--adjacency dense`, the default) is measured at --spots (default 20 000) on one GPU and says
            so.  `--adjacency coords --spots 200000` runs the BASELINE size on one GPU from the spot coordinates (matrix.SpotDistance):
            calculate_p, the AX build, a training epoch and refine, each timed; AX is checked on 64 sampled rows against an fp64
            sum over all columns before timing; plus the dense and the coordinate AX build on the same 20 000-spot input

    python benchmarks/configs.py --only 1,3 [--cells3 500000] [--precision3 bf16|tf32|tf32x3]
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


def config3_data(N, G=3000):
    """Configuration 3's inputs at N cells: (X log1p counts, Xraw counts, the gene graph with Xᵀ as its node features)."""
    from dance_b200 import ops, synth
    from dance_b200.transforms import FeatureFeatureGraph
    from dance_b200.data import AnnDataLite, Data
    dev = torch.device("cuda:0")
    Xraw = synth.expression_counts(N, G, seed=1, density=0.10, device=dev)
    X = Xraw.clone()
    ops.normalize_total_log1p_(X, normalize=False, log1p=True)
    # gene-gene graph from a 20 k-cell sample (the graph has G nodes; building it is outside the epoch)
    sample = Data(AnnDataLite(X[:20000].cpu().numpy()))
    FeatureFeatureGraph(threshold=0.05, normalize_edges=True)(sample)
    graph = sample.data.uns["FeatureFeatureGraph"]
    graph.ndata["feat"] = X.t().contiguous()       # node features of the gene graph = (log-)expression of ALL cells ([G, N], graphsci.py:126)
    return X, Xraw, graph


def config3_model(N, G, X, Xraw, graph, precision):
    from dance_b200.modules.graphsci import GraphSCI
    model = GraphSCI(num_cells=N, num_genes=G, dataset="synthetic", dropout=0.1, gpu=0, seed=0, precision=precision)
    model._bind_graph(graph)
    n_counts = Xraw.sum(1)
    model.size_factors = (n_counts / torch.median(n_counts)).contiguous()      # what fit() sets up (graphsci.py:270-276)
    model.lr, model.weight_decay = 1e-3, 1e-5
    return model


def config3(args):
    N, G = args.cells3, 3000
    dev = torch.device("cuda:0")
    torch.cuda.reset_peak_memory_stats()
    X, Xraw, graph = config3_data(N, G)
    model = config3_model(N, G, X, Xraw, graph, args.precision3)
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
            "dtype": DTYPE3[args.precision3], "n_gpus": 1, "schedule": model.schedule(),
            "peak_memory_gib": torch.cuda.max_memory_allocated() / 2**30,
            "data": "synthetic", "gene_graph_edges": int(graph.num_edges()), "card": _card()}


DTYPE3 = {
    "bf16": "bf16 GEMMs (operands rounded to bfloat16 in the kernel, fp32 accumulate; fp32 tensors and epilogue)",
    "tf32": "tf32 single-pass GEMMs",
    "tf32x3": "f32 (tf32x3 GEMMs)",
}


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


def _spot_weights64(xy, rows, c0, c1, l):
    from dance_b200 import ops
    r = xy[rows]
    D = ops.pairwise_l2_dense(torch.cat([r, xy[c0:c1]]))[:r.shape[0], r.shape[0]:].contiguous()
    return ops.exp_adj(D, l)[0].double()


def _check_ax_rows(xy, X, AX, l, n_check=64, chunk=8192):
    """64 sampled rows of AX against an fp64 sum over all columns of the dense path's fp32 weights; raises on a mismatch."""
    n = xy.shape[0]
    rows = torch.randperm(n, generator=torch.Generator().manual_seed(1))[:n_check].to(xy.device)
    ref = torch.zeros((n_check, X.shape[1]), dtype=torch.float64, device=xy.device)
    scale = torch.zeros_like(ref)
    for c0 in range(0, n, chunk):
        W = _spot_weights64(xy, rows, c0, min(n, c0 + chunk), l)
        ref += W @ X[c0:c0 + chunk].double()
        scale += W @ X[c0:c0 + chunk].double().abs()
    ratio = float(((AX[rows].double() - ref).abs() / (scale * 2.0**-21)).max())
    if not ratio < 8.0:
        raise RuntimeError(f"config 5 coords: AX differs from the fp64 sum by {ratio:.2f} x 2^-21 of W·|X|")
    return ratio


def _card():
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def config5_coords(args):
    from dance_b200 import ops, synth
    from dance_b200.matrix import SpotDistance
    from dance_b200.modules.spagcn import SimpleGCDEC, calculate_p, refine
    n, G, l = args.spots, 5000, 150.0
    dev = torch.device("cuda:0")
    X = synth.expression_counts(n, G, seed=2, density=0.10, device=dev)
    ops.normalize_total_log1p_(X, target_sum=1e4, max_fraction=1.0)
    pcs = ops.pca(X, 50)["scores"].contiguous()
    del X
    xy = synth.spatial_coordinates(n, seed=2, device=dev).contiguous()
    m = SpotDistance(xy.cpu().numpy())
    adj = m.exp(l)
    model = SimpleGCDEC(50, 50, device=dev)
    model.bind(pcs, adj)
    ax_ratio = _check_ax_rows(xy, pcs, model.AX, l)

    def timed(fn, reps):
        fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / reps * 1e3

    p_ms = timed(lambda: calculate_p(m, l), 3)
    bind_ms = timed(lambda: (setattr(model, "_bound", None), model.bind(pcs, adj)), 3)
    init = torch.randint(0, 7, (n, ), generator=torch.Generator().manual_seed(0)).numpy()
    model.fit(pcs, adj, lr=0.005, epochs=5, opt="admin", init_labels=init, tol=0)
    torch.cuda.synchronize()
    s, e = _ev(), _ev()
    epochs = 50
    s.record()
    model.fit(pcs, adj, lr=0.005, epochs=epochs, opt="admin", init_labels=init, tol=0)
    e.record()
    torch.cuda.synchronize()
    epoch_ms = s.elapsed_time(e) / epochs
    labels = model._labels.cpu().numpy()
    ids = list(range(n))
    refine_ms = timed(lambda: refine(ids, labels, m, shape="hexagon"), 1)
    # same input at 20 000 spots: the dense bind (N×N adjacency, tensor-core GEMM) against the coordinate bind
    k = min(n, 20_000)
    mk = SpotDistance(m.rows[:k])
    dense_adj = mk.exp(l).to_device()
    small = SimpleGCDEC(50, 50, device=dev)
    dense_bind_ms = timed(lambda: (setattr(small, "_bound", None), small.bind(pcs[:k], dense_adj)), 3)
    coords_bind_ms = timed(lambda: (setattr(small, "_bound", None), small.bind(pcs[:k], mk.exp(l))), 3)
    return {"config": 5, "workload": f"SpaGCN SimpleGCDEC {n} spots × {G} genes → 50 PCs, adjacency from the spot coordinates "
                                     "(SpotDistance, no N×N matrix), one GPU",
            "metric": "spots/sec per training epoch", "value": n / (epoch_ms / 1e3), "unit": "spots/s", "ms_per_epoch": epoch_ms,
            "calculate_p_ms": p_ms, "adj_x_build_ms": bind_ms, "refine_ms": refine_ms, "ax_check_max_err_over_2^-21": ax_ratio,
            f"bind_{k}_dense_ms": dense_bind_ms, f"bind_{k}_coords_ms": coords_bind_ms,
            "dtype": "f32 (tf32x3 weighted product)", "n_gpus": 1, "data": "synthetic", "card": _card()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", type=str, default="1,3,5")
    ap.add_argument("--cells3", type=int, default=500_000)
    ap.add_argument("--spots", type=int, default=20_000)
    ap.add_argument("--precision3", choices=sorted(DTYPE3), default="bf16", help="GEMM precision of config 3")
    ap.add_argument("--adjacency", choices=("dense", "coords"), default="dense", help="config 5: dense N×N adjacency or spot coordinates")
    args = ap.parse_args()
    fns = {"1": config1, "3": config3, "5": config5 if args.adjacency == "dense" else config5_coords}
    for k in args.only.split(","):
        try:
            print(json.dumps(fns[k.strip()](args)), flush=True)
        except Exception as ex:     # one failing configuration must not hide the others
            print(json.dumps({"config": int(k), "error": f"{type(ex).__name__}: {ex}"}), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
