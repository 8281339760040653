"""graph-sc (GraphSC) training throughput through the public model API: one JSON line.

Synthetic counts (dance_b200.synth through the dataset loader) go through normalize_total / log1p and
``PCACellFeatureGraph(50, normalize_edges=True, feat_norm_mode="standardize")``, then the default ``GraphSC()`` trains with batch
128.  Two sizes: 4 271 cells × 3 000 genes (the 10X PBMC example's size) and 100 000 cells × 3 000 genes.  Reported per size:
ms per epoch from device events after a warm-up epoch, the kernel launches per mini-batch, and the device time of each new entry
point (CUDA events around every call, measured in a separate epoch); plus the card's name and power limit.

    python benchmarks/graphsc.py [--cells 4271,100000] [--epochs 3]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

NEW = ("graphsc_block_degrees", "graphsc_block_aggregate_f32", "graphsc_batch_decoder_f32", "act_bwd_f32", "graphsc_scatter_rows_f32")


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in out.split(","))
        return name, power
    except Exception:       # noqa: BLE001  (the name still comes from torch)
        return torch.cuda.get_device_name(), "unknown"


def run(n_cells: int, epochs: int, tmp: str):
    os.environ["DANCE_B200_SYNTH"] = f"cells={n_cells},genes=3000,types=10"
    from dance_b200 import ops
    from dance_b200.datasets import CellTypeAnnotationDataset
    from dance_b200.modules.graphsc import GraphSC
    from dance_b200.transforms import AnnDataTransform, Compose
    from dance_b200.transforms.graph import PCACellFeatureGraph
    pipeline = Compose(AnnDataTransform("scanpy.pp.normalize_total"), AnnDataTransform("scanpy.pp.log1p"),
                       PCACellFeatureGraph(50, normalize_edges=True, feat_norm_mode="standardize"), log_level="WARNING")
    data = CellTypeAnnotationDataset(species="synthetic", tissue="tissue", data_dir=f"{tmp}/{n_cells}").load_data(transform=pipeline)
    g = data.data.uns["CellFeatureGraph"]
    torch.manual_seed(0)
    model = GraphSC(device="cuda")
    model.fit(g, epochs=1)                                                  # warm-up
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    model.fit(g, epochs=epochs)
    e.record()
    torch.cuda.synchronize()
    ms = s.elapsed_time(e) / epochs
    n_batches = -(-n_cells // 128)
    ops.reset_counters()
    model.fit(g, epochs=1)
    torch.cuda.synchronize()
    launches = ops.counters()["launches"] / n_batches
    ops.enable_kernel_timing(True)
    model.fit(g, epochs=1)
    times = ops.kernel_times()
    ops.enable_kernel_timing(False)
    kernels = {k: {"ms_per_batch": v["ms"] / n_batches, "calls_per_batch": v["n"] / n_batches} for k, v in times.items() if k in NEW}
    return {"cells": n_cells, "genes": 3000, "edges": int(g.number_of_edges()), "batches": n_batches, "ms_per_epoch": ms,
            "launches_per_batch": launches, "new_kernels": kernels}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=str, default="4271,100000")
    ap.add_argument("--epochs", type=int, default=3)
    args = ap.parse_args()
    name, power = _card()
    with tempfile.TemporaryDirectory(prefix="b2_graphsc_") as tmp:
        sizes = [run(int(n), args.epochs, tmp) for n in args.cells.split(",")]
    print(json.dumps({"workload": "GraphSC() default (agg sum, 1 layer, hidden 200 → 300, dropout 0.1), batch 128, lr 1e-5",
                      "metric": "ms per training epoch", "sizes": sizes, "dtype": "f32 (tf32x3 GEMMs)", "card": name,
                      "power_limit": power, "data": "synthetic"}), flush=True)


if __name__ == "__main__":
    main()
