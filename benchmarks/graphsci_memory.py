"""Time and peak device memory of GraphSCI's two training schedules on configuration 3's data (bf16 GEMMs, dropout 0.1).

  * at --small cells (default 200 000): the materialising and the lean schedule, alternated --repeats times in this one
    process, each from a fresh model (2 warm-up epochs, then --epochs timed with CUDA events);
  * at --large cells (default 500 000): the schedule GraphSCI chooses by itself ("auto").

Each line reports ms per epoch and torch.cuda.max_memory_allocated() from the model's creation to the last epoch (the
caller's X, Xraw, Xᵀ and mask included); the first line names the card and its power limit.

    python benchmarks/graphsci_memory.py [--small 200000] [--large 500000] [--repeats 2] [--epochs 3] [--out results.jsonl]
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from configs import _card, config3_data, config3_model  # noqa: E402

COEF = dict(le=1, la=1e-9, ke=1e2, ka=1)


def run(N, schedule, X, Xraw, graph, tm, epochs, precision):
    from dance_b200.modules import graphsci
    graphsci.SCHEDULE = schedule
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    model = config3_model(N, X.shape[1], X, Xraw, graph, precision)
    for _ in range(2):
        model.train(X, Xraw, graph, tm, tm, **COEF)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(epochs):
        model.train(X, Xraw, graph, tm, tm, **COEF)
    e.record()
    torch.cuda.synchronize()
    out = {"cells": N, "genes": X.shape[1], "requested": schedule, "schedule": model.schedule(), "ms_per_epoch": s.elapsed_time(e) / epochs,
           "peak_memory_gib": torch.cuda.max_memory_allocated() / 2**30, "train_loss": model.train_loss, "valid_loss": model.valid_loss,
           "precision": precision, "dropout": model.dropout}
    graphsci.SCHEDULE = "auto"
    del model
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--small", type=int, default=200_000)
    ap.add_argument("--large", type=int, default=500_000)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--precision", default="bf16")
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    lines = [{"card": _card(), "total_memory_gib": torch.cuda.get_device_properties(0).total_memory / 2**30}]
    print(json.dumps(lines[-1]), flush=True)
    for N, schedules in ((args.small, ["materialise", "lean"] * args.repeats), (args.large, ["auto"])):
        if N <= 0:
            continue
        X, Xraw, graph = config3_data(N)
        tm = torch.ones(X.shape, dtype=torch.uint8, device=X.device)
        for sch in schedules:
            lines.append(run(N, sch, X, Xraw, graph, tm, args.epochs, args.precision))
            print(json.dumps(lines[-1]), flush=True)
        del X, Xraw, graph, tm
        torch.cuda.empty_cache()
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text("".join(json.dumps(x) + "\n" for x in lines))


if __name__ == "__main__":
    main()
