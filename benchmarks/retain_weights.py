"""Time scGNN's Graph-AE with and without ``graph_AE_retain_weights`` at 1 M cells.

From one exact kNN (k = 15) of a clustered embedding:
  "build"    the union-symmetrised 0/1 graph (ops.knn_graph_build) and the weighted, directed graph (ops.knn_graph_weighted_build);
  "step"     GraphAEEngine.train_step on each graph (GCN branch, embedding 16, 128 input features);
  "decoder"  ops.gae_loss_grad with each label matrix, split into the all-pairs part (the same call with an empty label matrix)
             and the edge pass(es) (the difference): one pass over L for unit labels, one over L and one over Lᵀ for weighted ones.
Both configurations alternate step by step on the same card.  Prints the card (name, power limit), then one JSON line per
configuration with median and minimum times in ms."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from dance_b200 import ops  # noqa: E402
from dance_b200.engine import GraphAEEngine  # noqa: E402


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True,
                         text=True, check=True).stdout.strip().split(", ")
    return {"name": out[0], "power_limit_w": float(out[1]), "max_sm_clock_mhz": float(out[2])}


def timed(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    out = fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--k", type=int, default=15)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--emb", type=int, default=16)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    dev = torch.device("cuda:0")
    print(json.dumps({"card": card()}))
    n, k = args.n, args.k
    gen = torch.Generator(device=dev).manual_seed(0)
    centres = torch.randn(10, args.dim, device=dev, generator=gen)
    X = (torch.rand(n, args.dim, device=dev, generator=gen) * 0.1 + centres[torch.randint(0, 10, (n, ), device=dev, generator=gen)].abs() * 0.05)
    X = X.contiguous()
    idx, dist = ops.knn(X, k)
    build = {"plain": [], "weighted": []}
    for it in range(args.warmup + args.steps):
        t0, A = timed(lambda: ops.knn_graph_build(idx))
        t1, wg = timed(lambda: ops.knn_graph_weighted_build(idx, dist))
        if it >= args.warmup:
            build["plain"].append(t0)
            build["weighted"].append(t1)
    n_lab = A.nnz - n
    sum_w = wg.sum_w.item()
    configs = {
        "plain": dict(adj=A, adj_t=None, labels=ops.CSR(A.rowptr, A.colidx, None, A.shape), labels_t=None, sum_w=float(n_lab)),
        "weighted": dict(adj=wg.adj, adj_t=wg.adj_t, labels=wg.labels, labels_t=wg.labels_t, sum_w=sum_w),
    }
    empty = ops.CSR(torch.zeros(n + 1, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int32, device=dev), None, (n, n))
    eps = torch.randn(n, args.emb, device=dev, generator=gen)
    engines = {c: GraphAEEngine(args.dim, args.emb, device=dev, seed=0) for c in configs}
    times = {c: {"step": [], "decoder": [], "allpairs": []} for c in configs}
    for it in range(args.warmup + args.steps):
        for c, cfg in configs.items():
            pw = float(n * n - cfg["sum_w"]) / cfg["sum_w"]
            norm = n * n / float((n * n - cfg["sum_w"]) * 2)
            eng = engines[c]
            t_step, (z, mu, lv) = timed(lambda: eng.train_step(X, cfg["adj"], cfg["labels"], norm, pw, eps, adj_t=cfg["adj_t"],
                                                               labels_t=cfg["labels_t"]))
            z = z.clone()
            t_dec, _ = timed(lambda: ops.gae_loss_grad(z, cfg["labels"], norm, pw, mu, lv, labels_t=cfg["labels_t"]))
            t_ap, _ = timed(lambda: ops.gae_loss_grad(z, empty, norm, pw, mu, lv))
            if it >= args.warmup:
                times[c]["step"].append(t_step)
                times[c]["decoder"].append(t_dec)
                times[c]["allpairs"].append(t_ap)
    for c, t in times.items():
        step, dec, ap_ = (np.array(t[key]) for key in ("step", "decoder", "allpairs"))
        edges = dec - ap_
        print(json.dumps({"config": c, "n": n, "k": k, "emb": args.emb, "steps": args.steps, "label_entries": configs[c]["labels"].nnz,
                          "build_ms": round(float(np.median(build[c])), 2), "build_ms_min": round(float(np.min(build[c])), 2),
                          "step_ms": round(float(np.median(step)), 2), "step_ms_min": round(float(step.min()), 2),
                          "decoder_ms": round(float(np.median(dec)), 2), "allpairs_ms": round(float(np.median(ap_)), 2),
                          "edges_ms": round(float(np.median(edges)), 3), "edges_fraction_of_decoder": round(float(np.median(edges / dec)), 5),
                          "loss": float(engines[c].loss.item())}))


if __name__ == "__main__":
    main()
