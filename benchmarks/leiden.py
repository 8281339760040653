"""Leiden on the device (``dance_b200.leiden``) on the neighbour graph of a synthetic 10-cluster Gaussian mixture Z[N, dims]
(SURVEY §8(d); dims = 50 by default, 300 is graph-sc's embedding): one JSON line per (N, γ).

Reported separately, each from device events around a synchronised call after a warm-up run of the same size: the exact kNN
(``n_neighbors`` = 10 by default, the cell itself included; graph-sc's Leiden uses 300), the UMAP connectivities and Leiden; and
Leiden's levels, iterations, communities and quality (Q / W), and the peak device memory torch allocated for the size.  At γ = 1
the existing host Louvain (``ops.louvain_host``) runs on the same graph as a
reference point.  The card's name and power limit are read in the same run.

    python benchmarks/leiden.py [--cells 200000,1000000] [--resolutions 0.4,1.0] [--n_neighbors 10] [--dims 50]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in out.split(","))
        return name, power
    except Exception:       # noqa: BLE001  (the name still comes from torch)
        return torch.cuda.get_device_name(), "unknown"


def mixture(n: int, d: int = 50, clusters: int = 10, seed: int = 0) -> torch.Tensor:
    g = torch.Generator(device="cuda").manual_seed(seed)
    centres = torch.randn(clusters, d, generator=g, device="cuda") * 4.0
    which = torch.randint(0, clusters, (n, ), generator=g, device="cuda")
    return (centres[which] + torch.randn(n, d, generator=g, device="cuda")).contiguous()


def timed(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    out = fn()
    e.record()
    torch.cuda.synchronize()
    return out, s.elapsed_time(e)


def run(n: int, resolutions, n_neighbors: int, card, dims: int = 50):
    from dance_b200 import ops
    from dance_b200.leiden import leiden
    torch.cuda.reset_peak_memory_stats()
    Z = mixture(n, dims)
    ops.knn(Z, n_neighbors, include_rank0=True)                      # warm-up at this size
    (idx, dist), t_knn = timed(lambda: ops.knn(Z, n_neighbors, include_rank0=True))
    ops.umap_connectivities(idx, dist.float())
    A, t_conn = timed(lambda: ops.umap_connectivities(idx, dist.float()))
    rows = []
    for gamma in resolutions:
        leiden(A, resolution=gamma)
        res, t_leiden = timed(lambda: leiden(A, resolution=gamma))
        row = {"bench": "leiden", "cells": n, "dims": Z.shape[1], "n_neighbors": n_neighbors, "nnz": A.nnz, "resolution": gamma,
               "knn_ms": round(t_knn, 2), "connectivities_ms": round(t_conn, 2), "leiden_ms": round(t_leiden, 2),
               "levels": res.levels, "iterations": res.iterations, "communities": res.n_communities,
               "quality": round(res.quality, 6), "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2**30, 2),
               "card": card[0], "power_limit": card[1]}
        if gamma == 1.0:
            S = A.to_scipy()
            t0 = time.perf_counter()
            _, nc, mod = ops.louvain_host(S.indptr, S.indices, S.data)
            row.update(louvain_host_ms=round((time.perf_counter() - t0) * 1e3, 1), louvain_host_communities=nc,
                       louvain_host_modularity=round(mod, 6))
        rows.append(row)
        print(json.dumps(row), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", default="200000,1000000")
    ap.add_argument("--resolutions", default="0.4,1.0")
    ap.add_argument("--n_neighbors", type=int, default=10)
    ap.add_argument("--dims", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("benchmarks/leiden.py needs a CUDA device")
    card = _card()
    for n in (int(c) for c in args.cells.split(",")):
        run(n, [float(r) for r in args.resolutions.split(",")], args.n_neighbors, card, args.dims)


if __name__ == "__main__":
    main()
