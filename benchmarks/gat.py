"""Time GATEngine.train_step (scGNN's GAT Graph-AE, one epoch of graph_AE_handler) with and without GATLayer's dropout.

Two engines with the same weights, dropout 0 and --p, take turns step by step on the same graph, so both see the same card
state.  CUDA events split every step into
  "decoder"  the plain-BCE all-pairs decoder (ops.gae_loss_grad on z zᵀ), and
  "encoder"  everything else: both GAT layers forward and backward (with the dropout draws when p > 0) and Adam.
Default size: 1 M cells with 128 input features (the Feature-AE embedding), each sending k = 15 edges to uniformly random
targets, 2 heads, hidden 64, embedding 16.  Prints the card (name, power limit) and one JSON line per p with the median and
minimum times, then the encoder overhead of dropout."""
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
from dance_b200.engine import GATEngine  # noqa: E402


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True,
                         text=True, check=True).stdout.strip().split(", ")
    return {"name": out[0], "power_limit_w": float(out[1]), "max_sm_clock_mhz": float(out[2])}


class _DecoderTimer:
    """Wraps ops.gae_loss_grad (the engine calls it through the module) with CUDA events."""

    def __init__(self):
        self.inner, self.events = ops.gae_loss_grad, []

    def __call__(self, *a, **kw):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        out = self.inner(*a, **kw)
        e.record()
        self.events.append((s, e))
        return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--k", type=int, default=15)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--heads", type=int, default=2)
    ap.add_argument("--hid", type=int, default=64)
    ap.add_argument("--emb", type=int, default=16)
    ap.add_argument("--p", type=float, default=0.3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the GAT benchmark needs a CUDA device"
    dev = torch.device("cuda:0")
    print(json.dumps({"card": card()}))
    n, k = args.n, args.k
    gen = torch.Generator(device=dev).manual_seed(0)
    x = (torch.rand(n, args.dim, device=dev, generator=gen) * 0.1).contiguous()
    idx = torch.randint(0, n, (n, k), device=dev, dtype=torch.int32, generator=gen)
    src_csr = ops.CSR(torch.arange(0, n * k + 1, k, dtype=torch.int32, device=dev), idx.reshape(-1).contiguous(), None, (n, n))
    T, _ = ops.csr_transpose(src_csr)                     # rows = targets
    Tt, t_perm = ops.csr_transpose(T)
    A = ops.knn_graph_build(idx)
    labels = ops.CSR(A.rowptr, A.colidx, None, A.shape)
    engines = {p: GATEngine(args.dim, args.hid, args.emb, args.heads, device=dev, seed=0, dropout=p) for p in (0.0, args.p)}
    timer = _DecoderTimer()
    ops.gae_loss_grad = timer
    times = {p: {"step": [], "decoder": []} for p in engines}
    try:
        for it in range(args.warmup + args.steps):
            for p, eng in engines.items():
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                timer.events.clear()
                s.record()
                eng.train_step(x, T, Tt, t_perm, labels)
                e.record()
                e.synchronize()
                if it >= args.warmup:
                    times[p]["step"].append(s.elapsed_time(e))
                    times[p]["decoder"].append(sum(a.elapsed_time(b) for a, b in timer.events))
    finally:
        ops.gae_loss_grad = timer.inner
    enc = {}
    for p, t in times.items():
        step, dec = np.array(t["step"]), np.array(t["decoder"])
        enc[p] = step - dec
        print(json.dumps({"p": p, "n": n, "k": k, "heads": args.heads, "hid": args.hid, "emb": args.emb, "steps": args.steps,
                          "step_ms": round(float(np.median(step)), 2), "step_ms_min": round(float(step.min()), 2),
                          "encoder_ms": round(float(np.median(enc[p])), 2), "encoder_ms_min": round(float(enc[p].min()), 2),
                          "decoder_ms": round(float(np.median(dec)), 2), "loss": float(engines[p].loss.item())}))
    base, drop = float(np.median(enc[0.0])), float(np.median(enc[args.p]))
    print(json.dumps({"encoder_overhead_ms": round(drop - base, 2), "encoder_overhead_fraction": round(drop / base - 1, 4)}))


if __name__ == "__main__":
    main()
