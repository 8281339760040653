"""Time the exact all-pairs Graph-AE decoder (ops.gae_loss_grad, tensor-core path) at n cells for d = 8, 16 and 32.

CUDA events around each call after a warm-up; prints one JSON line per d with the median and minimum time, the logits per
second (n², every ordered pair) and the fraction of the SFU floor reached.  The floor: the kernel issues 64 ex2 + 64 rcp +
3 lg2 per 64 logits, and an SM completes 16 MUFU results per clock, so it cannot exceed 16 / (131 / 64) logits per clock per
SM at the card's reported maximum SM clock.  The card name, its power limit and that clock are printed with the numbers."""
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

MUFU_PER_LOGIT = (64 + 64 + 3) / 64
MUFU_PER_CLK_SM = 16


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True,
                         text=True, check=True).stdout.strip().split(", ")
    return {"name": out[0], "power_limit_w": float(out[1]), "max_sm_clock_mhz": float(out[2])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--d", type=str, default="8,16,32")
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the decoder benchmark needs a CUDA device"
    dev = torch.device("cuda:0")
    info = card()
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    floor = sms * info["max_sm_clock_mhz"] * 1e6 * MUFU_PER_CLK_SM / MUFU_PER_LOGIT
    print(json.dumps({"card": info, "sms": sms, "sfu_floor_logits_per_s": floor}))
    n = args.n
    gen = torch.Generator(device=dev).manual_seed(0)
    idx = torch.randint(0, n, (n, 10), device=dev, dtype=torch.int32, generator=gen)
    A = ops.knn_graph_build(idx.contiguous())
    L = ops.CSR(A.rowptr, A.colidx, None, A.shape)
    ops.set_path("gae", "tc")
    try:
        for d in (int(x) for x in args.d.split(",")):
            z = (torch.randn(n, d, device=dev, generator=gen) * 0.3).contiguous()
            for _ in range(args.warmup):
                ops.gae_loss_grad(z, L, 0.5, 50.0)
            torch.cuda.synchronize()
            ts = []
            for _ in range(args.iters):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                loss, _, _, _ = ops.gae_loss_grad(z, L, 0.5, 50.0)
                e.record()
                e.synchronize()
                ts.append(s.elapsed_time(e))
            ms = float(np.median(ts))
            rate = float(n) * n / (ms * 1e-3)
            print(json.dumps({"kernel": "gae_loss_grad", "n": n, "d": d, "ms": round(ms, 2), "ms_min": round(min(ts), 2),
                              "logits_per_s": rate, "sfu_floor_fraction": round(rate / floor, 3),
                              "loss": float(loss.item())}))
    finally:
        ops.set_path("gae", "auto")


if __name__ == "__main__":
    main()
