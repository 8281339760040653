"""Time the exact all-pairs Graph-AE decoder (ops.gae_loss_grad, tensor-core path) at n cells for d = 8, 16 and 32.

CUDA events around each call after a warm-up; prints one JSON line per d and kernel with the median and minimum time, the
ordered pairs per second (n², what the loss covers) and the logits the kernel evaluates per second with their fraction of the
SFU floor (and, for the triangle, of the tensor-instruction floor).  Two kernels run on the same z:
  "triangle"    the call over all rows (gae_tri_tc_kernel): each block sweeps the 64-column J tiles from its own 128-row
                block on, so it evaluates about n²/2 logits plus the diagonal blocks; S in tf32, the gradient products in fp16;
  "full_sweep"  the same rows as two row-shard calls (gae_allpairs_tc_kernel): every row against every column, n² logits
                (rounded up to whole 128-column tiles).
The SFU floor: the triangle issues 32 ex2 + 32 rcp + 2 lg2 per 32 logits, the full sweep 64 + 64 + 3 per 64, and an SM
completes 16 MUFU results per clock, so neither can exceed 16 / (MUFU per logit) logits per clock per SM at the card's reported
maximum SM clock.  The tensor-instruction floor: per 128 x 64 triangle tile (8 192 logits) the two consumer warpgroups issue
2 x 3·DP/8 S products m64n64k8 (32 clocks each), 2 x 4 dZ_I products m64n(2·DP)k16 + m64nDPk16 and the dZ_J warpgroup
2 x the same from shared memory; the clocks per instruction are those benchmarks/wgmma_rate.py measured at two warpgroups
(RS: 13 / 16 / 32 clocks at N = 16 / 32 / 64, SS: 20 / 24 / 32, N = 8 taken as N = 16).  The card name, its power limit and that clock are printed with the numbers."""
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

MUFU_PER_LOGIT = {"triangle": (32 + 32 + 2) / 32, "full_sweep": (64 + 64 + 3) / 64}
MUFU_PER_CLK_SM = 16
RS_CLK = {8: 13, 16: 13, 32: 16, 64: 32}
SS_CLK = {8: 20, 16: 20, 32: 24, 64: 32}


def tensor_clocks_per_tile(dp: int) -> int:
    """tensor-pipe clocks of one 128 x 64 triangle tile above the diagonal block (see the module docstring)"""
    k = 4                                          # fp16 k16 steps over 64 columns
    s = 2 * (3 * dp // 8) * 32
    dzi = 2 * k * (RS_CLK[2 * dp] + RS_CLK[dp])
    dzj = 2 * k * (SS_CLK[2 * dp] + SS_CLK[dp])
    return s + dzi + dzj


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True,
                         text=True, check=True).stdout.strip().split(", ")
    return {"name": out[0], "power_limit_w": float(out[1]), "max_sm_clock_mhz": float(out[2])}


def evaluated_logits(n: int, kernel: str) -> int:
    """Logits the kernel computes, padding included: 128-row blocks against whole J tiles."""
    nb = -(-n // 128)
    if kernel == "full_sweep":
        return (nb * 128) ** 2
    cols = -(-n // 64) * 64                  # block I sweeps the 64-column tiles from column 128·I to the last one
    return sum(128 * (cols - 128 * i) for i in range(nb))


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        out = fn()
        e.record()
        e.synchronize()
        ts.append(s.elapsed_time(e))
    return ts, out


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
    floor = {k: sms * info["max_sm_clock_mhz"] * 1e6 * MUFU_PER_CLK_SM / m for k, m in MUFU_PER_LOGIT.items()}
    print(json.dumps({"card": info, "sms": sms, "sfu_floor_logits_per_s": floor}))
    n = args.n
    gen = torch.Generator(device=dev).manual_seed(0)
    idx = torch.randint(0, n, (n, 10), device=dev, dtype=torch.int32, generator=gen)
    A = ops.knn_graph_build(idx.contiguous())
    L = ops.CSR(A.rowptr, A.colidx, None, A.shape)
    # the same rows as two row shards, split at a block boundary near the middle
    h = (n // 2) // 128 * 128
    rp = A.rowptr.long()
    top = ops.CSR(A.rowptr[:h + 1].contiguous(), A.colidx[:rp[h]].contiguous(), None, (h, n))
    bot = ops.CSR((A.rowptr[h:] - A.rowptr[h]).contiguous(), A.colidx[rp[h]:].contiguous(), None, (n - h, n))
    ops.set_path("gae", "tc")
    try:
        for d in (int(x) for x in args.d.split(",")):
            z = (torch.randn(n, d, device=dev, generator=gen) * 0.3).contiguous()
            runs = {
                "triangle": lambda: ops.gae_loss_grad(z, L, 0.5, 50.0)[0],
                "full_sweep": lambda: ops.gae_loss_grad(z, top, 0.5, 50.0, row_begin=0, n_rows=h)[0]
                + ops.gae_loss_grad(z, bot, 0.5, 50.0, row_begin=h, n_rows=n - h)[0],
            }
            for kernel, fn in runs.items():
                ts, loss = timed(fn, args.iters, args.warmup)
                ms = float(np.median(ts))
                evaluated = evaluated_logits(n, kernel) / (ms * 1e-3)
                row = {"kernel": kernel, "n": n, "d": d, "ms": round(ms, 2), "ms_min": round(min(ts), 2),
                       "pairs_per_s": float(n) * n / (ms * 1e-3), "evaluated_logits_per_s": evaluated,
                       "sfu_floor_fraction": round(evaluated / floor[kernel], 3), "loss": float(loss.item())}
                if kernel == "triangle":
                    dp = 8 if d <= 8 else 16 if d <= 16 else 32
                    tensor_floor = sms * info["max_sm_clock_mhz"] * 1e6 * 8192 / tensor_clocks_per_tile(dp)
                    row["tensor_floor_fraction"] = round(evaluated / tensor_floor, 3)
                print(json.dumps(row))
    finally:
        ops.set_path("gae", "auto")


if __name__ == "__main__":
    main()
