"""Tensor-core GEMM (ops.gemm) in tf32x3, tf32 and bf16 on the GraphSCI and Feature-AE shapes.  One JSON line per shape and
precision: ms per call, achieved TFLOP/s from 2·M·N·K, and that rate as a share of the H100 SXM data-sheet dense peak of the
type (989 TFLOP/s bf16, 495 tf32, 495/3 for tf32x3's three products).  The precisions are timed alternately, several rounds,
with CUDA events around `--iters` back-to-back calls; the reported ms is the median over rounds.  The first line names the
card and its power limit, read in the same run.  `--dump-outputs DIR` also writes each shape's C per precision as
DIR/<shape>.<precision>.npy, so that two builds can be compared element by element.

    python benchmarks/gemm.py [--iters 20] [--rounds 5] [--dump-outputs DIR]
"""
from __future__ import annotations

import argparse
import json
import re
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

PEAK = {"bf16": 989.0, "tf32": 495.0, "tf32x3": 495.0 / 3}
PRECISIONS = ("tf32x3", "tf32", "bf16")

# name, M, N, K, transA, transB
SHAPES = [
    ("graphsci X·zf", 100_000, 3000, 3000, False, False),
    ("graphsci X_dᵀ·dpre0", 3000, 3000, 100_000, True, False),
    ("graphsci f_d·W_conv1", 3000, 256, 100_000, False, False),
    ("feature-ae fc1 fwd", 12_800, 512, 2000, False, True),
    ("feature-ae fc1 wgrad (split-K)", 512, 2000, 12_800, True, False),
]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as ex:
        q = f"unavailable ({type(ex).__name__})"
    return {"gpu": name, "power_limit, max_sm_clock": q}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--dump-outputs", metavar="DIR", help="write C of every shape and precision here as .npy")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("benchmarks/gemm.py needs a CUDA device")
    from dance_b200 import ops
    dev = torch.device("cuda:0")
    print(json.dumps(card()), flush=True)
    g = torch.Generator(device=dev).manual_seed(0)
    for name, M, N, K, tA, tB in SHAPES:
        A = torch.randn((K, M) if tA else (M, K), device=dev, generator=g)
        B = torch.randn((N, K) if tB else (K, N), device=dev, generator=g)
        C = torch.empty(M, N, device=dev)
        ws = {p: int(ops.lib().b2_gemm_workspace_bytes(M, N, K, int(tA), int(tB), ops.PREC[p])) for p in PRECISIONS}
        for p in PRECISIONS:                                   # warm-up: module load, workspace allocation
            for _ in range(2):
                ops.gemm(A, B, transA=tA, transB=tB, out=C, precision=p)
        torch.cuda.synchronize()
        times = {p: [] for p in PRECISIONS}
        for _ in range(args.rounds):
            for p in PRECISIONS:
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                for _ in range(args.iters):
                    ops.gemm(A, B, transA=tA, transB=tB, out=C, precision=p)
                e.record()
                e.synchronize()
                times[p].append(s.elapsed_time(e) / args.iters)
        flop = 2.0 * M * N * K
        for p in PRECISIONS:
            t = sorted(times[p])
            ms = t[len(t) // 2]
            tflops = flop / (ms * 1e-3) / 1e12
            print(json.dumps({"shape": name, "M": M, "N": N, "K": K, "transA": tA, "transB": tB, "precision": p,
                              "ms": round(ms, 4), "ms_min": round(t[0], 4), "ms_max": round(t[-1], 4),
                              "tflops": round(tflops, 1), "share_of_peak": round(tflops / PEAK[p], 3), "peak_tflops": round(PEAK[p], 1),
                              "split_k_workspace_bytes": ws[p]}), flush=True)
        if args.dump_outputs:
            out = Path(args.dump_outputs)
            out.mkdir(parents=True, exist_ok=True)
            slug = re.sub(r"[^0-9A-Za-z]+", "_", name).strip("_")
            for p in PRECISIONS:
                ops.gemm(A, B, transA=tA, transB=tB, out=C, precision=p)
                np.save(out / f"{slug}.{p}.npy", C.cpu().numpy())
        del A, B, C
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
