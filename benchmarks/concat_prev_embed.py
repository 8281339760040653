"""Time the pieces of scGNN's ``*_concat_prev_embed`` at 1 M cells × 2 000 genes.

  "quantiles"  ops.quantiles(X, (0.9, 0.1)): the radix select's three histogram passes over the N×G expression matrix, against
               its HBM floor (three reads of X at 3.35 TB/s, the H100 SXM data-sheet bandwidth);
  "widen"      the fused widen kernel (b2_concat_scaled_f32, scaled): reads X and the 16-d embedding, writes the row-padded
               N×(G+16) matrix, against its own floor;
  "normalize"  ops.concat_normalized end to end (quantiles, column min / max, one synchronisation, widen);
  "feature_ae" one Feature-AE epoch (batch 12 800, "noregu") at G, G+16 and G+128 input columns;
  "knn"        the exact kNN (k = 10) of the N×128 embedding and of the widened N×144 one.
Prints the card (name, power limit), then one JSON line per measurement with median and minimum times in ms."""
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
from dance_b200.engine import FeatureAEEngine  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


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


def repeat(fn, steps, warmup):
    ts = []
    for it in range(warmup + steps):
        t, _ = timed(fn)
        if it >= warmup:
            ts.append(t)
    return np.array(ts)


def report(what, ts, **extra):
    line = {"what": what, "ms": round(float(np.median(ts)), 3), "ms_min": round(float(ts.min()), 3), "steps": len(ts)}
    line.update(extra)
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--genes", type=int, default=2000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--batch", type=int, default=12800)
    ap.add_argument("--knn-steps", type=int, default=1)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    dev = torch.device("cuda:0")
    print(json.dumps({"card": card()}), flush=True)
    n, G = args.n, args.genes
    gen = torch.Generator(device=dev).manual_seed(0)
    # log1p counts, about 90 % zeros, like a filtered scRNA-seq matrix
    X = torch.rand(n, G, device=dev, generator=gen)
    X = torch.where(X < 0.9, torch.zeros((), device=dev), torch.log1p(X * 20.0))
    ge = torch.randn(n, 16, device=dev, generator=gen)
    fe = torch.relu(torch.randn(n, 128, device=dev, generator=gen))
    xbytes = X.numel() * 4

    ts = repeat(lambda: ops.quantiles(X, (0.9, 0.1)), args.steps, args.warmup)
    floor = 3 * xbytes / HBM_BYTES_PER_S * 1e3
    report("quantiles", ts, n=n, genes=G, elements=X.numel(), hbm_floor_ms=round(floor, 3),
           floor_fraction=round(floor / float(np.median(ts)), 3), values=[float(v) for v in ops.quantiles(X, (0.9, 0.1))])

    cmin, cmax = ops.col_minmax(ge)
    pitch = (G + 16 + 3) // 4 * 4
    out = torch.empty(n, pitch, device=dev)
    lib = ops.lib()
    ws = torch.empty(lib.b2_concat_scaled_workspace_bytes(16), dtype=torch.uint8, device=dev)

    def widen():
        ops._call("b2_concat_scaled_f32", X.data_ptr(), G, G, ge.data_ptr(), 16, 16, n, cmin.data_ptr(), cmax.data_ptr(), 0.0, 1.0, 1,
                  out.data_ptr(), pitch, ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
    ts = repeat(widen, args.steps, args.warmup)
    wbytes = xbytes + ge.numel() * 4 + out.numel() * 4
    floor = wbytes / HBM_BYTES_PER_S * 1e3
    report("widen", ts, bytes=wbytes, hbm_floor_ms=round(floor, 3), floor_fraction=round(floor / float(np.median(ts)), 3))
    del out
    ts = repeat(lambda: ops.concat_normalized(X, ge, base=X), args.steps, args.warmup)
    report("normalize", ts, width=G + 16)

    for e, right in ((0, None), (16, ge), (128, fe)):
        Xw = X if right is None else ops.concat_normalized(X, right, base=X if e == 16 else None)
        eng = FeatureAEEngine(Xw.shape[1], device=dev, seed=0)

        def epoch():
            for b0 in range(0, n, args.batch):
                xb = Xw[b0:b0 + args.batch]
                eng.train_step(xb if xb.is_contiguous() else xb.contiguous(), None, 0.9, "noregu")
        ts = repeat(epoch, max(1, args.steps // 2), args.warmup)
        report("feature_ae_epoch", ts, input_columns=Xw.shape[1], row_pitch=Xw.stride(0), batch=args.batch)
        del Xw, eng
        torch.cuda.empty_cache()

    emb = torch.relu(torch.randn(n, 128, device=dev, generator=gen))
    for d, xe in ((128, emb), (144, ops.concat_normalized(emb, ge, base=emb))):
        ts = repeat(lambda: ops.knn(xe, 10), args.knn_steps, 1)
        report("knn", ts, dim=d, k=10)


if __name__ == "__main__":
    main()
