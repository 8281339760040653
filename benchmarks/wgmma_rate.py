"""Clocks per wgmma on the card at the decoder's small-N shapes: tf32 m64nNk8 against f16 m64nNk16, A from shared memory (ss)
or from registers (rs), N = 16 / 32 / 64, one and two warpgroups per CTA (one CTA per SM).

Compiles benchmarks/wgmma_rate.cu with nvcc for sm_90a into a temporary directory and runs it.  Prints the card (name, power
limit, maximum SM clock), one JSON line per shape, then for each form and N the ratio of an f16 k16 instruction to two tf32 k8
instructions at two warpgroups.  An f16 k16 product covers the K of two tf32 k8 products, so a ratio clearly below 1 (below
about 0.8, i.e. one f16 instruction under 1.6 tf32 ones) means the decoder's gradient products get cheaper as f16 hi / lo
products; a ratio near 1 means the tensor pipe is bound by MACs at these shapes and halving the instruction count buys
nothing."""
from __future__ import annotations

import json
import shutil
import subprocess
import sys
import tempfile
from pathlib import Path

SRC = Path(__file__).resolve().parent / "wgmma_rate.cu"


def card():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True,
                         text=True, check=True).stdout.strip().split(", ")
    return {"name": out[0], "power_limit_w": float(out[1]), "max_sm_clock_mhz": float(out[2])}


def main():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    info = card()
    print(json.dumps({"card": info}))
    with tempfile.TemporaryDirectory() as tmp:
        exe = Path(tmp) / "wgmma_rate"
        subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-o", str(exe), str(SRC)],
                       check=True)
        out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout
    rows = {}
    for line in out.split("\n"):
        if not line.strip():
            continue
        dtype, form, n, wgs, per_wg, per_sm, mhz = line.split()
        r = {"dtype": dtype, "form": form, "n": int(n), "warpgroups": int(wgs), "clocks_per_wgmma_per_warpgroup": float(per_wg),
             "clocks_per_wgmma_per_sm": float(per_sm), "sm_clock_mhz": float(mhz)}
        rows[(dtype, form, int(n), int(wgs))] = r
        print(json.dumps(r))
    for form in ("ss", "rs"):
        for n in (16, 32, 64):
            f16 = rows[("f16", form, n, 2)]["clocks_per_wgmma_per_sm"]
            tf32 = rows[("tf32", form, n, 2)]["clocks_per_wgmma_per_sm"]
            print(json.dumps({"form": form, "n": n, "f16_k16_over_two_tf32_k8": round(f16 / (2 * tf32), 3)}))


if __name__ == "__main__":
    sys.exit(main())
