"""Build the C-ABI shared library ``dance_b200/lib/libdance_b200.so`` with nvcc for sm_90a.

The library is built IN-TREE (git-ignored) so that the package is importable from the
repository tree.  ``python -m dance_b200.build`` or ``__graft_entry__.build()`` run this;
nothing is JIT-compiled at import time.
"""
from __future__ import annotations

import concurrent.futures as cf
import hashlib
import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIB_DIR = PKG / "lib"
OBJ_DIR = PKG / "lib" / "obj"
LIB_PATH = LIB_DIR / "libdance_b200.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "--expt-relaxed-constexpr", "--expt-extended-lambda",
    "-Xcompiler", "-fPIC",
    "-DB2_BUILDING",
]


def _nvcc() -> str:
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(cand):
        raise RuntimeError("nvcc not found; dance_b200 needs the CUDA toolkit to build its kernels")
    return cand


def _sources():
    return sorted(CSRC.glob("*.cu"))


def _digest(src: Path) -> str:
    h = hashlib.sha256()
    h.update(src.read_bytes())
    for hdr in sorted(CSRC.glob("*.cuh")) + [PKG.parent / "include" / "dance_b200.h"]:
        h.update(hdr.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()[:16]


def _compile_one(src: Path, verbose: bool) -> Path:
    obj = OBJ_DIR / f"{src.stem}.{_digest(src)}.o"
    if obj.exists():
        return obj
    for old in OBJ_DIR.glob(f"{src.stem}.*.o"):
        old.unlink()
    cmd = [_nvcc(), *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src.name}:\n{res.stdout}\n{res.stderr}")
    if verbose and res.stderr:
        sys.stderr.write(res.stderr)
    return obj


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every ``csrc/*.cu`` for sm_90a and link ``libdance_b200.so``; returns its path."""
    LIB_DIR.mkdir(exist_ok=True)
    OBJ_DIR.mkdir(exist_ok=True)
    if force:
        for o in OBJ_DIR.glob("*.o"):
            o.unlink()
    srcs = _sources()
    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(lambda s: _compile_one(s, verbose), srcs))
    stamp = LIB_DIR / "link.stamp"
    key = " ".join(o.name for o in objs)
    if LIB_PATH.exists() and stamp.exists() and stamp.read_text() == key and not force:
        return LIB_PATH
    cmd = [_nvcc(), "-shared", "-o", str(LIB_PATH), *map(str, objs),
           "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC", "-lcudart_static", "-ldl", "-lrt", "-lpthread"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"link failed:\n{res.stdout}\n{res.stderr}")
    stamp.write_text(key)
    return LIB_PATH


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(p)
