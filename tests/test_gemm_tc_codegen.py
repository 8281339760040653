"""What ptxas makes of the tensor-core GEMM (gemm_tc.cu) in every precision mode and tile width, checked without a GPU.

Compiles gemm_tc.cu with the library's own nvcc flags.  Each instantiation must keep a k-block's wgmmas in flight while the
rewrite warpgroup prepares the next plane stage: no serialisation warning (C751x: ptxas inserts a wait after every wgmma when
ordinary instructions also define the accumulators), one WARPGROUP.DEPBAR that leaves one group outstanding per k-block and no
wait between the HGMMAs of one k-block.  It must spill nothing (the setmaxnreg split leaves the consumers room for both
accumulators) and issue the expected tensor-core instruction the expected number of times per 32-wide k-block."""
import re
import shutil
import subprocess
from pathlib import Path

import pytest

from dance_b200.build import CSRC, NVCC_FLAGS, PKG

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CUOBJDUMP = str(Path(NVCC).with_name("cuobjdump"))
# mode name → (Mode value in gemm_tc.cu, HGMMA suffix after 64xBN, HGMMAs per k-block per warpgroup)
MODES = {
    "tf32": (0, "x8.F32.TF32", 4),        # BK / 8 m64nBNk8
    "tf32x3": (1, "x8.F32.TF32", 12),     # lo·hi, hi·lo, hi·hi per k-step
    "bf16": (2, "x16.F32.BF16", 2),       # BK / 16 m64nBNk16
}
CASES = [(mode, bn) for mode in MODES for bn in (32, 64, 128)]

pytestmark = pytest.mark.skipif(not (Path(NVCC).exists() and Path(CUOBJDUMP).exists()), reason="needs nvcc and cuobjdump")


def kernel_name(mode, bn):
    return f"_ZN2b22tc14gemm_tc_kernelILi{bn}ELi{MODES[mode][0]}EEEvNS0_6ParamsE"


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    obj = tmp_path_factory.mktemp("gemm_tc") / "gemm_tc.o"
    cmd = [NVCC, *NVCC_FLAGS, "-Xptxas=-v", "-I", str(PKG.parent / "include"), "-c", str(CSRC / "gemm_tc.cu"), "-o", str(obj)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    return obj, res.stderr


@pytest.mark.parametrize("mode,bn", CASES)
def test_gemm_not_serialised_and_no_spills(compiled, mode, bn):
    _, log = compiled
    name = kernel_name(mode, bn)
    serialised = [line for line in log.splitlines() if name in line and re.search(r"\(C751\d\)", line)]
    assert not serialised, "\n".join(serialised)
    m = re.search(re.escape(f"Function properties for {name}") + r"\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads", log)
    assert m, f"no ptxas report for {name}"
    assert m.groups() == ("0", "0", "0"), f"{name}: stack frame / spill stores / spill loads = {m.groups()}"


@pytest.mark.parametrize("mode,bn", CASES)
def test_gemm_sass(compiled, mode, bn):
    """Every run of HGMMAs is one whole k-block of the expected shape, closed by a wait that leaves it in flight (0x1)."""
    obj, _ = compiled
    _, suffix, per_kblock = MODES[mode]
    sass = subprocess.run([CUOBJDUMP, "-sass", "-fun", kernel_name(mode, bn), str(obj)], capture_output=True, text=True,
                          check=True).stdout
    hgmma = re.findall(r"\bHGMMA\.(\S+)", sass)
    assert hgmma and all(h == f"64x{bn}{suffix}" for h in hgmma), hgmma
    runs, count = [], 0                   # (HGMMAs since the previous wait, the wait that ends them)
    for tok in re.findall(r"\bHGMMA\.|WARPGROUP\.DEPBAR\.LE gsb0, (0x[0-9a-f]+)", sass):
        if tok == "":
            count += 1
        else:
            runs.append((count, tok))
            count = 0
    assert count == 0, "HGMMAs after the last wait"
    issued = [r for r in runs if r[0]]
    assert issued and all(r == (per_kblock, "0x1") for r in issued), runs
