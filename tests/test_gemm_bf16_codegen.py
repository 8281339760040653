"""What ptxas makes of the bf16 instantiations of the tensor-core GEMM (gemm_tc.cu), checked without a GPU.

Compiles gemm_tc.cu with the library's own nvcc flags: each bf16 kernel must keep its k-block's wgmmas in flight while the
next stage is rewritten (no serialisation warning, a WARPGROUP.DEPBAR that leaves one group outstanding), spill nothing,
and issue the m64nBNk16 bf16 tensor-core instruction."""
import re
import shutil
import subprocess
from pathlib import Path

import pytest

from dance_b200.build import CSRC, NVCC_FLAGS, PKG

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CUOBJDUMP = str(Path(NVCC).with_name("cuobjdump"))
MODE_BF16 = 2
KERNELS = {bn: f"_ZN2b22tc14gemm_tc_kernelILi{bn}ELi{MODE_BF16}EEEvNS0_6ParamsE" for bn in (32, 64, 128)}

pytestmark = pytest.mark.skipif(not (Path(NVCC).exists() and Path(CUOBJDUMP).exists()), reason="needs nvcc and cuobjdump")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    obj = tmp_path_factory.mktemp("gemm_tc") / "gemm_tc.o"
    cmd = [NVCC, *NVCC_FLAGS, "-Xptxas=-v", "-I", str(PKG.parent / "include"), "-c", str(CSRC / "gemm_tc.cu"), "-o", str(obj)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    return obj, res.stderr


@pytest.mark.parametrize("bn", sorted(KERNELS))
def test_gemm_bf16_not_serialised_and_no_spills(compiled, bn):
    _, log = compiled
    name = KERNELS[bn]
    serialised = [line for line in log.splitlines() if name in line and re.search(r"\(C751[1-8]\)", line)]
    assert not serialised, "\n".join(serialised)
    m = re.search(re.escape(f"Function properties for {name}") + r"\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads", log)
    assert m, f"no ptxas report for {name}"
    assert m.groups() == ("0", "0", "0"), f"{name}: stack frame / spill stores / spill loads = {m.groups()}"


@pytest.mark.parametrize("bn", sorted(KERNELS))
def test_gemm_bf16_sass(compiled, bn):
    """Two HGMMA.64xBNx16.F32.BF16 per 32-wide k-block, and no wait for them until the next k-block has been rewritten."""
    obj, _ = compiled
    sass = subprocess.run([CUOBJDUMP, "-sass", "-fun", KERNELS[bn], str(obj)], capture_output=True, text=True, check=True).stdout
    hgmma = re.findall(r"\bHGMMA\.(\S+)", sass)
    assert hgmma and all(h == f"64x{bn}x16.F32.BF16" for h in hgmma), hgmma
    waits = re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, (0x[0-9a-f]+)", sass)
    assert "0x1" in waits, waits
