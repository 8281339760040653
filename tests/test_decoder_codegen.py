"""What ptxas makes of the tensor-core decoder (gae_tc.cu), checked without a GPU.

The decoder is only fast while its wgmma batches stay in flight: ptxas serialises every wgmma of a kernel (one
WARPGROUP.DEPBAR after each) when the register operands of a batch do not fit, and says so with C7511 / C7512 / C7518.
Compiles gae_tc.cu with the library's own nvcc flags and checks the messages, the spills and the SASS."""
import re
import shutil
import subprocess
from pathlib import Path

import pytest

from dance_b200.build import CSRC, NVCC_FLAGS, PKG

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CUOBJDUMP = str(Path(NVCC).with_name("cuobjdump"))
KERNELS = {dp: f"_ZN2b23gtc22gae_allpairs_tc_kernelILi{dp}EEEvNS0_6ParamsE" for dp in (8, 16, 32)}

pytestmark = pytest.mark.skipif(not (Path(NVCC).exists() and Path(CUOBJDUMP).exists()), reason="needs nvcc and cuobjdump")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    obj = tmp_path_factory.mktemp("gae_tc") / "gae_tc.o"
    cmd = [NVCC, *NVCC_FLAGS, "-Xptxas=-v", "-I", str(PKG.parent / "include"), "-c", str(CSRC / "gae_tc.cu"), "-o", str(obj)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    return obj, res.stderr


@pytest.mark.parametrize("dp", sorted(KERNELS))
def test_decoder_wgmma_not_serialised_and_no_spills(compiled, dp):
    _, log = compiled
    name = KERNELS[dp]
    serialised = [line for line in log.splitlines() if name in line and re.search(r"\(C751[128]\)", line)]
    assert not serialised, "\n".join(serialised)
    m = re.search(re.escape(f"Function properties for {name}") + r"\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads", log)
    assert m, f"no ptxas report for {name}"
    assert m.groups() == ("0", "0", "0"), f"{name}: stack frame / spill stores / spill loads = {m.groups()}"


def test_decoder_dp16_waits_once_per_batch(compiled):
    """One wait per batch (S: 6 HGMMAs, dZ: 48) instead of one per HGMMA."""
    obj, _ = compiled
    sass = subprocess.run([CUOBJDUMP, "-sass", "-fun", KERNELS[16], str(obj)], capture_output=True, text=True, check=True).stdout
    hgmma = len(re.findall(r"\bHGMMA\.", sass))
    depbar = len(re.findall(r"\bWARPGROUP\.DEPBAR\b", sass))
    assert hgmma >= 54, f"expected the S and dZ batches in the SASS, found {hgmma} HGMMA"
    assert depbar * 8 <= hgmma, f"{depbar} WARPGROUP.DEPBAR for {hgmma} HGMMA"
