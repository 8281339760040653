"""What ptxas makes of the triangle sweep of the tensor-core decoder (gae_tri_tc_kernel in gae_tc.cu), checked without a GPU.

The same three checks as for the full sweep (test_decoder_codegen.py), for every instantiation: no serialised wgmmas
(C7511 / C7512 / C7515 / C7518), no spills, and one WARPGROUP.DEPBAR per batch rather than one per HGMMA.  The source is
compiled through a wrapper that also asserts, at compile time, that the dynamic shared memory each instantiation asks for
fits the 227 KB a CTA may have."""
import re
import shutil
import subprocess
from pathlib import Path

import pytest

from dance_b200.build import CSRC, NVCC_FLAGS, PKG

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CUOBJDUMP = str(Path(NVCC).with_name("cuobjdump"))
KERNELS = {dp: f"_ZN2b23gtc17gae_tri_tc_kernelILi{dp}EEEvNS0_6ParamsE" for dp in (8, 16, 32)}

pytestmark = pytest.mark.skipif(not (Path(NVCC).exists() and Path(CUOBJDUMP).exists()), reason="needs nvcc and cuobjdump")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("gae_tri")
    src = tmp / "gae_tri_probe.cu"
    src.write_text(f'#include "{CSRC / "gae_tc.cu"}"\n' + "".join(
        f"static_assert(b2::gtc::Tiles<{dp}, true>::SMEM <= 227 * 1024, \"triangle DP = {dp}: shared memory\");\n" for dp in KERNELS))
    obj = tmp / "gae_tri_probe.o"
    cmd = [NVCC, *NVCC_FLAGS, "-Xptxas=-v", "-I", str(PKG.parent / "include"), "-c", str(src), "-o", str(obj)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    return obj, res.stderr


@pytest.mark.parametrize("dp", sorted(KERNELS))
def test_triangle_wgmma_not_serialised_and_no_spills(compiled, dp):
    _, log = compiled
    name = KERNELS[dp]
    serialised = [line for line in log.splitlines() if name in line and re.search(r"\(C751[1258]\)", line)]
    assert not serialised, "\n".join(serialised)
    m = re.search(re.escape(f"Function properties for {name}") + r"\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads", log)
    assert m, f"no ptxas report for {name}"
    assert m.groups() == ("0", "0", "0"), f"{name}: stack frame / spill stores / spill loads = {m.groups()}"


@pytest.mark.parametrize("dp", sorted(KERNELS))
def test_triangle_waits_once_per_batch(compiled, dp):
    """S (3·DP/8 HGMMAs) and dZ_I + dZ_J (2·8 + 2·8) each end in one wait, not one per HGMMA."""
    obj, _ = compiled
    sass = subprocess.run([CUOBJDUMP, "-sass", "-fun", KERNELS[dp], str(obj)], capture_output=True, text=True, check=True).stdout
    hgmma = len(re.findall(r"\bHGMMA\.", sass))
    depbar = len(re.findall(r"\bWARPGROUP\.DEPBAR\b", sass))
    assert hgmma >= 2 * (3 * dp // 8 + 32), f"expected the S and dZ batches in the SASS, found {hgmma} HGMMA"
    assert depbar * 8 <= hgmma, f"{depbar} WARPGROUP.DEPBAR for {hgmma} HGMMA"
