"""What ptxas makes of the dropout instantiations of the GAT kernels (gat.cu) and of the dropout kernel (dropout.cu), checked
without a GPU: compiled with the library's own nvcc flags, none of them spills."""
import re
import shutil
import subprocess
from pathlib import Path

import pytest

from dance_b200.build import CSRC, NVCC_FLAGS, PKG

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"

pytestmark = pytest.mark.skipif(not Path(NVCC).exists(), reason="needs nvcc")

# mangled-name fragments of the new instantiations: DROP / IDENTITY = true, the identity backward, the dropout kernel
NEW = {"gat.cu": ("gat_aggregate_fwd_kernelILb1E", "gat_bwd_target_kernelILb1E", "gat_bwd_source_kernelILb1E",
                  "gat_combine_fwd_kernelILb1E", "gat_combine_bwd_identity_kernel"),
       "dropout.cu": ("dropout_kernel", )}


@pytest.mark.parametrize("src", sorted(NEW))
def test_new_gat_dropout_kernels_do_not_spill(tmp_path, src):
    obj = tmp_path / "k.o"
    cmd = [NVCC, *NVCC_FLAGS, "-Xptxas=-v", "-I", str(PKG.parent / "include"), "-c", str(CSRC / src), "-o", str(obj)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    reports = dict(re.findall(r"Function properties for (\S+)\s*\n\s*(\d+ bytes stack frame, \d+ bytes spill stores, \d+ bytes spill loads)",
                              res.stderr))
    for frag in NEW[src]:
        names = [n for n in reports if frag in n]
        assert names, f"no ptxas report for {frag}"
        for n in names:
            assert reports[n] == "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", f"{n}: {reports[n]}"
