"""What ptxas makes of the normalizer kernels (quantile.cu), checked without a GPU: compiled with the library's own nvcc flags,
no kernel spills, and the scaling path of the widen kernel and numpy's lerp of the quantiles carry no fused multiply-add — sklearn
and numpy round the product and the sum separately, so an FFMA there would change the result's last bit."""
import re
import shutil
import subprocess
from pathlib import Path

import pytest

from dance_b200.build import CSRC, NVCC_FLAGS, PKG

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CUOBJDUMP = str(Path(NVCC).parent / "cuobjdump")

pytestmark = pytest.mark.skipif(not Path(NVCC).exists(), reason="needs nvcc")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    obj = tmp_path_factory.mktemp("quantile") / "quantile.o"
    cmd = [NVCC, *NVCC_FLAGS, "-Xptxas=-v", "-I", str(PKG.parent / "include"), "-c", str(CSRC / "quantile.cu"), "-o", str(obj)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    return obj, res.stderr


def test_quantile_kernels_do_not_spill(compiled):
    _, log = compiled
    reports = dict(re.findall(r"Function properties for (\S+)\s*\n\s*(\d+ bytes stack frame, \d+ bytes spill stores, \d+ bytes spill loads)",
                              log))
    for frag in ("radix_hist_kernelILi0", "radix_hist_kernelILi1", "radix_hist_kernelILi2", "radix_scan_kernelILi0",
                 "radix_scan_kernelILi1", "radix_scan_kernelILi2", "quantile_finish_kernel", "col_minmax_kernel", "concat_kernelILb1",
                 "concat_kernelILb0", "minmax_params_kernel"):
        names = [n for n in reports if frag in n]
        assert names, f"no ptxas report for {frag}"
        for n in names:
            assert reports[n] == "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", f"{n}: {reports[n]}"


def _sass_by_function(obj):
    res = subprocess.run([CUOBJDUMP, "-sass", str(obj)], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    funcs, cur = {}, None
    for line in res.stdout.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur is not None:
            funcs[cur].append(line)
    return funcs


@pytest.mark.skipif(not Path(CUOBJDUMP).exists(), reason="needs cuobjdump")
def test_scale_and_lerp_paths_have_no_ffma(compiled):
    obj, _ = compiled
    funcs = _sass_by_function(obj)
    for frag in ("concat_kernelILb1", "quantile_finish_kernel"):
        names = [n for n in funcs if frag in n]
        assert names, f"no SASS for {frag}"
        for n in names:
            body = "\n".join(funcs[n])
            assert "FFMA" not in body, f"{n} contracts a multiply and an add"
            assert "FMUL" in body and "FADD" in body, f"{n}: expected separately rounded FMUL / FADD"
