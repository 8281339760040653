"""Compile one of the library's CUDA sources and read what ptxas and cuobjdump make of it, without a GPU.

The codegen tests check the ptxas report (stack frame, spills, and the C751x messages with which ptxas says it serialised a
kernel's wgmmas, a wait after each one) and the SASS that a kernel's speed depends on.  Each source is compiled once per
process with the library's own nvcc flags plus -Xptxas=-v, which prints the report without changing the code, so the one
object serves both the report and the SASS checks."""
import functools
import re
import shutil
import subprocess
import tempfile
from pathlib import Path

import pytest

from dance_b200.build import CSRC, NVCC_FLAGS, PKG

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CUOBJDUMP = str(Path(NVCC).with_name("cuobjdump"))

needs_nvcc = pytest.mark.skipif(not Path(NVCC).exists(), reason="needs nvcc")
needs_cuobjdump = pytest.mark.skipif(not (Path(NVCC).exists() and Path(CUOBJDUMP).exists()), reason="needs nvcc and cuobjdump")

_FRAME = re.compile(r"Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads")
_SERIALISED = re.compile(r"\(C751\d\)")


class Compiled:
    def __init__(self, source: str):
        self._tmp = tempfile.TemporaryDirectory(prefix="codegen-")
        self.obj = Path(self._tmp.name) / (Path(source).stem + ".o")
        cmd = [NVCC, *NVCC_FLAGS, "-Xptxas=-v", "-I", str(PKG.parent / "include"), "-c", str(CSRC / source), "-o", str(self.obj)]
        res = subprocess.run(cmd, capture_output=True, text=True)
        assert res.returncode == 0, res.stderr
        self.log = res.stderr
        self._frames = {name: tuple(int(x) for x in f) for name, *f in _FRAME.findall(self.log)}

    def kernels(self, fragment: str):
        """The mangled names in the ptxas report that contain `fragment`."""
        names = sorted(n for n in self._frames if fragment in n)
        assert names, f"no ptxas report for a function named *{fragment}*"
        return names

    def frame(self, name: str):
        """(stack frame, spill stores, spill loads) in bytes."""
        assert name in self._frames, f"no ptxas report for {name}"
        return self._frames[name]

    def serialised(self, name: str):
        """The ptxas lines saying that `name`'s wgmmas are serialised."""
        return [line for line in self.log.splitlines() if name in line and _SERIALISED.search(line)]

    def sass(self, name: str) -> str:
        assert name in self._sass, f"no SASS for {name}"
        return self._sass[name]

    @functools.cached_property
    def _sass(self):
        res = subprocess.run([CUOBJDUMP, "-sass", str(self.obj)], capture_output=True, text=True)
        assert res.returncode == 0, res.stderr
        funcs, cur = {}, None
        for line in res.stdout.splitlines():
            m = re.search(r"Function : (\S+)", line)
            if m:
                cur = m.group(1)
                funcs[cur] = []
            elif cur is not None:
                funcs[cur].append(line)
        return {name: "\n".join(lines) for name, lines in funcs.items()}


@functools.cache
def compiled(source: str) -> Compiled:
    """dance_b200/csrc/<source>, compiled for sm_90a once per process."""
    return Compiled(source)
