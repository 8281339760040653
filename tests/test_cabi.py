"""The C-ABI library loads and exports every symbol include/dance_b200.h declares (no GPU needed)."""
import ctypes
import re
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


def _declared():
    text = (ROOT / "include" / "dance_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b2_[a-z0-9_]+)\s*\(", text)))


def test_header_declares_something():
    names = _declared()
    assert "b2_spmm_csr_f32" in names and "b2_gemm_f32" in names and len(names) >= 20


def test_library_exports_every_declared_symbol():
    from dance_b200 import _lib
    from dance_b200.build import build
    build()  # nvcc cross-compiles for sm_90a without a GPU
    handle = ctypes.CDLL(str(_lib.lib_path()))
    missing = [n for n in _declared() if not hasattr(handle, n)]
    assert not missing, f"symbols declared in dance_b200.h but not exported: {missing}"


def test_python_binding_covers_header():
    from dance_b200 import _lib
    assert sorted(_lib.declared_symbols()) == _declared()


def test_binding_types_come_from_the_header():
    """The ctypes signatures are generated from dance_b200.h: spot checks of each mapping, and a type without one raises."""
    from dance_b200 import _lib
    sigs = _lib.parse_header((ROOT / "include" / "dance_b200.h").read_text())
    assert sorted(sigs) == _declared()
    assert sigs["b2_last_error"] == (ctypes.c_char_p, [])
    res, args = sigs["b2_radius_graph_count"]
    assert res is ctypes.c_int and args[4] is ctypes.c_double and args[0] is ctypes.c_void_p
    args = sigs["b2_dropout_f32"][1]
    assert args[5] is ctypes.c_uint32 and args[6] is ctypes.c_uint32 and args[4] is ctypes.c_float
    assert len(sigs["b2_gemm_f32"][1]) == 20 and sigs["b2_gemm_workspace_bytes"][0] is ctypes.c_size_t
    assert _lib.parse_header("typedef struct s s;\nint b2_f(const s* p, int64_t n, void* stream);") == \
        {"b2_f": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p])}
    for bad in ("int b2_f(long n);", "int b2_f(unsigned int n);", "long b2_f(void);", "int b2_f(int);", "struct s { int a; };"):
        with pytest.raises(_lib.B2Error):
            _lib.parse_header(bad)


def test_error_reporting_without_gpu():
    from dance_b200 import _lib
    lib = _lib.lib()
    assert lib.b2_version() >= 100
    # argument validation happens before any CUDA call, so it can be exercised on the CPU box
    rc = lib.b2_spmm_csr_f32(None, None, None, None, 0, None, 0, 1, 1, 4, 0, 0, None, None)
    assert rc == -1
    assert b"null pointer" in lib.b2_last_error()


def test_ops_refuse_cpu_tensors():
    import torch
    from dance_b200 import ops
    from dance_b200._lib import B2Error
    with pytest.raises(B2Error):
        ops.gemm(torch.zeros(4, 4), torch.zeros(4, 4))


def test_sass_is_sm90a():
    """The shipped library carries sm_90a SASS (and nothing else)."""
    import shutil
    import subprocess
    from dance_b200 import _lib
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    out = subprocess.run([cuobjdump, "-lelf", str(_lib.lib_path())], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_(\d+a?)", out))
    assert archs == {"90a"}, archs


def test_library_contains_hopper_tensor_core_and_tma_code():
    """The shipped .so is sm_90a code that really uses the warpgroup tensor-core MMA and TMA: the SASS of the GEMM, decoder
    and kNN-filter kernels must contain HGMMA (wgmma.mma_async), UTMALDG (cp.async.bulk.tensor) and UBLKCP (cp.async.bulk).
    Needs cuobjdump (CUDA toolkit); skipped where it is not installed."""
    import shutil
    import subprocess
    from dance_b200 import _lib
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(cuobjdump).exists():
        pytest.skip("cuobjdump not available")
    lib_path = Path(_lib.__file__).resolve().parent / "lib" / "libdance_b200.so"
    elf = subprocess.run([cuobjdump, "-lelf", str(lib_path)], capture_output=True, text=True, timeout=120).stdout
    assert "sm_90a" in elf
    sass = subprocess.run([cuobjdump, "-sass", str(lib_path)], capture_output=True, text=True, timeout=300).stdout
    for mnemonic in ("HGMMA", "UTMALDG", "UBLKCP"):
        assert mnemonic in sass, mnemonic
    for kernel in ("gemm_tc_kernel", "gae_allpairs_tc_kernel", "knn_candidates_tc_kernel"):
        assert kernel in sass, kernel


def test_header_is_plain_c(tmp_path):
    """The boundary is a C ABI: include/dance_b200.h must compile as C99 (no C++ constructs, no torch / CUDA types)."""
    import shutil
    import subprocess
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    src = tmp_path / "probe.c"
    hdr = Path(__file__).resolve().parent.parent / "include"
    src.write_text('#include "dance_b200.h"\nint main(void) { return b2_version() < 0; }\n')
    res = subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-pedantic", "-fsyntax-only", f"-I{hdr}", str(src)], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    code = re.sub(r"/\*.*?\*/", "", (hdr / "dance_b200.h").read_text(), flags=re.S)      # declarations only, comments stripped
    for banned in ("std::", "template", "class ", "Tensor", "cudaStream_t", "torch"):
        assert banned not in code, banned


def test_selector_tables_match_the_header():
    """ops.set_path / ops.set_tuning index the library's selector arrays by the header's constants: the Python tables must name
    every B2_PATH_* / B2_TUNE_* selector with the header's number, and an out-of-range selector is refused by the library."""
    import re
    from pathlib import Path
    from dance_b200 import _lib, ops
    hdr = (Path(__file__).resolve().parent.parent / "include" / "dance_b200.h").read_text()
    consts = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define\s+(B2_(?:PATH|TUNE)_[A-Z_]+)\s+(\d+)", hdr)}
    assert consts["B2_PATH_COUNT"] == 3 and consts["B2_TUNE_COUNT"] == 1
    assert {k: v[0] for k, v in ops._PATHS.items()} == {"gae": consts["B2_PATH_GAE_DECODER"], "knn": consts["B2_PATH_KNN_FILTER"],
                                                         "spmm": consts["B2_PATH_SPMM"]}
    lib = _lib.lib()
    assert lib.b2_set_path(consts["B2_PATH_COUNT"], 0) != 0 and lib.b2_set_tuning(consts["B2_TUNE_COUNT"], 0) != 0
    assert lib.b2_set_path(consts["B2_PATH_SPMM"], 1) == 0 and lib.b2_get_path(consts["B2_PATH_SPMM"]) == 1
    assert lib.b2_set_path(consts["B2_PATH_SPMM"], 0) == 0
    assert lib.b2_set_path(consts["B2_PATH_GAE_DECODER"], 2) == 0 and lib.b2_set_path(consts["B2_PATH_GAE_DECODER"], 3) != 0
    assert lib.b2_set_path(consts["B2_PATH_GAE_DECODER"], 6) != 0
    assert lib.b2_set_path(consts["B2_PATH_GAE_DECODER"], 0) == 0
    for knob, idx in (("gae_splits", consts["B2_TUNE_GAE_SPLITS"]),):
        assert lib.b2_set_tuning(idx, 1) == 0
    ops.set_tuning("gae_splits", 0)   # the default
