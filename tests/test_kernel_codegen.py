"""What ptxas makes of the hand-written kernels, checked without a GPU (see kernel_codegen.py).

Every kernel below keeps a zero stack frame and spills nothing under the library's own nvcc flags.  The tensor-core kernels
(the decoder's two sweeps in gae_tc.cu, the GEMM in gemm_tc.cu) are only fast while their wgmma batches stay in flight: ptxas
serialises every wgmma of a kernel, a WARPGROUP.DEPBAR after each, when the register operands of a batch do not fit or
ordinary instructions also define the accumulators, and says so with a C751x message.  Each GEMM instantiation issues the
expected tensor-core instruction per 32-wide k-block with one wait that leaves the k-block in flight while the rewrite
warpgroup prepares the next plane stage.  The normalizer's scaling path and numpy's lerp of the quantiles (quantile.cu) carry
no fused multiply-add: sklearn and numpy round the product and the sum separately, so an FFMA there would change the result's
last bit."""
import re

import pytest

from kernel_codegen import compiled, needs_cuobjdump, needs_nvcc

# gemm_tc.cu: mode name → (Mode value, HGMMA suffix after 64xBN, HGMMAs per k-block per warpgroup)
GEMM_MODES = {
    "tf32": (0, "x8.F32.TF32", 4),        # BK / 8 m64nBNk8
    "tf32x3": (1, "x8.F32.TF32", 12),     # lo·hi, hi·lo, hi·hi per k-step
    "bf16": (2, "x16.F32.BF16", 2),       # BK / 16 m64nBNk16
}
GEMM = [(mode, bn) for mode in GEMM_MODES for bn in (32, 64, 128)]


def gemm_kernel(mode, bn):
    return f"gemm_tc_kernelILi{bn}ELi{GEMM_MODES[mode][0]}E"


# source → fragments of the mangled kernel names checked in it
KERNELS = {
    "gae_tc.cu": tuple(f"gae_{sweep}_tc_kernelILi{dp}E" for sweep in ("allpairs", "tri") for dp in (8, 16, 32)),
    "gemm_tc.cu": tuple(gemm_kernel(mode, bn) for mode, bn in GEMM),
    "gat.cu": ("gat_aggregate_fwd_kernelILb1E", "gat_bwd_target_kernelILb1E", "gat_bwd_source_kernelILb1E",
               "gat_combine_fwd_kernelILb1E", "gat_combine_bwd_kernel", "gat_combine_bwd_identity_kernel"),
    "dropout.cu": ("dropout_kernel",),
    "optim.cu": ("act_fwd_kernel", "act_bwd_kernel"),
    "quantile.cu": ("radix_hist_kernelILi0", "radix_hist_kernelILi1", "radix_hist_kernelILi2", "radix_scan_kernelILi0",
                    "radix_scan_kernelILi1", "radix_scan_kernelILi2", "quantile_finish_kernel", "col_minmax_kernel",
                    "concat_kernelILb1", "concat_kernelILb0", "minmax_params_kernel"),
}
ALL = [(src, frag) for src, frags in KERNELS.items() for frag in frags]
TENSOR_CORE = [(src, frag) for src, frag in ALL if src in ("gae_tc.cu", "gemm_tc.cu")]


@needs_nvcc
@pytest.mark.parametrize("src,frag", ALL)
def test_no_stack_frame_or_spills(src, frag):
    c = compiled(src)
    for name in c.kernels(frag):
        assert c.frame(name) == (0, 0, 0), f"{name}: stack frame / spill stores / spill loads = {c.frame(name)}"


@needs_nvcc
@pytest.mark.parametrize("src,frag", TENSOR_CORE)
def test_wgmma_not_serialised(src, frag):
    c = compiled(src)
    for name in c.kernels(frag):
        assert not c.serialised(name), "\n".join(c.serialised(name))


@needs_cuobjdump
@pytest.mark.parametrize("mode,bn", GEMM)
def test_gemm_sass(mode, bn):
    """Every run of HGMMAs is one whole k-block of the expected shape, closed by a wait that leaves it in flight (0x1)."""
    _, suffix, per_kblock = GEMM_MODES[mode]
    c = compiled("gemm_tc.cu")
    name, = c.kernels(gemm_kernel(mode, bn))
    sass = c.sass(name)
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


@needs_cuobjdump
def test_scale_and_lerp_paths_have_no_ffma():
    c = compiled("quantile.cu")
    for frag in ("concat_kernelILb1", "quantile_finish_kernel"):
        for name in c.kernels(frag):
            body = c.sass(name)
            assert "FFMA" not in body, f"{name} contracts a multiply and an add"
            assert "FMUL" in body and "FADD" in body, f"{name}: expected separately rounded FMUL / FADD"
