"""Tensor-core GEMM at the k-block counts where its rings turn over, in every precision and operand layout, against float64.

The rewrite warpgroup hands k-blocks to the consumers through a raw ring and a plane ring (at BN = 128: 3 raw and 2 plane
stages in tf32x3, 4 and 3 in tf32, 4 and 4 in bf16).  The shapes cover a single k-block, one k-block more than each ring
holds, and a split-K plan whose last split has a single k-block."""
import numpy as np
import pytest
import torch

from bf16_ref import bf16
from conftest import rel_err

pytestmark = pytest.mark.gpu

# the bounds of test_gpu_gemm_tc.py (tf32x3, tf32) and test_gpu_gemm_bf16.py (bf16 against its rounded operands)
TOL = {"tf32x3": 1e-5, "tf32": 2e-3, "bf16": 1e-5}

SHAPES = [
    (384, 256, 32),      # a single k-block
    (256, 384, 96),      # 3 k-blocks: one more than the tf32x3 plane ring
    (384, 256, 128),     # 4 k-blocks: one more than the tf32x3 raw ring and the tf32 plane ring
    (384, 256, 160),     # 5 k-blocks: one more than the tf32 raw ring and both bf16 rings
    (128, 128, 1300),    # split-K, 41 k-blocks in 9 splits of 5 on 132 SMs: the last split has one k-block, K tail included
]


@pytest.mark.parametrize("precision", ["tf32x3", "tf32", "bf16"])
@pytest.mark.parametrize("transA,transB", [(0, 1), (0, 0), (1, 0), (1, 1)])
@pytest.mark.parametrize("shape", SHAPES)
def test_gemm_tc_ring_turnover(cuda, precision, transA, transB, shape):
    from dance_b200 import ops
    M, N, K = shape
    rng = np.random.default_rng(M * 7 + N * 3 + K)
    A = torch.from_numpy(rng.normal(size=(K, M) if transA else (M, K)).astype(np.float32)).to(cuda)
    B = torch.from_numpy(rng.normal(size=(N, K) if transB else (K, N)).astype(np.float32)).to(cuda)
    a, b = (A.t() if transA else A), (B.t() if transB else B)
    ref = bf16(a) @ bf16(b) if precision == "bf16" else a.double() @ b.double()
    C = ops.gemm(A, B, transA=bool(transA), transB=bool(transB), precision=precision)
    torch.cuda.synchronize()
    assert rel_err(C, ref) < TOL[precision]
