"""Tensor-core GEMM (TMA + wgmma tf32) against an fp64 reference: every operand layout,
ragged shapes, split-K, all tile widths, fused epilogue; 3xTF32 must be fp32-accurate."""
import numpy as np
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu

# tf32x3: operands are exact (hi/lo split); the tensor-core accumulate is not fp32-exact, which over K≈2000-3000 leaves a few
# 1e-6; plain tf32 truncates the operands (~8e-4).
TOL = {"tf32x3": 1e-5, "tf32": 2e-3}

SHAPES = [
    (256, 128, 64),      # exact tiles
    (300, 200, 100),     # ragged M, N, K (K tail zero-filled by TMA)
    (1000, 512, 2000),   # Feature-AE layer 1 slice
    (1000, 2000, 512),   # layer 4 slice (N not a multiple of 128)
    (640, 32, 128),      # GCN projection, BN = 32
    (640, 48, 36),       # BN = 64 path, tiny K
    (128, 512, 12800),   # weight-gradient shape: few tiles, long K → split-K
    (2000, 512, 3000),
]


@pytest.mark.parametrize("precision", ["tf32x3", "tf32"])
@pytest.mark.parametrize("transA,transB", [(0, 1), (0, 0), (1, 0), (1, 1)])
@pytest.mark.parametrize("shape", SHAPES)
def test_gemm_tc_layouts(cuda, precision, transA, transB, shape):
    from dance_b200 import ops
    M, N, K = shape
    if transA and M % 4:
        M += 4 - M % 4           # TMA needs 16-byte row pitch; other pitches are routed to the CUDA-core kernel
    if not transB and N % 4:
        N += 4 - N % 4
    rng = np.random.default_rng(M * 7 + N * 3 + K)
    A = rng.normal(size=(K, M) if transA else (M, K)).astype(np.float32)
    B = rng.normal(size=(N, K) if transB else (K, N)).astype(np.float32)
    ref = (A.T if transA else A).astype(np.float64) @ (B.T if transB else B).astype(np.float64)
    C = ops.gemm(torch.from_numpy(A).to(cuda), torch.from_numpy(B).to(cuda), transA=bool(transA), transB=bool(transB),
                 precision=precision)
    torch.cuda.synchronize()
    assert rel_err(C.cpu().numpy(), ref) < TOL[precision]


@pytest.mark.parametrize("precision", ["tf32x3", "tf32"])
def test_gemm_tc_epilogue(cuda, precision):
    from dance_b200 import ops
    rng = np.random.default_rng(1)
    M, N, K = 700, 260, 520
    A = rng.normal(size=(M, K)).astype(np.float32)
    W = rng.normal(size=(N, K)).astype(np.float32)
    bias = rng.normal(size=N).astype(np.float32)
    mask = rng.normal(size=(M, N)).astype(np.float32)
    C0 = rng.normal(size=(M, N)).astype(np.float32)
    ref = np.maximum(A.astype(np.float64) @ W.T + bias, 0) * (mask > 0) + C0
    out = torch.from_numpy(C0.copy()).to(cuda)
    ops.gemm(torch.from_numpy(A).to(cuda), torch.from_numpy(W).to(cuda), transB=True, bias=torch.from_numpy(bias).to(cuda),
             act="relu", mask=torch.from_numpy(mask).to(cuda), out=out, accumulate=True, precision=precision)
    assert rel_err(out.cpu().numpy(), ref) < TOL[precision]


def test_gemm_tc_splitk_epilogue_and_padded_ld(cuda):
    """Split-K path applies the epilogue in the reduction kernel; operands with padded leading dimensions."""
    from dance_b200 import ops
    rng = np.random.default_rng(2)
    K, M, N = 6000, 128, 256
    Abig = torch.from_numpy(rng.normal(size=(K, M + 12)).astype(np.float32)).to(cuda)
    Bbig = torch.from_numpy(rng.normal(size=(K, N + 8)).astype(np.float32)).to(cuda)
    A, B = Abig[:, :M], Bbig[:, :N]
    bias = torch.from_numpy(rng.normal(size=N).astype(np.float32)).to(cuda)
    ref = np.tanh(A.cpu().numpy().astype(np.float64).T @ B.cpu().numpy().astype(np.float64) + bias.cpu().numpy())
    C = ops.gemm(A, B, transA=True, bias=bias, act="tanh", precision="tf32x3")
    assert rel_err(C.cpu().numpy(), ref) < 1e-5


def test_gemm_tc_many_tiles_persistent(cuda):
    """More tiles than SMs (several waves of CTAs) with a long K loop: exercises the TMA ring wrap-around and both plane buffers."""
    from dance_b200 import ops
    A = torch.randn(12800, 512, device=cuda)
    B = torch.randn(2000, 512, device=cuda)
    C = ops.gemm(A, B, transB=True, precision="tf32x3")
    ref = (A.double() @ B.double().t())
    assert rel_err(C.cpu().numpy(), ref.cpu().numpy()) < 1e-5
