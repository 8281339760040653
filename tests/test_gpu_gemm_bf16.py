"""bf16 mode of the tensor-core GEMM (precision="bf16"): operands rounded to bfloat16 in the kernel, fp32 accumulate.

Two float64 references: *exact* multiplies the operands as torch rounds them (``.to(torch.bfloat16)``, round-to-nearest-even),
so only the fp32 accumulation of the tensor cores differs from it; *plain* multiplies the fp32 operands unrounded."""
import ctypes as C

import numpy as np
import pytest
import torch

from bf16_ref import bf16
from conftest import rel_err

pytestmark = pytest.mark.gpu

# Bounds (norm-wise), from errors measured on an H100 80 GB HBM3: against *exact* the error is the fp32 accumulation alone
# (the same argument as the tf32x3 bound of test_gpu_gemm_tc.py), at most 9.8e-7 over the layout cases; against *plain* it
# is the operand rounding, 2^-9 relative per operand: 2.3e-3 to 2.4e-3 over the layout cases, and in the epilogue cases up
# to 9.3e-3 with tanh at K = 6 000, which magnifies the rounding of pre-activations near zero.
TOL_EXACT = 1e-5
TOL_PLAIN = 4e-3
TOL_PLAIN_TANH = 3e-2

SHAPES = [
    (256, 128, 64),      # exact tiles
    (300, 200, 100),     # ragged M, N, K (K tail shorter than a k-block, zero-filled by TMA)
    (1000, 512, 2000),   # Feature-AE layer 1 slice
    (1000, 2000, 512),   # layer 4 slice (N not a multiple of 128)
    (640, 32, 128),      # GCN projection, BN = 32
    (640, 48, 36),       # BN = 64 path, tiny K
    (128, 512, 12800),   # weight-gradient shape: few tiles, long K → split-K
    (2000, 512, 3000),
    (12800, 2000, 512),  # many tiles: several waves of CTAs, ring wrap-around
]


def _refs(A, B, transA, transB):
    a, b = (A.t() if transA else A), (B.t() if transB else B)
    return bf16(a) @ bf16(b), a.double() @ b.double()


def _ws_bytes(M, N, K, transA, transB):
    from dance_b200 import ops
    return int(ops.lib().b2_gemm_workspace_bytes(M, N, K, int(transA), int(transB), ops.PREC["bf16"]))


@pytest.mark.parametrize("transA,transB", [(0, 1), (0, 0), (1, 0), (1, 1)])
@pytest.mark.parametrize("shape", SHAPES)
def test_gemm_bf16_layouts(cuda, transA, transB, shape):
    from dance_b200 import ops
    M, N, K = shape
    if transA and M % 4:
        M += 4 - M % 4           # TMA needs a 16-byte row pitch; other pitches are routed to the CUDA-core kernel
    if not transB and N % 4:
        N += 4 - N % 4
    g = torch.Generator(device=cuda).manual_seed(M * 7 + N * 3 + K)
    A = torch.randn((K, M) if transA else (M, K), device=cuda, generator=g)
    B = torch.randn((N, K) if transB else (K, N), device=cuda, generator=g)
    exact, plain = _refs(A, B, transA, transB)
    C = ops.gemm(A, B, transA=bool(transA), transB=bool(transB), precision="bf16")
    assert rel_err(C, exact) < TOL_EXACT
    assert rel_err(C, plain) < TOL_PLAIN
    if shape == (128, 512, 12800):
        assert _ws_bytes(M, N, K, transA, transB) > 0          # the split-K path ran


def _rounding_cases(rows):
    """fp32 values, as bits, that tell round-to-nearest-even from any other rounding: exact ties (low 16 bits 0x8000) with an
    even and an odd kept LSB, one ulp either side of a tie, random low bits; magnitudes from the smallest normals up to 2^126
    (finite after rounding); both signs."""
    rng = np.random.default_rng(7)
    hi = rng.integers(0x0080, 0x7E80, size=rows * 8).astype(np.uint32)          # exponent 1..252, 7 mantissa bits
    low = np.array([0x8000, 0x7FFF, 0x8001, 0x0000, 0xFFFF, 0x0001], dtype=np.uint32)
    lo = np.concatenate([np.resize(low, rows * 4), rng.integers(0, 1 << 16, size=rows * 4).astype(np.uint32)])
    sign = (rng.integers(0, 2, size=rows * 8).astype(np.uint32) << 31)
    bits = sign | (hi << 16) | lo
    bits[:8] = [0x3F808000, 0x3F818000, 0x3F807FFF, 0x3F808001, 0xBF808000, 0xBF818000, 0x7E7F8000, 0xFE7E8000]
    return torch.from_numpy(bits.view(np.float32).reshape(rows, 8).copy())


def _subnormal_cases(rows):
    """fp32 subnormals (exponent 0), which are also bf16 subnormals after rounding; ties and random low bits."""
    rng = np.random.default_rng(8)
    mant = rng.integers(1, 0x80, size=rows * 4).astype(np.uint32) << 16
    lo = np.concatenate([np.resize(np.array([0x8000, 0x7FFF, 0x8001], np.uint32), rows * 2),
                         rng.integers(0, 1 << 16, size=rows * 2).astype(np.uint32)])
    sign = (rng.integers(0, 2, size=rows * 4).astype(np.uint32) << 31)
    return torch.from_numpy((sign | mant | lo).view(np.float32).reshape(rows, 4).copy())


def test_gemm_bf16_rounding_is_rne_bit_for_bit(cuda):
    """C = I·B with a one-hot (identity) A: every output is one operand rounded by the kernel, times 1.0, plus zero products.
    It must equal torch's round-to-nearest-even bit for bit; a truncating or round-half-away conversion fails on the ties.
    Zeros are compared by value: the fp32 accumulator starts at +0 and adds +0 products, so a -0 operand comes out as +0
    whatever the conversion does."""
    from dance_b200 import ops
    K = 64
    normal = _rounding_cases(K)                                             # [K, 8]
    sub = _subnormal_cases(K)                                               # [K, 4]
    zeros = torch.tensor([0.0, -0.0]).repeat(K, 1)                          # [K, 2]
    filler = torch.randn(K, 128 - 14, generator=torch.Generator().manual_seed(3))
    B = torch.cat([normal, sub, zeros, filler], 1).contiguous().to(cuda)   # [K, 128]
    A = torch.eye(K, device=cuda)
    C = ops.gemm(A, B, precision="bf16")
    want = B.to(torch.bfloat16).float()
    keep = torch.ones(128, dtype=torch.bool)
    keep[12:14] = False
    assert torch.equal(C[:, keep].view(torch.int32), want[:, keep].view(torch.int32)), \
        f"{int((C[:, keep].view(torch.int32) != want[:, keep].view(torch.int32)).sum())} elements differ in their bits"
    assert torch.equal(C[:, 12:14], want[:, 12:14])
    # the subnormal columns are kept, not flushed: they match torch, which keeps them, and are not zero
    assert bool((C[:, 8:12] != 0).all())
    # the same B, transposed storage (the M/N-contiguous rewrite branch)
    Ct = ops.gemm(A, B.t().contiguous(), transB=True, precision="bf16")
    assert torch.equal(Ct.view(torch.int32)[:, keep], C.view(torch.int32)[:, keep])


@pytest.mark.parametrize("act", ["none", "relu", "elu", "tanh"])
@pytest.mark.parametrize("split", [False, True])
def test_gemm_bf16_epilogue(cuda, act, split):
    """bias, activation, ReLU mask and accumulate=True, with padded leading dimensions of A, B, C and the mask; on the
    tensor-core epilogue and through the split-K reduction."""
    from dance_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(11)
    M, N, K = (128, 256, 6000) if split else (1500, 900, 520)      # 2 output tiles → split-K; 96 tiles → one CTA per tile
    A = torch.randn(M, K + 4, device=cuda, generator=g)[:, :K]
    W = torch.randn(N, K + 8, device=cuda, generator=g)[:, :K]
    bias = torch.randn(N, device=cuda, generator=g)
    mask = torch.randn(M, N + 3, device=cuda, generator=g)[:, :N]
    C0 = torch.randn(M, N + 12, device=cuda, generator=g)
    assert (_ws_bytes(M, N, K, 0, 1) > 0) == split
    out = C0.clone()
    ops.gemm(A, W, transB=True, bias=bias, act=act, mask=mask, out=out[:, :N], accumulate=True, precision="bf16")

    def ref(prod):
        x = prod + bias.double()
        x = {"none": x, "relu": torch.relu(x), "elu": torch.nn.functional.elu(x), "tanh": torch.tanh(x)}[act]
        return x * (mask > 0) + C0[:, :N].double()
    exact = ref(bf16(A) @ bf16(W).t())
    assert rel_err(out[:, :N], exact) < TOL_EXACT
    # tanh at K = 6 000 turns the operand rounding of pre-activations near zero into larger output errors
    assert rel_err(out[:, :N], ref(A.double() @ W.double().t())) < (TOL_PLAIN_TANH if act == "tanh" else TOL_PLAIN)
    assert torch.equal(out[:, N:], C0[:, N:])                              # the padding is not written


@pytest.mark.parametrize("shape", [(128, 512, 12800), (1536, 1024, 512)])
def test_gemm_bf16_workspace_is_exact(cuda, shape):
    """b2_gemm_f32 called directly with a workspace of exactly b2_gemm_workspace_bytes(…, B2_PREC_BF16) bytes: B2_OK and the
    right result; on the split-K shape, one float less is refused with B2_ERR_WORKSPACE before anything runs."""
    from dance_b200 import ops
    M, N, K = shape
    g = torch.Generator(device=cuda).manual_seed(5)
    A = torch.randn(K, M, device=cuda, generator=g)                        # transA: the weight-gradient layout
    B = torch.randn(K, N, device=cuda, generator=g)
    nbytes = _ws_bytes(M, N, K, 1, 0)
    assert (nbytes > 0) == (K == 12800)
    C_out = torch.full((M, N), float("nan"), device=cuda)
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=cuda)
    lib = ops.lib()
    stream = torch.cuda.current_stream().cuda_stream

    def call(ws_bytes):
        return lib.b2_gemm_f32(A.data_ptr(), M, 1, B.data_ptr(), N, 0, C_out.data_ptr(), N, M, N, K, None, 0, None, 0,
                               C.c_float(0.0), ops.PREC["bf16"], ws.data_ptr() if nbytes else None, ws_bytes, stream)
    if nbytes:
        assert call(nbytes - 4) == -4                                      # B2_ERR_WORKSPACE
    assert call(nbytes) == 0                                               # B2_OK
    torch.cuda.synchronize()
    assert rel_err(C_out, bf16(A).t() @ bf16(B)) < TOL_EXACT


@pytest.mark.parametrize("case", ["small", "unaligned_pitch"])
def test_gemm_bf16_fallback_is_fp32(cuda, case):
    """Shapes the tensor-core kernel does not take run on the CUDA-core fp32 kernel in bf16 mode too: they match *plain* at
    fp32 accuracy, far closer than any bf16 rounding of the operands would allow."""
    from dance_b200 import ops
    g = torch.Generator(device=cuda).manual_seed(9)
    if case == "small":
        A = torch.randn(40, 50, device=cuda, generator=g)                  # M·N·K = 60 000 < 2^18
        B = torch.randn(50, 30, device=cuda, generator=g)
    else:
        A = torch.randn(300, 1999, device=cuda, generator=g)               # row pitch 1 999 floats: not a multiple of 16 B
        B = torch.randn(1999, 256, device=cuda, generator=g)
    C = ops.gemm(A, B, precision="bf16")
    plain = A.double() @ B.double()
    assert rel_err(C, plain) < 1e-6
    assert rel_err(bf16(A) @ bf16(B), plain) > 1e-4                        # what bf16 rounding would have cost
