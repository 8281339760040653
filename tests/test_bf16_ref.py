"""The bf16 restatement used by the GPU tests (tests/bf16_ref.py), checked on the CPU against explicit formulas."""
import numpy as np
import torch

from bf16_ref import Bf16MatMul, bf16, feature_ae_step_bf16
from oracle.scgnn_step_ref import FEATURE_AE_PARAMS, feature_ae_step


def _rne_bits(x32: np.ndarray) -> np.ndarray:
    """fp32 → bf16 round-to-nearest-even on the bit pattern, back as fp32 (finite inputs)."""
    u = x32.view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32)


def test_bf16_rounding_is_rne():
    rng = np.random.default_rng(0)
    bits = rng.integers(0x00800000, 0x7E800000, size=4096).astype(np.uint32)
    bits[:6] = [0x3F808000, 0x3F818000, 0x3F807FFF, 0x3F808001, 0x00018000, 0x00028000]     # ties (even / odd), ±1 ulp, subnormal ties
    x = bits.view(np.float32)
    got = bf16(torch.from_numpy(x)).numpy()
    assert np.array_equal(got.astype(np.float32).view(np.uint32), _rne_bits(x).view(np.uint32))
    assert got[0] == np.float32(1.0) and got[1] == np.float32(1.015625)      # 1 + 2^-8 (odd) ties up to 1 + 2^-7


def test_bf16_matmul_forward_and_backward():
    g = torch.Generator().manual_seed(1)
    a = torch.randn(7, 5, dtype=torch.float64, generator=g).requires_grad_()
    b = torch.randn(5, 3, dtype=torch.float64, generator=g).requires_grad_()
    w = torch.randn(7, 3, dtype=torch.float64, generator=g)
    out = Bf16MatMul.apply(a, b)
    ra, rb, rw = (t.detach().to(torch.bfloat16).double() for t in (a, b, w))
    assert torch.equal(out, ra @ rb)
    (out * w).sum().backward()
    assert torch.equal(a.grad, rw @ rb.t())
    assert torch.equal(b.grad, ra.t() @ rw)


def test_feature_ae_step_bf16_close_to_float64_step():
    """Same step as the float64 oracle up to the bf16 rounding of the products (8-bit mantissas: relative 2^-9 per operand)."""
    g = torch.Generator().manual_seed(2)
    dim, B, H, E = 48, 64, 32, 16
    shapes = {"fc1.weight": (H, dim), "fc1.bias": (H, ), "fc2.weight": (E, H), "fc2.bias": (E, ), "fc3.weight": (H, E),
              "fc3.bias": (H, ), "fc4.weight": (dim, H), "fc4.bias": (dim, )}
    params = {k: torch.randn(s, generator=g) * 0.3 for k, s in shapes.items()}
    x = torch.rand(B, dim, generator=g)
    got = feature_ae_step_bf16(x, params, "LTMG", 0.9, None)
    ref = feature_ae_step(x, params, "LTMG", 0.9, None)
    err = abs(got["loss"].item() - ref["loss"].item()) / ref["loss"].item()
    assert 1e-6 < err < 2e-2
    for k in FEATURE_AE_PARAMS:
        d = (got["grads"][k] - ref["grads"][k]).norm() / ref["grads"][k].norm()
        assert 0 < d < 5e-2, (k, float(d))
    # forward: z is relu(round(h1) · round(W2ᵀ) + b2), the explicit formula
    h1 = torch.relu(bf16(x) @ bf16(params["fc1.weight"]).t() + params["fc1.bias"].double())
    z = torch.relu(bf16(h1) @ bf16(params["fc2.weight"]).t() + params["fc2.bias"].double())
    assert torch.allclose(got["z"], z, rtol=0, atol=1e-12)
