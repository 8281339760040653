"""The triangle decoder's fp16 gradient products (gae_tri_f16_tc_kernel, the call over all rows) at the edges of fp16's range.

dZ_I += G·Z_J and dZ_J += Gᵀ·Z_I run as fp16 hi / lo products of G·2^14 and of each 64-row tile of z scaled by a power of two
chosen from the tile's largest |z|; the fp32 tile sums are unscaled exactly.  S, σ and softplus are the tf32 triangle's.  The
ordinary shapes and step splits are covered by test_gpu_decoder_triangle.py, whose "tc" path now runs this kernel; here:
embeddings far outside fp16's range, a tile mixing tiny and large rows, zero rows, one-hot rows whose products land in fp16
subnormals, and the same z through the tf32 triangle ("tc_tf32"), which must give the same loss and gradient."""
import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle.scgnn_step_ref import gae_reference_rows

pytestmark = pytest.mark.gpu


def _graph(cuda, n, seed):
    from dance_b200 import ops
    gen = torch.Generator(device=cuda).manual_seed(seed)
    idx = torch.randint(0, n, (n, 5), device=cuda, dtype=torch.int32, generator=gen)
    A = ops.knn_graph_build(idx.contiguous())
    return A, ops.CSR(A.rowptr, A.colidx, None, A.shape), gen


def _run(z, L, path, norm=0.5, pw=50.0):
    from dance_b200 import ops
    ops.set_path("gae", path)
    try:
        loss, dz, _, _ = ops.gae_loss_grad(z, L, norm, pw)
    finally:
        ops.set_path("gae", "auto")
    return loss.item(), dz


def _check(z, A, L, loss_tol, dz_tol):
    """against fp64, block by block.  For large |z| the tf32 S of both triangles decides σ of the logits near 0 with an
    absolute error that grows with |z|², so there the fp16 triangle may be as far from fp64 as the tf32 one, but no further."""
    n = z.shape[0]
    ref_loss, ref_dz = gae_reference_rows(z, A.rowptr, A.colidx, 0.5, 50.0, torch.arange(n, device=z.device))
    loss, dz = _run(z, L, "tc")
    _, dz32 = _run(z, L, "tc_tf32")
    assert bool(torch.isfinite(dz).all()) and np.isfinite(loss)
    assert abs(loss - ref_loss) <= loss_tol * abs(ref_loss), (loss, ref_loss)
    for b0 in [None] + list(range(0, n, 128)):
        blk = slice(None) if b0 is None else slice(b0, b0 + 128)
        err, err32 = rel_err(dz[blk], ref_dz[blk]), rel_err(dz32[blk], ref_dz[blk])
        assert err < max(dz_tol, 1.5 * err32), (b0, err, err32)


@pytest.mark.parametrize("scale", [3.0e4, 1.0e6])
@pytest.mark.parametrize("d", [8, 16, 32])
def test_f16_triangle_large_embeddings(cuda, d, scale):
    """|z| ~ 3·10⁴ and ~ 10⁶, where z itself is outside fp16's range: each tile is scaled into it"""
    n = 1500
    A, L, gen = _graph(cuda, n, n + d)
    z = (torch.randn(n, d, device=cuda, generator=gen) * scale).contiguous()
    _check(z, A, L, 5e-6, 5e-5)


@pytest.mark.parametrize("d", [8, 16, 32])
def test_f16_triangle_mixed_and_zero_rows(cuda, d):
    """64-row tiles that mix rows of norm 1e-4 and 1e4, and all-zero rows (a whole zero tile gets scale 1)"""
    n = 1300
    A, L, gen = _graph(cuda, n, 7 * n + d)
    z = torch.randn(n, d, device=cuda, generator=gen)
    z = z / z.norm(dim=1, keepdim=True)
    big = torch.rand(n, device=cuda, generator=gen) < 0.5
    z = z * torch.where(big, 1e4, 1e-4)[:, None]
    z[200:264] = 0.0            # one whole 64-row tile
    z[700:705] = 0.0
    z[1299] = 0.0
    _check(z.contiguous(), A, L, 5e-6, 5e-5)


@pytest.mark.parametrize("d", [8, 16, 32])
def test_f16_triangle_one_hot_rows(cuda, d):
    """one-hot rows: most logits are 0 (G = 1/2) and the lo halves of G·z are zero or fp16 subnormals"""
    n = 1100
    A, L, gen = _graph(cuda, n, 3 * n + d)
    hot = torch.randint(0, d, (n,), device=cuda, generator=gen)
    val = torch.where(torch.rand(n, device=cuda, generator=gen) < 0.5, 3e-3, 2.5)
    z = torch.zeros(n, d, device=cuda)
    z[torch.arange(n, device=cuda), hot] = val
    _check(z.contiguous(), A, L, 2e-6, 2e-5)


@pytest.mark.parametrize("scale", [0.3, 3.0e4])
@pytest.mark.parametrize("d", [8, 16, 32])
@pytest.mark.parametrize("n", [129, 1281, 8200])
def test_f16_triangle_matches_tf32_triangle(cuda, n, d, scale):
    """the same z through both triangles: S is the same tf32 product, so the loss differs only by the order of the atomic
    double adds; the gradients agree to 1e-6"""
    A, L, gen = _graph(cuda, n, n + 31 * d)
    z = (torch.randn(n, d, device=cuda, generator=gen) * scale / d ** 0.5).contiguous()
    loss16, dz16 = _run(z, L, "tc")
    loss32, dz32 = _run(z, L, "tc_tf32")
    assert abs(loss16 - loss32) <= 1e-12 * abs(loss32), (loss16, loss32)
    assert rel_err(dz16, dz32) < 1e-6
