"""The triangle sweep of the tensor-core decoder (gae_tri_tc_kernel, the call over all rows) against the fp64 closed form and
against the full sweep.

Block I sweeps only the 64-column J tiles on and above its diagonal block; each tile above it counts its loss twice and adds
dZ_J += Gᵀ·Z_I into the rows of block J with atomics.  dZ_I += G·Z_J and dZ_J run as fp16 hi / lo products of G·2^14 and of
each 64-row tile of z scaled by a power of two chosen from the tile's largest |z|; the fp32 tile sums are unscaled exactly.
These cases cover a single partial block, exact multiples of 128 and one past them, odd and even block counts, J sweeps cut
into step ranges (including more ranges than some blocks have tiles), that nothing is written past row n, and the edges of
fp16's range: embeddings of |z| ~ 3·10⁴ and 10⁶ (z itself outside it), tiles mixing tiny and large rows, zero rows, and
one-hot rows whose products land in fp16 subnormals.

The full sweep (gae_allpairs_tc_kernel) is the same rows as two row-shard calls split at a block boundary, as
benchmarks/decoder.py runs it.  It shares the triangle's S and σ / softplus but none of its tiles, transposed products, fp16
gradient products or schedule, so the two check each other on the same z."""
import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle.scgnn_step_ref import gae_reference_rows

pytestmark = pytest.mark.gpu


def _graph(n, gen):
    from dance_b200 import ops
    idx = torch.randint(0, n, (n, 5), device=gen.device, dtype=torch.int32, generator=gen)
    A = ops.knn_graph_build(idx.contiguous())
    return A, ops.CSR(A.rowptr, A.colidx, None, A.shape)


def _problem(cuda, n, d, scale, seed):
    gen = torch.Generator(device=cuda).manual_seed(seed)
    z = (torch.randn(n, d, device=cuda, generator=gen) * scale).contiguous()
    return (z, *_graph(n, gen))


def _run(z, L, norm, pw, splits=0, dz=None):
    from dance_b200 import ops
    ops.set_path("gae", "tc")
    try:
        ops.set_tuning("gae_splits", splits)
        loss, dz, _, _ = ops.gae_loss_grad(z, L, norm, pw, dz=dz)
    finally:
        ops.set_tuning("gae_splits", 0)
        ops.set_path("gae", "auto")
    return loss.item(), dz


def _full_sweep(z, A, norm, pw):
    """the same rows as two row-shard calls (the full sweep), split at a block boundary near the middle"""
    from dance_b200 import ops
    n = z.shape[0]
    h = max(128, (n // 2) // 128 * 128)
    rp = A.rowptr.long()
    top = ops.CSR(A.rowptr[:h + 1].contiguous(), A.colidx[:rp[h]].contiguous(), None, (h, n))
    bot = ops.CSR((A.rowptr[h:] - A.rowptr[h]).contiguous(), A.colidx[rp[h]:].contiguous(), None, (n - h, n))
    ops.set_path("gae", "tc")
    try:
        loss_t, dz_t, _, _ = ops.gae_loss_grad(z, top, norm, pw, row_begin=0, n_rows=h)
        loss_b, dz_b, _, _ = ops.gae_loss_grad(z, bot, norm, pw, row_begin=h, n_rows=n - h)
    finally:
        ops.set_path("gae", "auto")
    return loss_t.item() + loss_b.item(), torch.cat([dz_t, dz_b])


def _block_rows(n):
    """every row of the first, a middle and the last 128-row block"""
    nb = (n + 127) // 128
    return sorted({r for b in (0, nb // 2, nb - 1) for r in range(128 * b, min(n, 128 * b + 128))})


@pytest.mark.parametrize("d", [8, 16, 32])
@pytest.mark.parametrize("n", [100, 128, 129, 255, 256, 1281, 8200])
def test_gae_triangle_matches_fp64(cuda, n, d):
    z, A, L = _problem(cuda, n, d, 0.9 / d ** 0.5, n * 13 + d)
    norm, pw = 0.5, 40.0
    rows = torch.arange(n, device=cuda) if n <= 1281 else torch.tensor(_block_rows(n), device=cuda)
    ref_loss, _ = gae_reference_rows(z, A.rowptr, A.colidx, norm, pw, torch.arange(n, device=cuda))
    _, ref_rows = gae_reference_rows(z, A.rowptr, A.colidx, norm, pw, rows)
    loss, dz = _run(z, L, norm, pw)
    assert abs(loss - ref_loss) < 2e-6 * abs(ref_loss), (loss, ref_loss)
    assert rel_err(dz[rows], ref_rows) < 2e-5
    # block by block, so that an error confined to one block is not averaged away
    br = _block_rows(n)
    pos = {r: i for i, r in enumerate(rows.tolist())}
    for b0 in sorted({r // 128 for r in br}):
        sel = [pos[r] for r in br if r // 128 == b0]
        assert rel_err(dz[rows[sel]], ref_rows[sel]) < 2e-5, b0


@pytest.mark.parametrize("n,d,splits", [(1281, 16, 1), (1281, 16, 2), (1281, 32, 7), (8200, 8, 2), (8200, 16, 7),
                                        (2049, 16, 40), (1281, 8, 1000)])
def test_gae_triangle_step_splits(cuda, n, d, splits):
    """J sweeps cut into step ranges: with 40 and 1000 ranges most blocks have fewer tiles than ranges (empty CTAs)."""
    z, A, L = _problem(cuda, n, d, 0.5, n + 17 * splits + d)
    norm, pw = 0.5, 55.0
    rows = torch.tensor(_block_rows(n), device=cuda)
    ref_loss, _ = gae_reference_rows(z, A.rowptr, A.colidx, norm, pw, torch.arange(n, device=cuda))
    _, ref_rows = gae_reference_rows(z, A.rowptr, A.colidx, norm, pw, rows)
    loss1, dz1 = _run(z, L, norm, pw, splits=1)
    loss, dz = _run(z, L, norm, pw, splits=splits)
    assert abs(loss - ref_loss) < 2e-6 * abs(ref_loss), (loss, ref_loss)
    assert rel_err(dz[rows], ref_rows) < 2e-5
    assert rel_err(dz, dz1) < 2e-6 and abs(loss - loss1) < 2e-6 * abs(loss1)


@pytest.mark.parametrize("d", [16, 32])
def test_gae_triangle_large_embedding(cuda, d):
    """|z| ~ 3·10⁴: the per-tile scale and the fp16 hi / lo split of G and Z_I keep the transposed product as exact as the row
    product."""
    n = 3000
    z, A, L = _problem(cuda, n, d, 3.0e4, n + d)
    ref_loss, ref_dz = gae_reference_rows(z, A.rowptr, A.colidx, 0.5, 50.0, torch.arange(n, device=cuda))
    loss, dz = _run(z, L, 0.5, 50.0)
    assert bool(torch.isfinite(dz).all()) and np.isfinite(loss)
    assert abs(loss - ref_loss) < 5e-6 * abs(ref_loss), (loss, ref_loss)
    assert rel_err(dz, ref_dz) < 5e-5


@pytest.mark.parametrize("n,d,shift", [(129, 16, 0), (1281, 32, 0), (1300, 8, 1)])
def test_gae_triangle_writes_only_rows_below_n(cuda, n, d, shift):
    """dz handed in as n rows inside a larger buffer: the elements after them (the rest of the last J tile and a whole row block
    past n) and the one before keep their contents.  shift = 1 puts dz at an odd float offset, where the dZ_J rows are added
    with scalar instead of 64-bit atomics."""
    z, A, L = _problem(cuda, n, d, 0.4, 5 * n + d)
    flat = torch.full(((n + 256) * d + 1,), 1234.5, device=cuda)
    loss, dz = _run(z, L, 0.5, 30.0, dz=flat[shift:shift + n * d].view(n, d))
    assert dz.data_ptr() == flat.data_ptr() + 4 * shift
    assert bool((flat[:shift] == 1234.5).all()) and bool((flat[shift + n * d:] == 1234.5).all())
    ref_loss, ref_dz = gae_reference_rows(z, A.rowptr, A.colidx, 0.5, 30.0, torch.arange(n, device=cuda))
    assert abs(loss - ref_loss) < 2e-6 * abs(ref_loss), (loss, ref_loss)
    assert rel_err(dz, ref_dz) < 2e-5


def _check(z, A, L, loss_tol, dz_tol):
    """against fp64, block by block.  For large |z| the tf32 S decides σ of the logits near 0 with an absolute error that grows
    with |z|², so there the triangle may be as far from fp64 as the full sweep, which computes the same S, but no further."""
    n = z.shape[0]
    ref_loss, ref_dz = gae_reference_rows(z, A.rowptr, A.colidx, 0.5, 50.0, torch.arange(n, device=z.device))
    loss, dz = _run(z, L, 0.5, 50.0)
    _, dz_full = _full_sweep(z, A, 0.5, 50.0)
    assert bool(torch.isfinite(dz).all()) and np.isfinite(loss)
    assert abs(loss - ref_loss) <= loss_tol * abs(ref_loss), (loss, ref_loss)
    for b0 in [None] + list(range(0, n, 128)):
        blk = slice(None) if b0 is None else slice(b0, b0 + 128)
        err, err_full = rel_err(dz[blk], ref_dz[blk]), rel_err(dz_full[blk], ref_dz[blk])
        assert err < max(dz_tol, 1.5 * err_full), (b0, err, err_full)


@pytest.mark.parametrize("scale", [3.0e4, 1.0e6])
@pytest.mark.parametrize("d", [8, 16, 32])
def test_gae_triangle_outside_fp16_range(cuda, d, scale):
    """|z| ~ 3·10⁴ and ~ 10⁶, where z itself is outside fp16's range: each tile is scaled into it"""
    n = 1500
    gen = torch.Generator(device=cuda).manual_seed(n + d)
    A, L = _graph(n, gen)
    z = (torch.randn(n, d, device=cuda, generator=gen) * scale).contiguous()
    _check(z, A, L, 5e-6, 5e-5)


@pytest.mark.parametrize("d", [8, 16, 32])
def test_gae_triangle_mixed_and_zero_rows(cuda, d):
    """64-row tiles that mix rows of norm 1e-4 and 1e4, and all-zero rows (a whole zero tile gets scale 1)"""
    n = 1300
    gen = torch.Generator(device=cuda).manual_seed(7 * n + d)
    A, L = _graph(n, gen)
    z = torch.randn(n, d, device=cuda, generator=gen)
    z = z / z.norm(dim=1, keepdim=True)
    big = torch.rand(n, device=cuda, generator=gen) < 0.5
    z = z * torch.where(big, 1e4, 1e-4)[:, None]
    z[200:264] = 0.0            # one whole 64-row tile
    z[700:705] = 0.0
    z[1299] = 0.0
    _check(z.contiguous(), A, L, 5e-6, 5e-5)


@pytest.mark.parametrize("d", [8, 16, 32])
def test_gae_triangle_one_hot_rows(cuda, d):
    """one-hot rows: most logits are 0 (G = 1/2) and the lo halves of G·z are zero or fp16 subnormals"""
    n = 1100
    gen = torch.Generator(device=cuda).manual_seed(3 * n + d)
    A, L = _graph(n, gen)
    hot = torch.randint(0, d, (n,), device=cuda, generator=gen)
    val = torch.where(torch.rand(n, device=cuda, generator=gen) < 0.5, 3e-3, 2.5)
    z = torch.zeros(n, d, device=cuda)
    z[torch.arange(n, device=cuda), hot] = val
    _check(z.contiguous(), A, L, 2e-6, 2e-5)


@pytest.mark.parametrize("n,d,splits,scale",
                         [(n, d, 0, scale) for n in (129, 1281, 8200) for d in (8, 16, 32) for scale in (0.3, 3.0e4)]
                         + [(129, 16, 1, 0.9), (129, 16, 2, 0.9), (1281, 16, 1, 0.9), (1281, 16, 3, 0.9), (8200, 16, 1, 0.9),
                            (8200, 16, 7, 0.9), (1281, 16, 2, 1.2e5)])
def test_triangle_matches_full_sweep(cuda, n, d, splits, scale):
    """the same z (rows of norm ~ scale) through the triangle, with its J sweeps cut into `splits` step ranges (0: automatic),
    and through the full sweep.  The gradients agree to 1e-6, except at n = 8200 with small |z|, where the full sweep's own
    error against fp64 grows to 1e-6 (the triangle's stays below 4e-7); the losses to 2e-7."""
    gen = torch.Generator(device=cuda).manual_seed(n * 31 + 7 * d + splits)
    A, L = _graph(n, gen)
    z = (torch.randn(n, d, device=cuda, generator=gen) * scale / d ** 0.5).contiguous()
    norm, pw = 0.5, 40.0
    ref_loss, _ = gae_reference_rows(z, A.rowptr, A.colidx, norm, pw, torch.arange(n, device=cuda))
    loss, dz = _run(z, L, norm, pw, splits=splits)
    loss_full, dz_full = _full_sweep(z, A, norm, pw)
    assert bool(torch.isfinite(dz).all()) and np.isfinite(loss)
    assert abs(loss - ref_loss) < (2e-6 if scale < 1 else 5e-6) * abs(ref_loss), (loss, ref_loss)
    assert abs(loss - loss_full) < 2e-7 * abs(loss_full), (loss, loss_full)
    tol = 1e-6 if n < 8200 or scale > 1 else {8: 4e-6, 16: 3e-6, 32: 2e-6}[d]
    assert rel_err(dz, dz_full) < tol
    # block by block, so that an error confined to one block is not averaged away
    for b0 in range(0, n, 128):
        assert rel_err(dz[b0:b0 + 128], dz_full[b0:b0 + 128]) < tol, b0
