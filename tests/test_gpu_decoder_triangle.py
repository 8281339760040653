"""The triangle sweep of the tensor-core decoder (gae_tri_tc_kernel, the call over all rows) against the fp64 closed form.

Block I sweeps only the 64-column J tiles on and above its diagonal block; each tile above it counts its loss twice and adds
dZ_J += Gᵀ·Z_I into the rows of block J with atomics.  These cases cover a single partial block, exact multiples of 128 and one
past them, odd and even block counts, J sweeps cut into step ranges (including more ranges than some blocks have tiles),
embeddings of |z| ~ 3·10⁴, and that nothing is written past row n."""
import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle.scgnn_step_ref import gae_reference_rows

pytestmark = pytest.mark.gpu


def _problem(cuda, n, d, scale, seed):
    from dance_b200 import ops
    gen = torch.Generator(device=cuda).manual_seed(seed)
    z = (torch.randn(n, d, device=cuda, generator=gen) * scale).contiguous()
    idx = torch.randint(0, n, (n, 5), device=cuda, dtype=torch.int32, generator=gen)
    A = ops.knn_graph_build(idx.contiguous())
    return z, A, ops.CSR(A.rowptr, A.colidx, None, A.shape)


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
    """|z| ~ 3·10⁴: the tf32 hi / lo split of G and Z_I keeps the transposed product as exact as the row product."""
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
