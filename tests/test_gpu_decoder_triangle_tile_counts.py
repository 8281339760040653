"""The triangle sweep (gae_tri_tc_kernel) at every J-tile count a CTA can have from 1 to 5, against the fp64 closed form.

At DP = 8 the consumer loop alternates S between two accumulators and is unrolled by two, so an even and an odd number of
tiles after the first end in different code (which accumulator the last dZ reads), and one tile takes neither turn.  With
n_jt = 10 64-column tiles (5 row blocks, the last one partial for n = 600) block I has 10 − 2·I tiles; cut into two step ranges,
the CTAs of blocks 0 .. 4 sweep 5, 4, 3, 2 and 1 tiles.  DP = 16 and 32 run the same cases through their own schedule."""
import numpy as np
import pytest
import torch

from conftest import rel_err
from oracle.scgnn_step_ref import gae_reference_rows

pytestmark = pytest.mark.gpu


def _tiles_per_cta(n, splits):
    """J tiles of each non-empty CTA, as decoder_sweep splits a block's sweep (see test_decoder_triangle_schedule.py)"""
    nb, n_jt = -(-n // 128), -(-n // 64)
    out = []
    for blk in range(nb):
        first = 2 * blk
        per = -(-(n_jt - first) // splits)
        for y in range(splits):
            jt0 = first + y * per
            if jt0 < n_jt:
                out.append(min(n_jt, jt0 + per) - jt0)
    return out


def _run(cuda, n, d, scale, splits, seed):
    from dance_b200 import ops
    gen = torch.Generator(device=cuda).manual_seed(seed)
    z = (torch.randn(n, d, device=cuda, generator=gen) * scale).contiguous()
    idx = torch.randint(0, n, (n, 5), device=cuda, dtype=torch.int32, generator=gen)
    A = ops.knn_graph_build(idx.contiguous())
    L = ops.CSR(A.rowptr, A.colidx, None, A.shape)
    ops.set_path("gae", "tc")
    try:
        ops.set_tuning("gae_splits", splits)
        loss, dz, _, _ = ops.gae_loss_grad(z, L, 0.5, 45.0)
    finally:
        ops.set_tuning("gae_splits", 0)
        ops.set_path("gae", "auto")
    ref_loss, ref_dz = gae_reference_rows(z, A.rowptr, A.colidx, 0.5, 45.0, torch.arange(n, device=cuda))
    return loss.item(), dz, ref_loss, ref_dz


@pytest.mark.parametrize("n", [600, 640])
def test_cases_cover_one_to_five_tiles(n):
    assert set(_tiles_per_cta(n, 2)) == {1, 2, 3, 4, 5}


@pytest.mark.parametrize("d", [8, 16, 32])
@pytest.mark.parametrize("n", [600, 640])
def test_triangle_every_tile_count(cuda, n, d):
    loss, dz, ref_loss, ref_dz = _run(cuda, n, d, 0.9 / d ** 0.5, 2, 31 * n + d)
    assert abs(loss - ref_loss) < 2e-6 * abs(ref_loss), (loss, ref_loss)
    assert rel_err(dz, ref_dz) < 2e-5
    for b in range(-(-n // 128)):      # block by block, so that one wrong CTA is not averaged away
        assert rel_err(dz[128 * b:128 * b + 128], ref_dz[128 * b:128 * b + 128]) < 2e-5, b


@pytest.mark.parametrize("d", [8, 16, 32])
def test_triangle_every_tile_count_large_embedding(cuda, d):
    """|z| ~ 3·10⁴ through the same tile counts"""
    loss, dz, ref_loss, ref_dz = _run(cuda, 600, d, 3.0e4, 2, 7 + d)
    assert bool(torch.isfinite(dz).all()) and np.isfinite(loss)
    assert abs(loss - ref_loss) < 5e-6 * abs(ref_loss), (loss, ref_loss)
    assert rel_err(dz, ref_dz) < 5e-5
