"""Interior and edge tiles of the tensor-core decoder at d = 8 and d = 32.

The kernel evaluates a J tile without the per-logit mask when all 128 columns are real (j < n) and every row of its 128-row
block is in range, and with the mask otherwise.  These cases put both kinds next to each other: n a multiple of 128 (no ragged
J tile) and one past it (a last tile with a single live column), a row range that starts in the middle of a block and ends in
the middle of another, and J sweeps cut into step ranges of one and two tiles (the first tile of a sweep is also its last)."""
import pytest
import torch

from conftest import rel_err
from oracle.scgnn_step_ref import gae_reference_rows

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("d", [8, 32])
@pytest.mark.parametrize("n", [1280, 1281])
@pytest.mark.parametrize("splits", [1, 3, 10])
def test_gae_tc_interior_and_edge_tiles(cuda, d, n, splits):
    from dance_b200 import ops
    gen = torch.Generator(device=cuda).manual_seed(n * 7 + d + splits)
    z = (torch.randn(n, d, device=cuda, generator=gen) * (0.9 / d ** 0.5)).contiguous()
    idx = torch.randint(0, n, (n, 5), device=cuda, dtype=torch.int32, generator=gen)
    A = ops.knn_graph_build(idx.contiguous())
    norm, pw = 0.5, 40.0
    r0, r1 = 200, n - 75                 # starts 72 rows into block 1, ends inside the last full block
    rp = A.rowptr.long()
    sub = ops.CSR((A.rowptr[r0:r1 + 1] - A.rowptr[r0]).contiguous(), A.colidx[rp[r0]:rp[r1]].contiguous(), None, (r1 - r0, n))
    full = ops.CSR(A.rowptr, A.colidx, None, A.shape)
    ref_loss, ref_dz = gae_reference_rows(z, A.rowptr, A.colidx, norm, pw, torch.arange(n, device=cuda))
    ref_sub, _ = gae_reference_rows(z, A.rowptr, A.colidx, norm, pw, torch.arange(r0, r1, device=cuda))
    ops.set_path("gae", "tc")
    try:
        ops.set_tuning("gae_splits", splits)
        loss, dz, _, _ = ops.gae_loss_grad(z, full, norm, pw)
        loss_s, dz_s, _, _ = ops.gae_loss_grad(z, sub, norm, pw, row_begin=r0, n_rows=r1 - r0)
    finally:
        ops.set_tuning("gae_splits", 0)
        ops.set_path("gae", "auto")
    assert abs(loss.item() - ref_loss) < 2e-6 * abs(ref_loss), (loss.item(), ref_loss)
    assert rel_err(dz, ref_dz) < 2e-5
    assert abs(loss_s.item() - ref_sub) < 2e-6 * abs(ref_sub), (loss_s.item(), ref_sub)
    assert rel_err(dz_s, ref_dz[r0:r1]) < 2e-5
    # every row of the range, including the first and last ones of the partial blocks
    for rows in (slice(0, 56), slice(r1 - r0 - 53, r1 - r0)):
        assert rel_err(dz_s[rows], ref_dz[r0:r1][rows]) < 2e-5
