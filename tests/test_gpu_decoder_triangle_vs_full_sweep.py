"""The d = 16 triangle (gae_tri_tc_kernel, the call over all rows) against the full sweep (gae_allpairs_tc_kernel) on the same z.

The full sweep is the same rows as two row-shard calls split at a block boundary, as benchmarks/decoder.py runs it; it shares
the triangle's workspace planes and elementwise math but none of its tiles, transposed products or schedule, so the two check
each other at the width the benchmark runs.  The cases cover a single-tile block (n = 129), odd and even tile counts, J sweeps
cut into step ranges and an embedding of |z| ~ 3·10⁴; the tolerances are those of the fp64 tests in
test_gpu_decoder_triangle.py."""
import numpy as np
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu

D = 16


def _full_sweep(z, A, norm, pw):
    from dance_b200 import ops
    n = z.shape[0]
    h = max(128, (n // 2) // 128 * 128)
    rp = A.rowptr.long()
    top = ops.CSR(A.rowptr[:h + 1].contiguous(), A.colidx[:rp[h]].contiguous(), None, (h, n))
    bot = ops.CSR((A.rowptr[h:] - A.rowptr[h]).contiguous(), A.colidx[rp[h]:].contiguous(), None, (n - h, n))
    loss_t, dz_t, _, _ = ops.gae_loss_grad(z, top, norm, pw, row_begin=0, n_rows=h)
    loss_b, dz_b, _, _ = ops.gae_loss_grad(z, bot, norm, pw, row_begin=h, n_rows=n - h)
    return loss_t.item() + loss_b.item(), torch.cat([dz_t, dz_b])


@pytest.mark.parametrize("n,splits,scale,tol", [(129, 1, 0.225, 2e-5), (129, 2, 0.225, 2e-5), (1281, 1, 0.225, 2e-5),
                                                (1281, 3, 0.225, 2e-5), (8200, 1, 0.225, 2e-5), (8200, 7, 0.225, 2e-5),
                                                (1281, 2, 3.0e4, 5e-5)])
def test_triangle_matches_full_sweep_d16(cuda, n, splits, scale, tol):
    from dance_b200 import ops
    gen = torch.Generator(device=cuda).manual_seed(n * 31 + splits)
    z = (torch.randn(n, D, device=cuda, generator=gen) * scale).contiguous()
    idx = torch.randint(0, n, (n, 5), device=cuda, dtype=torch.int32, generator=gen)
    A = ops.knn_graph_build(idx.contiguous())
    L = ops.CSR(A.rowptr, A.colidx, None, A.shape)
    norm, pw = 0.5, 40.0
    ops.set_path("gae", "tc")
    try:
        ref_loss, ref_dz = _full_sweep(z, A, norm, pw)
        ops.set_tuning("gae_splits", splits)
        loss, dz, _, _ = ops.gae_loss_grad(z, L, norm, pw)
        loss = loss.item()
    finally:
        ops.set_tuning("gae_splits", 0)
        ops.set_path("gae", "auto")
    assert bool(torch.isfinite(dz).all()) and np.isfinite(loss)
    assert abs(loss - ref_loss) < tol / 10 * abs(ref_loss), (loss, ref_loss)
    assert rel_err(dz, ref_dz) < tol
    if scale < 1:
        # block by block, so that an error confined to one block is not averaged away
        for b0 in range(0, n, 128):
            assert rel_err(dz[b0:b0 + 128], ref_dz[b0:b0 + 128]) < tol, b0
