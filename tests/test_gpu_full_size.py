"""Size-independent properties at BASELINE.json's full headline size (1 M cells): the oracle cannot reach this size, so the
checks are invariants — sortedness / idempotence of the exact kNN, symmetry and the D^-1/2 fixed point of the normalised
graph, linearity of the aggregate, additivity of the row-sharded decoder loss.
The decoder is additionally checked in absolute terms on sampled rows against the fp64 closed form."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

N, D, K = 1_000_000, 128, 15


@pytest.fixture(scope="module")
def embedding(cuda):
    gen = torch.Generator(device=cuda).manual_seed(0)
    centres = torch.randn(10, D, device=cuda, generator=gen) * 3
    lab = torch.randint(0, 10, (N, ), device=cuda, generator=gen)
    return torch.randn(N, D, device=cuda, generator=gen) + centres[lab]


def test_knn_graph_invariants_at_one_million_cells(cuda, embedding):
    from dance_b200 import ops
    idx, dist = ops.knn(embedding, K)
    assert idx.shape == (N, K) and int(idx.min()) >= 0 and int(idx.max()) < N
    assert bool((dist[:, 1:] >= dist[:, :-1]).all())                              # ranked by fp64 distance
    assert not bool((idx == torch.arange(N, device=cuda, dtype=idx.dtype).unsqueeze(1)).any())   # rank 0 (self) dropped
    idx2, _ = ops.knn(embedding, K, return_dist=False)
    assert torch.equal(idx, idx2)                                                 # deterministic / idempotent
    part, _ = ops.knn(embedding, K, q_begin=250_000, q_end=500_000, return_dist=False)
    assert torch.equal(part, idx[250_000:500_000])                                # the multi-GPU query sharding
    A = ops.knn_graph_build(idx)
    assert A.nnz >= N * (K + 1) and A.nnz <= N * (2 * K + 1)
    At, _ = ops.csr_transpose(A)
    assert torch.equal(At.rowptr, A.rowptr) and torch.equal(At.colidx, A.colidx)  # Â is symmetric …
    assert torch.allclose(At.vals, A.vals, rtol=1e-6, atol=0)                     # … in its values too
    deg = (A.rowptr[1:] - A.rowptr[:-1]).float().sqrt().unsqueeze(1).repeat(1, 4).contiguous()
    out = ops.spmm(A, deg)                                                        # D^-1/2 (A+I) D^-1/2 · sqrt(deg) = sqrt(deg)
    assert float((out - deg).abs().max() / deg.abs().max()) < 1e-4                # fp32 sums over hub rows of several thousand entries
    x, y = embedding[:, :32].contiguous(), embedding[:, 32:64].contiguous()
    lin = ops.spmm(A, 2 * x + y)
    ref = 2 * ops.spmm(A, x) + ops.spmm(A, y)
    assert float((lin - ref).norm() / ref.norm()) < 1e-4                          # linearity of the aggregate (fp32 rounding of 2x+y)


def test_decoder_loss_additive_over_row_shards_at_one_million_cells(cuda, embedding):
    from dance_b200 import ops
    gen = torch.Generator(device=cuda).manual_seed(1)
    idx = torch.randint(0, N, (N, K), device=cuda, dtype=torch.int32, generator=gen)
    A = ops.knn_graph_build(idx.contiguous())
    z = (embedding[:, :16] * 0.1).contiguous()
    L = ops.CSR(A.rowptr, A.colidx, None, A.shape)
    full, dz, _, _ = ops.gae_loss_grad(z, L, 0.5, 100.0)
    h = 437_519
    rp = A.rowptr.long()
    top = ops.CSR(A.rowptr[:h + 1].contiguous(), A.colidx[:rp[h]].contiguous(), None, (h, N))
    bot = ops.CSR((A.rowptr[h:] - A.rowptr[h]).contiguous(), A.colidx[rp[h]:].contiguous(), None, (N - h, N))
    la, dza, _, _ = ops.gae_loss_grad(z, top, 0.5, 100.0, row_begin=0, n_rows=h)
    lb, dzb, _, _ = ops.gae_loss_grad(z, bot, 0.5, 100.0, row_begin=h, n_rows=N - h)
    assert abs(la.item() + lb.item() - full.item()) < 1e-5 * abs(full.item())
    both = torch.cat([dza, dzb])
    # the row-sharded calls split the J sweep differently from the full call (other CTA counts, other summation order); the fp64
    # rows below are the arbiter
    assert float((both - dz).norm() / dz.norm()) < 2e-3
    assert np.isfinite(full.item())
    # absolute check of the exact path the benchmark times: sampled rows against the fp64 closed form
    from test_gpu_kernels import gae_reference_rows
    rows = torch.tensor([0, 1, 127, 128, 4097, 437_518, 437_519, 999_999] + list(range(600_000, 600_056)), device=cuda)
    _, ref_rows = gae_reference_rows(z, A.rowptr, A.colidx, 0.5, 100.0, rows)
    err = float((dz[rows].double() - ref_rows).norm() / ref_rows.norm())
    assert err < 2e-5, err
