"""The library's paths that launch kernels with more than 48 KB of dynamic shared memory, run in one process on device 0 and then
on device 1.

A kernel must opt in to such a size, and the opt-in belongs to the kernel as loaded on one device: a library that opted in once
per process would launch on the second device without it, and the launch would fail.  Each path below runs on device 0, then
on device 1 with the same inputs, and the two results agree to the tolerance the operation's own tests use."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from conftest import rel_err

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two CUDA devices")]


def _gemm(dev, rng):
    """tf32x3 tensor-core GEMM, BN = 128 (the whole 227 KB budget)"""
    from dance_b200 import ops
    A, B = rng.normal(size=(1000, 2000)).astype(np.float32), rng.normal(size=(2000, 512)).astype(np.float32)
    return ops.gemm(torch.from_numpy(A).to(dev), torch.from_numpy(B).to(dev), precision="tf32x3")


def _gae(dev, rng):
    """tensor-core decoder, n² ≥ 2²²: the triangle (all rows) and the full sweep (a row shard)"""
    from dance_b200 import ops
    n, d, h = 2500, 16, 1280
    z = torch.from_numpy(rng.normal(size=(n, d)).astype(np.float32)).to(dev)
    A = ops.knn_graph_build(torch.from_numpy(rng.integers(0, n, (n, 5), dtype=np.int32)).to(dev))
    L = ops.CSR(A.rowptr, A.colidx, None, A.shape)
    top = ops.CSR(A.rowptr[:h + 1].contiguous(), A.colidx[:int(A.rowptr[h])].contiguous(), None, (h, n))
    ops.set_path("gae", "tc")
    try:
        loss, dz, _, _ = ops.gae_loss_grad(z, L, 0.7, 3.0)
        loss_t, dz_t, _, _ = ops.gae_loss_grad(z, top, 0.7, 3.0, row_begin=0, n_rows=h)
    finally:
        ops.set_path("gae", "auto")
    return loss, dz, loss_t, dz_t


def _knn(dev, rng):
    """n·n_q ≥ 2²⁴: the tensor-core candidate filter, then the SIMT one"""
    from dance_b200 import ops
    X = torch.from_numpy(rng.normal(size=(4500, 16)).astype(np.float32)).to(dev)
    idx, dist = ops.knn(X, 10)
    ops.set_path("knn", "simt")
    try:
        idx_s, dist_s = ops.knn(X, 10)
    finally:
        ops.set_path("knn", "auto")
    return idx, dist, idx_s, dist_s


def _spmm(dev, rng):
    """fp32, F = 32: 128-byte operand rows take the nnz-stream kernel"""
    from dance_b200 import ops
    n, c = 20_000, 15_000
    rows = np.repeat(np.arange(n), rng.integers(0, 60, n))
    m = sp.csr_matrix((rng.normal(size=rows.size).astype(np.float32), (rows, rng.integers(0, c, rows.size))), shape=(n, c))
    m.sum_duplicates()
    X = torch.from_numpy(rng.normal(size=(c, 32)).astype(np.float32)).to(dev)
    return ops.spmm(ops.CSR.from_scipy(m, dev), X)


def _kmeans(dev, rng):
    """k·d·4 = 60 000 bytes of centres in shared memory"""
    from dance_b200 import ops
    k, d = 100, 150
    X = torch.from_numpy((rng.normal(size=(3000, d)) + rng.integers(0, k, size=(3000, 1)) * 2.5).astype(np.float32)).to(dev)
    labels, inertia, _ = ops.kmeans(X, X[:k].clone(), max_iter=5)
    return labels, inertia


def _spatial(dev, rng):
    """exp-adjacency product at N = 64 (X of 64 columns, non-negative so that W·|X| = W·X)"""
    from dance_b200 import spatial_ops
    P = torch.from_numpy(rng.uniform(0, 100, size=(3000, 2)).astype(np.float32)).to(dev)
    X = torch.from_numpy(rng.uniform(0, 1, size=(3000, 64)).astype(np.float32)).to(dev)
    return spatial_ops.spatial_exp_adj_matmul(P, P, 20.0, X)


def _agree_gemm(a, b):
    assert rel_err(b, a) < 1e-5


def _agree_gae(a, b):
    for loss, dz, loss1, dz1 in ((a[0], a[1], b[0], b[1]), (a[2], a[3], b[2], b[3])):
        assert abs(loss1.item() - loss.item()) < 2e-6 * abs(loss.item()) and rel_err(dz1, dz) < 2e-6


def _agree_knn(a, b):
    for x, y in zip(a, b):
        assert torch.equal(x.cpu(), y.cpu())                  # indices and fp64 distances: bit-exact


def _agree_spmm(a, b):
    assert rel_err(b, a) < 1e-6


def _agree_kmeans(a, b):
    assert (a[0].cpu() == b[0].cpu()).double().mean() > 0.999 and abs(b[1] - a[1]) < 1e-3 * a[1]


def _agree_spatial(a, b):
    # each device is within the operation's bound, 4 · 2⁻²¹ · W·|X| per element, of the exact product (W·|X| = W·X here)
    a, b = a.double().cpu(), b.double().cpu()
    assert bool(((b - a).abs() <= 2.0**-18 * a).all())


PATHS = {"gemm_tc": (_gemm, _agree_gemm), "gae_tc": (_gae, _agree_gae), "knn": (_knn, _agree_knn), "spmm_stream": (_spmm, _agree_spmm),
         "kmeans": (_kmeans, _agree_kmeans), "spatial_exp_adj_matmul": (_spatial, _agree_spatial)}


@pytest.mark.parametrize("path", PATHS)
def test_second_device_after_the_first(cuda, path):
    run, agree = PATHS[path]
    out = []
    for i in (0, 1):
        dev = torch.device("cuda", i)
        with torch.cuda.device(dev):
            out.append(run(dev, np.random.default_rng(7)))
            torch.cuda.synchronize()
    agree(*out)
