"""Parity of every CUDA kernel (called through the C-ABI) against the oracle / golden fixtures."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from conftest import rel_err
from oracle.scgnn_step_ref import gae_reference_rows

pytestmark = pytest.mark.gpu


def _rand_csr(n_rows, n_cols, density, seed, empty_rows=True):
    rng = np.random.default_rng(seed)
    m = sp.random(n_rows, n_cols, density=density, random_state=rng, format="csr", dtype=np.float32)
    m.data = rng.normal(size=m.data.shape).astype(np.float32)
    if empty_rows and n_rows > 4:
        m = m.tolil()
        m[1, :] = 0
        m[n_rows - 1, :] = 0
        m = m.tocsr()
        m.eliminate_zeros()
    m.sort_indices()
    return m


@pytest.mark.parametrize("F", [4, 8, 16, 32, 48, 64, 128, 200, 400, 512])
@pytest.mark.parametrize("reduce", ["sum", "mean"])
def test_spmm_matches_cpu_csr(cuda, F, reduce):
    from dance_b200 import ops
    m = _rand_csr(257, 301, 0.05, seed=F)
    X = np.random.default_rng(1).normal(size=(301, F)).astype(np.float32)
    ref = (m.astype(np.float64) @ X.astype(np.float64))
    if reduce == "mean":
        deg = np.diff(m.indptr)
        ref = ref / np.maximum(deg, 1)[:, None]
    A = ops.CSR.from_scipy(m, cuda)
    Y = ops.spmm(A, torch.from_numpy(X).to(cuda), reduce=reduce).cpu().numpy()
    assert rel_err(Y, ref) < 1e-6
    assert np.all(Y[1] == 0) and np.all(Y[-1] == 0)  # empty rows


def test_spmm_unweighted_relu_and_padded_ld(cuda):
    from dance_b200 import ops
    m = _rand_csr(500, 500, 0.03, seed=5, empty_rows=False)
    X = torch.randn(500, 64, device=cuda)
    Xv = X[:, :32]  # leading dimension 64, F = 32
    A = ops.CSR.from_scipy(m, cuda, with_values=False)
    ones = m.copy()
    ones.data[:] = 1
    ref = np.maximum(ones.astype(np.float64) @ Xv.cpu().numpy().astype(np.float64), 0)
    Y = ops.spmm(A, Xv, act="relu").cpu().numpy()
    assert rel_err(Y, ref) < 1e-6


def test_spmm_skewed_degrees(cuda):
    """A few very long rows among short ones (gene-side rows of the cell×gene graph)."""
    from dance_b200 import ops
    rng = np.random.default_rng(0)
    n, c = 2000, 3000
    rows = np.concatenate([np.zeros(2500, int), np.full(2900, 7), rng.integers(0, n, 20000)])
    cols = np.concatenate([rng.choice(c, 2500, replace=False), rng.choice(c, 2900, replace=False), rng.integers(0, c, 20000)])
    m = sp.csr_matrix((rng.normal(size=rows.size).astype(np.float32), (rows, cols)), shape=(n, c))
    m.sum_duplicates()
    m.sort_indices()
    X = rng.normal(size=(c, 32)).astype(np.float32)
    Y = ops.spmm(ops.CSR.from_scipy(m, cuda), torch.from_numpy(X).to(cuda)).cpu().numpy()
    assert rel_err(Y, m.astype(np.float64) @ X.astype(np.float64)) < 1e-6


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("F", [8, 16, 32, 64, 104, 256])
@pytest.mark.parametrize("reduce", ["sum", "mean"])
def test_spmm_16bit_operand(cuda, dtype, F, reduce):
    """bf16 / fp16 operand, fp32 accumulation: exact (to summation order) against the fp64 product with the ROUNDED operand, and
    within the storage format's rounding of the fp32 aggregate; conversion kernel == torch's round-to-nearest-even cast."""
    from dance_b200 import ops
    m = _rand_csr(333, 301, 0.08, seed=F)
    X = torch.from_numpy(np.random.default_rng(2).normal(size=(301, F)).astype(np.float32)).to(cuda)
    X16 = ops.to_x16(X, dtype)
    assert torch.equal(X16, X.to(dtype))
    bias = torch.randn(F, device=cuda)
    A = ops.CSR.from_scipy(m, cuda)
    Y = ops.spmm(A, X16, reduce=reduce, act="relu", bias=bias)
    ref = m.astype(np.float64) @ X16.double().cpu().numpy()
    if reduce == "mean":
        ref = ref / np.maximum(np.diff(m.indptr), 1)[:, None]
    ref = np.maximum(ref + bias.double().cpu().numpy(), 0)
    assert Y.dtype == torch.float32 and rel_err(Y, ref) < 1e-6
    # 16-bit output copy (feeds the next layer) and agreement with the fp32-operand kernel at storage precision
    out16 = torch.empty(333, F, dtype=dtype, device=cuda)
    Y2 = ops.spmm(A, X16, reduce=reduce, act="relu", bias=bias, out=torch.empty_like(Y), out16=out16)
    assert torch.equal(Y2, Y) and torch.equal(out16, Y.to(dtype))
    Y32 = ops.spmm(A, X, reduce=reduce, act="relu", bias=bias)
    assert rel_err(Y, Y32) < (4e-3 if dtype == torch.bfloat16 else 5e-4)
    # padded leading dimension + unweighted graph
    wide = torch.zeros(301, F + 24, dtype=dtype, device=cuda)
    wide[:, :F] = X16
    Au = ops.CSR.from_scipy(m, cuda, with_values=False)
    ones = m.copy(); ones.data[:] = 1
    Yu = ops.spmm(Au, wide[:, :F])
    assert rel_err(Yu, ones.astype(np.float64) @ X16.double().cpu().numpy()) < 1e-6
    assert np.all(Yu[1].cpu().numpy() == 0)   # empty row


@pytest.mark.parametrize("F,dtype", [(8, torch.float32), (16, torch.float32), (32, torch.float32), (16, torch.bfloat16), (32, torch.bfloat16),
                                     (64, torch.float16)])
def test_spmm_stream_kernel_against_rowgroup_and_fp64(cuda, F, dtype):
    """The nnz-stream aggregate (operand rows of 32 / 64 / 128 bytes: spmm_stream.cu) on a graph with every row shape it has to
    handle — runs of empty rows longer than its 32-row pointer window, hub rows spanning hundreds of 32-entry blocks, rows ending
    exactly on block boundaries, an empty tail — against fp64 and against the row-per-lane-group kernels (ops.set_path)."""
    from dance_b200 import ops
    rng = np.random.default_rng(F)
    n, c = 20_011, 15_000
    deg = rng.integers(0, 60, n)
    deg[100:180] = 0                      # > 2 pointer windows of empty rows
    deg[500] = 7000; deg[501] = 0; deg[502] = 3333
    deg[1000:1064] = 32                   # rows ending exactly on block boundaries
    deg[-700:] = 0                        # empty tail
    rows = np.repeat(np.arange(n), deg)
    cols = rng.integers(0, c, rows.size)
    m = sp.csr_matrix((rng.normal(size=rows.size).astype(np.float32), (rows, cols)), shape=(n, c))
    m.sum_duplicates(); m.sort_indices()
    X = torch.from_numpy(rng.normal(size=(c, F)).astype(np.float32)).to(cuda)
    Xop = X if dtype == torch.float32 else ops.to_x16(X, dtype)
    bias = torch.randn(F, device=cuda)
    A = ops.CSR.from_scipy(m, cuda)
    ref = m.astype(np.float64) @ Xop.double().cpu().numpy()
    for reduce in ("sum", "mean"):
        r = ref / np.maximum(np.diff(m.indptr), 1)[:, None] if reduce == "mean" else ref
        r = np.maximum(r + bias.double().cpu().numpy(), 0)
        ops.set_path("spmm", "auto")
        Y = ops.spmm(A, Xop, reduce=reduce, act="relu", bias=bias)
        try:
            ops.set_path("spmm", "rowgroup")
            Yg = ops.spmm(A, Xop, reduce=reduce, act="relu", bias=bias)
        finally:
            ops.set_path("spmm", "auto")
        assert rel_err(Y, r) < 1e-6 and rel_err(Yg, r) < 1e-6
        assert rel_err(Y, Yg.cpu().numpy()) < 1e-6
        assert torch.all(Y[100:180] == torch.relu(bias)) and torch.all(Y[-700:] == torch.relu(bias))
    # unit weights, padded leading dimension, one-row and all-empty matrices
    Au = ops.CSR.from_scipy(m, cuda, with_values=False)
    wide = torch.zeros(c, F + 8, dtype=Xop.dtype, device=cuda)
    wide[:, :F] = Xop
    ones = m.copy(); ones.data[:] = 1
    assert rel_err(ops.spmm(Au, wide[:, :F]), ones.astype(np.float64) @ Xop.double().cpu().numpy()) < 1e-6
    one = sp.csr_matrix((np.ones(3, np.float32), ([0, 0, 0], [1, 5, 7])), shape=(1, c))
    assert rel_err(ops.spmm(ops.CSR.from_scipy(one, cuda), Xop), Xop[[1, 5, 7]].double().sum(0, keepdim=True).cpu().numpy()) < 1e-6
    assert torch.all(ops.spmm(ops.CSR.from_scipy(sp.csr_matrix((37, c), dtype=np.float32), cuda), Xop) == 0)


def test_spmm_empty_matrix(cuda):
    from dance_b200 import ops
    m = sp.csr_matrix((10, 10), dtype=np.float32)
    Y = ops.spmm(ops.CSR.from_scipy(m, cuda), torch.ones(10, 8, device=cuda))
    assert torch.all(Y == 0)


def test_csr_transpose_is_exact_and_deterministic(cuda):
    from dance_b200 import ops
    m = _rand_csr(300, 211, 0.04, seed=2)
    A = ops.CSR.from_scipy(m, cuda)
    At, perm = ops.csr_transpose(A)
    mt = m.T.tocsr()
    mt.sort_indices()
    assert np.array_equal(At.rowptr.cpu().numpy(), mt.indptr)
    assert np.array_equal(At.colidx.cpu().numpy(), mt.indices)
    assert np.array_equal(At.vals.cpu().numpy(), mt.data)
    assert np.array_equal(m.data[perm.cpu().numpy()], mt.data)


@pytest.mark.parametrize("transA,transB", [(0, 0), (0, 1), (1, 0), (1, 1)])
@pytest.mark.parametrize("shape", [(130, 70, 50), (257, 129, 33), (64, 512, 128), (1, 5, 3)])
def test_gemm_simt_all_layouts(cuda, transA, transB, shape):
    from dance_b200 import ops
    M, N, K = shape
    rng = np.random.default_rng(M + N + K)
    A = rng.normal(size=(K, M) if transA else (M, K)).astype(np.float32)
    B = rng.normal(size=(N, K) if transB else (K, N)).astype(np.float32)
    bias = rng.normal(size=N).astype(np.float32)
    ref = (A.T if transA else A).astype(np.float64) @ (B.T if transB else B).astype(np.float64) + bias
    C = ops.gemm(torch.from_numpy(A).to(cuda), torch.from_numpy(B).to(cuda), transA=bool(transA), transB=bool(transB),
                 bias=torch.from_numpy(bias).to(cuda), precision="fp32").cpu().numpy()
    assert rel_err(C, ref) < 1e-6


def test_gemm_epilogue_act_mask_accumulate(cuda):
    from dance_b200 import ops
    rng = np.random.default_rng(0)
    A = rng.normal(size=(100, 40)).astype(np.float32)
    B = rng.normal(size=(40, 60)).astype(np.float32)
    mask = rng.normal(size=(100, 60)).astype(np.float32)
    C0 = rng.normal(size=(100, 60)).astype(np.float32)
    ref = np.maximum(A.astype(np.float64) @ B, 0) * (mask > 0) + C0
    out = torch.from_numpy(C0.copy()).to(cuda)
    ops.gemm(torch.from_numpy(A).to(cuda), torch.from_numpy(B).to(cuda), act="relu", mask=torch.from_numpy(mask).to(cuda),
             out=out, accumulate=True, precision="fp32")
    assert rel_err(out.cpu().numpy(), ref) < 1e-6


def test_colsum(cuda):
    from dance_b200 import ops
    X = torch.randn(1237, 77, device=cuda)
    assert rel_err(ops.colsum(X).cpu().numpy(), X.double().sum(0).cpu().numpy()) < 1e-6


def test_mse_loss_grad(cuda):
    from dance_b200 import ops
    rng = np.random.default_rng(3)
    r = np.maximum(rng.normal(size=(50, 30)), 0).astype(np.float32)
    x = rng.normal(size=(50, 30)).astype(np.float32)
    T = rng.random(size=(50, 30)).astype(np.float32)
    for ltmg, s in ((None, 0.0), (None, 0.9), (T, 0.9)):
        w = (1 - s) + (s * T if ltmg is not None else 0)
        ref_loss = (w * (r - x)**2).sum()
        ref_grad = 2 * w * (r - x) * (r > 0)
        loss, grad = ops.mse_sum_loss_grad(torch.from_numpy(r).to(cuda), torch.from_numpy(x).to(cuda),
                                           None if ltmg is None else torch.from_numpy(T).to(cuda), s, relu_mask=True)
        assert abs(loss.item() - ref_loss) < 1e-5 * ref_loss
        assert rel_err(grad.cpu().numpy(), ref_grad) < 1e-6


def test_adam_matches_torch(cuda):
    from dance_b200 import ops
    torch.manual_seed(0)
    p_ref = torch.nn.Parameter(torch.randn(1000, dtype=torch.float32))
    opt = torch.optim.Adam([p_ref], lr=1e-2, weight_decay=0.0)
    p = p_ref.detach().clone().to(cuda)
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    for step in range(1, 6):
        g = torch.randn(1000)
        p_ref.grad = g.clone()
        opt.step()
        ops.adam_step(p, g.to(cuda), m, v, step, lr=1e-2)
        assert torch.allclose(p.cpu(), p_ref.detach(), rtol=1e-6, atol=1e-7)


@pytest.mark.parametrize("n,d,k", [(300, 16, 10), (257, 24, 15), (1000, 128, 15), (130, 3, 6), (90, 50, 40)])
def test_knn_bit_exact_vs_oracle(cuda, n, d, k):
    from dance_b200 import ops
    from oracle import port
    X = port.synthetic_embedding(n, d=d, n_clusters=4, seed=n + d)
    idx_ref, dist_ref = port.knn_indices(X, k, return_dist=True)
    idx, dist = ops.knn(torch.from_numpy(X).to(cuda), k)
    assert np.array_equal(idx.cpu().numpy().astype(np.int64), idx_ref)          # neighbour indices: bit-exact
    assert np.array_equal(dist.cpu().numpy(), dist_ref)                         # fp64 distances: bit-exact


@pytest.mark.parametrize("n,d,k", [(6000, 128, 15), (5000, 50, 15), (4500, 16, 10)])
def test_knn_tensor_core_filter_bit_exact(cuda, n, d, k):
    """n·n_q ≥ 2^24 routes the candidate filter through wgmma (fp16 hi/lo split); the fp64 refine + proof keep the result
    bit-exact with the reference ranking; duplicates, a query range, and the SIMT filter (ops.set_path("knn", "simt")) agree."""
    import os
    from dance_b200 import ops
    from oracle import port
    X = port.synthetic_embedding(n, d=d, n_clusters=5, seed=n + d)
    X[17] = X[4000]                                  # exact duplicate far apart in index
    X[100:110] *= 40.0                               # a few large-norm rows: stresses the error bound / scale
    idx_ref, dist_ref = port.knn_indices(X, k, return_dist=True)
    Xc = torch.from_numpy(X).to(cuda)
    idx, dist = ops.knn(Xc, k)
    assert np.array_equal(idx.cpu().numpy().astype(np.int64), idx_ref)
    assert np.array_equal(dist.cpu().numpy(), dist_ref)
    ops.set_path("knn", "simt")
    try:
        idx_s, _ = ops.knn(Xc, k)
    finally:
        ops.set_path("knn", "auto")
    assert torch.equal(idx, idx_s)
    part, _ = ops.knn(Xc, k, q_begin=300, q_end=n - 200)      # n·n_q still above the threshold: sharded queries on the TC path
    assert torch.equal(part, idx[300:n - 200])


def test_knn_golden_and_graph_build(cuda, golden):
    from dance_b200 import ops
    g = golden("knn_graph")
    X, k = torch.from_numpy(g["X"]).to(cuda), int(g["k"])
    idx, dist = ops.knn(X, k)
    assert np.array_equal(idx.cpu().numpy(), g["knn_idx"])
    assert np.array_equal(1 / (dist.cpu().numpy() + 1e-16), g["knn_w"])
    A = ops.knn_graph_build(idx)
    assert np.array_equal(A.rowptr.cpu().numpy(), g["norm_indptr"])
    assert np.array_equal(A.colidx.cpu().numpy(), g["norm_indices"])
    assert np.array_equal(A.vals.cpu().numpy(), g["norm_data"])                 # D^-1/2 (A+I) D^-1/2 values: bit-exact
    # Σ A (no diagonal) = nnz - n is what pos_weight / norm are computed from (scgnn2.py:567-569)
    n = X.shape[0]
    s = A.nnz - n
    assert float(n * n - s) / s == float(g["pos_weight"])


def test_knn_with_duplicates_and_rank0(cuda):
    """Ties are broken by the smaller index; include_rank0 keeps the self slot."""
    from dance_b200 import ops
    X = np.random.default_rng(0).normal(size=(64, 5)).astype(np.float32)
    X[10] = X[3]
    idx, dist = ops.knn(torch.from_numpy(X).to(cuda), 4, include_rank0=True)
    idx = idx.cpu().numpy()
    assert idx[3, 0] == 3 and idx[3, 1] == 10 and idx[10, 0] == 3 and idx[10, 1] == 10
    assert dist[3, 1].item() == 0.0


def test_knn_query_range(cuda):
    """Row-sharded queries (the multi-GPU decomposition) reproduce the full result."""
    from dance_b200 import ops
    from oracle import port
    X = torch.from_numpy(port.synthetic_embedding(500, d=32, seed=1)).to(cuda)
    full, _ = ops.knn(X, 15)
    a, _ = ops.knn(X, 15, q_begin=0, q_end=200)
    b, _ = ops.knn(X, 15, q_begin=200, q_end=500)
    assert torch.equal(full, torch.cat([a, b]))


def test_pairwise_dense_golden(cuda, golden):
    from dance_b200 import ops
    g = golden("pairwise")
    D = ops.pairwise_l2_dense(torch.from_numpy(g["X"]).to(cuda)).cpu().numpy()
    assert np.array_equal(D, g["D"])   # bit-exact vs the reference's numba kernel


def test_normalize_total_reference_known_answers(cuda, assert_ary_isclose):
    # reference tests/transforms/test_normalize.py:8-43
    from dance_b200 import ops
    x = torch.tensor([[1, 1, 1], [1, 1, 1], [3, 0, 0]], dtype=torch.float32, device=cuda)
    a = ops.normalize_total_log1p_(x.clone(), target_sum=30, max_fraction=0.99, log1p=False)
    assert_ary_isclose(a.cpu().numpy(), np.array([[15.0, 15.0, 15.0], [15.0, 15.0, 15.0], [3.0, 0.0, 0.0]]))
    b = ops.normalize_total_log1p_(a.clone(), target_sum=30, max_fraction=1.0, log1p=False)
    assert_ary_isclose(b.cpu().numpy(), np.array([[10.0, 10.0, 10.0], [10.0, 10.0, 10.0], [30.0, 0.0, 0.0]]))
    c = ops.normalize_total_log1p_(x.clone(), normalize=False, log1p=True)
    assert_ary_isclose(c.cpu().numpy(), np.log1p(x.cpu().numpy()))


@pytest.mark.parametrize("target,maxfrac", [(1e4, 1.0), (None, 1.0), (None, 0.05), (50.0, 0.2)])
def test_normalize_total_log1p_vs_oracle(cuda, target, maxfrac):
    from dance_b200 import ops
    from oracle import port
    X = port.synthetic_expression(333, 203, density=0.2, seed=4, log_normalize=False)
    X[7] = 0  # an all-zero cell stays untouched
    ref = port.log1p(port.normalize_total(X, target_sum=target, exclude_highly_expressed=maxfrac < 1, max_fraction=maxfrac), base=2)
    out = ops.normalize_total_log1p_(torch.from_numpy(X).to(cuda), target_sum=target, max_fraction=maxfrac, base=2)
    assert np.allclose(out.cpu().numpy(), ref, rtol=2e-6, atol=1e-7)
    assert np.all(out[7].cpu().numpy() == 0)


def test_gae_loss_matches_dense_reference_formula(cuda, golden):
    """Matrix-free decoder loss == dense BCE-with-logits on z zᵀ (scgnn2.py:423-426,603-619)."""
    import torch.nn.functional as F
    from dance_b200 import ops
    from oracle import port
    g = golden("knn_graph")
    gg = golden("graph_ae_gcn")
    n = len(g["X"])
    adj = sp.csr_matrix((np.ones(len(g["adj_indices"])), g["adj_indices"], g["adj_indptr"]), shape=(n, n))
    labels_sp = (adj + sp.eye(n)).tocsr()
    labels_sp.sort_indices()
    z = torch.from_numpy(gg["train_z"]).requires_grad_()
    mu = torch.from_numpy(gg["eval_mu"]).requires_grad_()
    lv = torch.from_numpy(gg["eval_logvar"]).requires_grad_()
    pw, norm = float(g["pos_weight"]), float(g["norm"])
    ref = port.gae_loss(z @ z.t(), torch.from_numpy(labels_sp.toarray()).float(), mu, lv, n, norm, pw)
    ref.backward()
    L = ops.CSR.from_scipy(labels_sp, cuda, with_values=False)
    loss, dz, dmu, dlv = ops.gae_loss_grad(z.detach().to(cuda), L, norm, pw, mu.detach().to(cuda), lv.detach().to(cuda))
    assert abs(loss.item() - ref.item()) < 2e-6 * abs(ref.item())
    assert rel_err(dz.cpu().numpy(), z.grad.numpy()) < 1e-5
    assert rel_err(dmu.cpu().numpy(), mu.grad.numpy()) < 1e-5
    assert rel_err(dlv.cpu().numpy(), lv.grad.numpy()) < 1e-5
    # plain BCE (GAT branch, scgnn2.py:618-619)
    z2 = z.detach().clone().requires_grad_()
    ref2 = F.binary_cross_entropy_with_logits(z2 @ z2.t(), torch.from_numpy(labels_sp.toarray()).float())
    ref2.backward()
    loss2, dz2, _, _ = ops.gae_loss_grad(z2.detach().to(cuda), L, 1.0, 1.0, use_pos_weight=False)
    assert abs(loss2.item() - ref2.item()) < 2e-6 * abs(ref2.item())
    assert rel_err(dz2.cpu().numpy(), z2.grad.numpy()) < 1e-5


def _dense_gae_reference(z, L_dense, norm, pw, mu=None, lv=None):
    """fp64 dense restatement of gae_loss_function on the GPU (same formula as oracle.port.gae_loss)."""
    import torch.nn.functional as F
    z = z.double().requires_grad_()
    logits = z @ z.t()
    n = z.shape[0]
    cost = norm * F.binary_cross_entropy_with_logits(logits, L_dense, pos_weight=L_dense * pw)
    cost.backward()
    return cost.item(), z.grad


def test_gae_loss_tensor_core_single_column_range(cuda):
    """The tensor-core decoder at 150 row blocks, more than one wave of SMs.  The call over all rows runs the triangle, which adds
    into dz atomically; the row shards run the full sweep, where a CTA of the long shard sweeps ALL columns and adds without
    atomics.  Checked against the fp64 closed form evaluated in row chunks, full and row-sharded."""
    from dance_b200 import ops
    n, d, k = 19_200, 16, 7
    gen = torch.Generator(device=cuda).manual_seed(11)
    z = (torch.randn(n, d, device=cuda, generator=gen) * 0.45).contiguous()
    idx = torch.randint(0, n, (n, k), device=cuda, dtype=torch.int32, generator=gen)
    A = ops.knn_graph_build(idx.contiguous())
    L = ops.CSR(A.rowptr, A.colidx, None, A.shape)
    norm, pw = 0.5003, 1234.5
    ref_loss, ref_dz = gae_reference_rows(z, A.rowptr, A.colidx, norm, pw, torch.arange(n, device=cuda))
    loss, dz, _, _ = ops.gae_loss_grad(z, L, norm, pw)
    assert abs(loss.item() - ref_loss) < 2e-6 * abs(ref_loss), (loss.item(), ref_loss)
    assert rel_err(dz, ref_dz) < 2e-5
    # one shard with more row blocks than SMs (no J split) + a short one (J sweep split over CTAs)
    h = 148 * 128 + 3
    rp = A.rowptr.long()
    top = ops.CSR(A.rowptr[:h + 1].contiguous(), A.colidx[:rp[h]].contiguous(), None, (h, n))
    bot = ops.CSR((A.rowptr[h:] - A.rowptr[h]).contiguous(), A.colidx[rp[h]:].contiguous(), None, (n - h, n))
    la, dza, _, _ = ops.gae_loss_grad(z, top, norm, pw, row_begin=0, n_rows=h)
    lb, dzb, _, _ = ops.gae_loss_grad(z, bot, norm, pw, row_begin=h, n_rows=n - h)
    assert abs(la.item() + lb.item() - ref_loss) < 2e-6 * abs(ref_loss)
    assert rel_err(torch.cat([dza, dzb]), ref_dz) < 2e-5


@pytest.mark.parametrize("n,d", [(128, 16), (100, 16), (256, 16), (300, 16), (384, 8), (1000, 16), (1537, 16), (1664, 8), (2048, 16), (2049, 16)])
def test_gae_symmetric_decoder_small_graphs(cuda, n, d):
    """The triangle (the call over all rows, forced onto the tensor cores) on small graphs: 1, 2, 3, 8, 13, 16, 17 row blocks, a
    ragged last block and a ragged last 64-column tile, against the fp64 closed form and against the CUDA-core kernel."""
    from dance_b200 import ops
    gen = torch.Generator(device=cuda).manual_seed(n * 31 + d)
    z = (torch.randn(n, d, device=cuda, generator=gen) * 0.6).contiguous()
    idx = torch.randint(0, n, (n, 5), device=cuda, dtype=torch.int32, generator=gen)
    A = ops.knn_graph_build(idx.contiguous())
    L = ops.CSR(A.rowptr, A.colidx, None, A.shape)
    norm, pw = 0.51, 37.0
    ref_loss, ref_dz = gae_reference_rows(z, A.rowptr, A.colidx, norm, pw, torch.arange(n, device=cuda))
    ops.set_path("gae", "tc")
    try:
        loss, dz, _, _ = ops.gae_loss_grad(z, L, norm, pw)
        loss2, dz2, _, _ = ops.gae_loss_grad(z, L, norm, pw)
    finally:
        ops.set_path("gae", "auto")
    assert abs(loss.item() - ref_loss) < 2e-6 * abs(ref_loss), (loss.item(), ref_loss)
    assert rel_err(dz, ref_dz) < 2e-5
    assert rel_err(dz2, dz) < 1e-6 and abs(loss2.item() - loss.item()) < 1e-6 * abs(loss.item())   # atomics reorder sums only
    ops.set_path("gae", "cuda")
    try:
        loss_r, dz_r, _, _ = ops.gae_loss_grad(z, L, norm, pw)
    finally:
        ops.set_path("gae", "auto")
    assert rel_err(dz, dz_r) < 2e-5 and abs(loss.item() - loss_r.item()) < 2e-6 * abs(ref_loss)


@pytest.mark.parametrize("n,splits", [(1537, 2), (2049, 3), (2049, 5), (8200, 2), (8200, 3), (8200, 8)])
def test_gae_symmetric_decoder_step_splits(cuda, n, splits):
    """The triangle's J sweep of each row block (its tiles from the diagonal block on) cut into `splits` step ranges, one CTA each:
    the same loss and gradient as the unsplit sweep and as the fp64 closed form — including parts of one or two tiles, and more
    parts than the last row blocks have tiles."""
    from dance_b200 import ops
    gen = torch.Generator(device=cuda).manual_seed(n + splits)
    z = (torch.randn(n, 16, device=cuda, generator=gen) * 0.5).contiguous()
    idx = torch.randint(0, n, (n, 6), device=cuda, dtype=torch.int32, generator=gen)
    A = ops.knn_graph_build(idx.contiguous())
    L = ops.CSR(A.rowptr, A.colidx, None, A.shape)
    norm, pw = 0.5, 55.0
    rows = torch.arange(n, device=cuda) if n <= 2049 else torch.randint(0, n, (300, ), device=cuda, generator=gen)
    _, ref_rows = gae_reference_rows(z, A.rowptr, A.colidx, norm, pw, rows)
    ops.set_path("gae", "tc")
    try:
        ops.set_tuning("gae_splits", 1)
        loss1, dz1, _, _ = ops.gae_loss_grad(z, L, norm, pw)
        ops.set_tuning("gae_splits", splits)
        loss, dz, _, _ = ops.gae_loss_grad(z, L, norm, pw)
    finally:
        ops.set_tuning("gae_splits", 0)
        ops.set_path("gae", "auto")
    assert rel_err(dz[rows], ref_rows) < 2e-5 and rel_err(dz, dz1) < 2e-6
    assert abs(loss.item() - loss1.item()) < 2e-6 * abs(loss1.item())


@pytest.mark.parametrize("n,path,scale", [(4500, "tc", 3.0e4), (4500, "tc", 40.0), (3000, "cuda", 3.0e4)])
def test_gae_decoder_large_embedding(cuda, n, path, scale):
    """Embeddings far beyond the fp16 operand range (an untrained Graph-AE at 1 M cells draws z = mu + eps·exp(logvar) with logvar ≈ 14,
    |z| ~ 1e6): the tensor-core kernel's tf32 hi/lo operands keep the fp32 exponent range, so its result stays finite and equal to
    the fp64 closed form, like the CUDA-core kernel's (the reference's BCE-with-logits is finite for any logit)."""
    from dance_b200 import ops
    gen = torch.Generator(device=cuda).manual_seed(n)
    z = (torch.randn(n, 16, device=cuda, generator=gen) * scale).contiguous()
    idx = torch.randint(0, n, (n, 5), device=cuda, dtype=torch.int32, generator=gen)
    A = ops.knn_graph_build(idx.contiguous())
    L = ops.CSR(A.rowptr, A.colidx, None, A.shape)
    ref_loss, ref_dz = gae_reference_rows(z, A.rowptr, A.colidx, 0.5, 50.0, torch.arange(n, device=cuda))
    ops.set_path("gae", path)
    try:
        loss, dz, _, _ = ops.gae_loss_grad(z, L, 0.5, 50.0)
    finally:
        ops.set_path("gae", "auto")
    assert bool(torch.isfinite(dz).all()) and np.isfinite(loss.item())
    assert abs(loss.item() - ref_loss) < 5e-6 * abs(ref_loss), (loss.item(), ref_loss)
    assert rel_err(dz, ref_dz) < 5e-5


@pytest.mark.parametrize("n,parts", [(5000, 2), (19_333, 3)])
def test_gae_symmetric_decoder_pair_sharded(cuda, n, parts):
    """b2_gae_loss_grad_sym_f32: contiguous super-block ranges + row ranges of the label terms; the summed partial gradients and
    loss shares equal the single-call result and the fp64 closed form (the multi-GPU decomposition, run on one device)."""
    from dance_b200 import ops
    from dance_b200.parallel import shard_bounds
    d = 16
    gen = torch.Generator(device=cuda).manual_seed(n)
    z = (torch.randn(n, d, device=cuda, generator=gen) * 0.5).contiguous()
    mu = torch.randn(n, d, device=cuda, generator=gen) * 0.3
    lv = torch.randn(n, d, device=cuda, generator=gen) * 0.1
    idx = torch.randint(0, n, (n, 6), device=cuda, dtype=torch.int32, generator=gen)
    A = ops.knn_graph_build(idx.contiguous())
    L = ops.CSR(A.rowptr, A.colidx, None, A.shape)
    norm, pw = 0.5002, 900.0
    full_loss, full_dz, full_dmu, full_dlv = ops.gae_loss_grad(z, L, norm, pw, mu, lv)
    nsb = ops.gae_sym_super_blocks(n)
    rp = A.rowptr.long()
    dz_sum = torch.zeros(n, d, device=cuda)
    loss_sum = 0.0
    dmu_parts, dlv_parts = [], []
    for (s0, s1), (r0, r1) in zip(shard_bounds(nsb, parts), shard_bounds(n, parts)):
        sub = ops.CSR((A.rowptr[r0:r1 + 1] - A.rowptr[r0]).contiguous(), A.colidx[rp[r0]:rp[r1]].contiguous(), None, (r1 - r0, n))
        l, dzf, dmu, dlv = ops.gae_loss_grad_sym(z, sub, norm, pw, s0, s1, mu[r0:r1].contiguous(), lv[r0:r1].contiguous(), row_begin=r0,
                                                 n_rows=r1 - r0)
        dz_sum += dzf
        loss_sum += l.item()
        dmu_parts.append(dmu); dlv_parts.append(dlv)
    assert abs(loss_sum - full_loss.item()) < 2e-6 * abs(full_loss.item())
    assert rel_err(dz_sum, full_dz) < 1e-5
    assert rel_err(torch.cat(dmu_parts), full_dmu) < 1e-6 and rel_err(torch.cat(dlv_parts), full_dlv) < 1e-6
    rows = torch.arange(0, n, 37, device=cuda)
    _, ref_rows = gae_reference_rows(z, A.rowptr, A.colidx, norm, pw, rows)
    assert rel_err(dz_sum[rows], ref_rows) < 2e-5


@pytest.mark.parametrize("with_mu", [False, True])
@pytest.mark.parametrize("form,launches", [("rows-tc", 4), ("rows-cuda", 3), ("sym", 4), ("sym-empty", 3)])
def test_gae_launches_per_call(cuda, form, launches, with_mu):
    """Kernels one decoder call launches: the all-pairs part (tensor cores: the split of z and the sweep; an empty super-block
    range: the split only; CUDA cores: one kernel), the label terms, KLD when mu / logvar are given, and the finish."""
    from dance_b200 import ops
    n, d = 300, 16
    gen = torch.Generator(device=cuda).manual_seed(3)
    z = (torch.randn(n, d, device=cuda, generator=gen) * 0.5).contiguous()
    mu, lv = (torch.randn(n, d, device=cuda, generator=gen), torch.randn(n, d, device=cuda, generator=gen)) if with_mu else (None, None)
    A = ops.knn_graph_build(torch.randint(0, n, (n, 5), device=cuda, dtype=torch.int32, generator=gen))
    L = ops.CSR(A.rowptr, A.colidx, None, A.shape)
    nsb = ops.gae_sym_super_blocks(n)
    ops.set_path("gae", "cuda" if form == "rows-cuda" else "tc")
    try:
        ops.reset_counters()
        if form.startswith("rows"):
            ops.gae_loss_grad(z, L, 0.5, 20.0, mu, lv)
        else:
            sb = (0, nsb) if form == "sym" else (nsb, nsb)
            ops.gae_loss_grad_sym(z, L, 0.5, 20.0, *sb, mu, lv)
        got = ops.counters()["launches"]
    finally:
        ops.set_path("gae", "auto")
    assert got == launches + with_mu


@pytest.mark.parametrize("labels", ["unit", "weighted"])
@pytest.mark.parametrize("path", ["auto", "tc"])
def test_gae_loss_no_rows(cuda, path, labels):
    """The row form with n_rows = 0 (a row shard of no rows, labels [0, n]), with unit labels and with label values (plus the
    transposed labels): nothing to sweep, the loss share is 0 and no row of dz, dmu or dlogvar is written.  Called through the
    C-ABI, which refuses null pointers: torch gives an empty tensor none, so the row buffers point into a guard buffer that must
    stay as it is."""
    from dance_b200 import _lib, ops
    n, d, r = 300, 16, 120
    lib = _lib.lib()
    z = torch.randn(n, d, device=cuda)
    rowptr = torch.zeros(1, dtype=torch.int32, device=cuda)
    colidx = torch.zeros(1, dtype=torch.int32, device=cuda)
    guard = torch.full((4, d), 5.0, device=cuda)
    loss = torch.full((1,), 7.0, device=cuda)
    ws = torch.empty(lib.b2_gae_loss_workspace_bytes(n, d), dtype=torch.uint8, device=cuda)
    g = guard.data_ptr()
    ops.set_path("gae", path)
    try:
        lab = [rowptr.data_ptr(), colidx.data_ptr()]
        lab += [None] * 4 if labels == "unit" else [g, rowptr.data_ptr(), colidx.data_ptr(), g]
        status = lib.b2_gae_loss_grad_f32(z.data_ptr(), d, g, g, d, *lab, n, d, r, 0, 0.5, 20.0, 1, g, g, g, d, loss.data_ptr(),
                                          ws.data_ptr(), ws.numel(), ops._stream())
    finally:
        ops.set_path("gae", "auto")
    assert status == 0
    assert loss.item() == 0.0 and torch.all(guard == 5.0)


@pytest.mark.parametrize("n,d", [(3000, 16), (2500, 16), (4133, 8), (2304, 32)])
def test_gae_loss_tensor_core_path(cuda, n, d):
    """Tensor-core decoder (S in registers → SFU → G in registers → dZ) vs the dense fp64 formula and vs the CUDA-core kernel."""
    import os
    from dance_b200 import ops
    from oracle import port
    rng = np.random.default_rng(n)
    z = torch.from_numpy((rng.normal(size=(n, d)) * 0.4).astype(np.float32)).to(cuda)
    adj, _ = port.feature2adj(port.synthetic_embedding(n, d=8, seed=1), 6)
    Lsp = (adj + sp.eye(n)).tocsr()
    Lsp.sort_indices()
    L = ops.CSR.from_scipy(Lsp, cuda, with_values=False)
    Ld = torch.from_numpy(Lsp.toarray()).to(cuda).double()
    pw, norm = port.gae_norm_constants(adj)
    ref_loss, ref_dz = _dense_gae_reference(z, Ld, norm, pw)
    loss_tc, dz_tc, _, _ = ops.gae_loss_grad(z, L, norm, pw)
    ops.set_path("gae", "cuda")
    try:
        loss_cc, dz_cc, _, _ = ops.gae_loss_grad(z, L, norm, pw)
    finally:
        ops.set_path("gae", "auto")
    assert abs(loss_tc.item() - ref_loss) < 2e-6 * abs(ref_loss), (loss_tc.item(), ref_loss)
    assert abs(loss_cc.item() - ref_loss) < 2e-6 * abs(ref_loss)
    assert rel_err(dz_tc.cpu().numpy(), ref_dz.cpu().numpy()) < 2e-5
    assert rel_err(dz_cc.cpu().numpy(), ref_dz.cpu().numpy()) < 2e-5
    # row-sharded form: two shards reproduce the full gradient and the loss is additive
    h = n // 2 + 7
    la, dza, _, _ = ops.gae_loss_grad(z, ops.CSR.from_scipy(Lsp[:h], cuda, with_values=False), norm, pw, row_begin=0, n_rows=h)
    lb, dzb, _, _ = ops.gae_loss_grad(z, ops.CSR.from_scipy(Lsp[h:], cuda, with_values=False), norm, pw, row_begin=h, n_rows=n - h)
    assert abs(la.item() + lb.item() - ref_loss) < 2e-6 * abs(ref_loss)
    assert rel_err(torch.cat([dza, dzb]).cpu().numpy(), ref_dz.cpu().numpy()) < 2e-5
