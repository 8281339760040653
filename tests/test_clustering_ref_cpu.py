"""The float64 restatements of tests/clustering_ref.py against independent definitions (no GPU needed): the DEC gradient
against autograd of oracle/port.py's target and loss, one Lloyd step against scikit-learn, and the regulariser weights' closed
forms against the dense N × N np.matrix definition."""
import numpy as np
import pytest
import torch

import clustering_ref as ref


@pytest.mark.parametrize("K,h,alpha", [(1, 3, 0.2), (2, 1, 1.0), (7, 5, 0.2), (40, 9, 1.0)])
def test_dec_gradient_equals_autograd_of_port(K, h, alpha):
    """Chunked d²-autograd + the closed-form assembly of dz / dμ equals float64 autograd of the whole loss with respect to z and
    μ, written with port.spagcn_target / port.spagcn_kl; the closed form of ∂L/∂d² equals its autograd."""
    from oracle import port
    rng = np.random.default_rng(K * 100 + h)
    n = 57
    z32 = rng.normal(size=(n, h)).astype(np.float32)
    mu32 = rng.normal(size=(K, h)).astype(np.float32)
    z = torch.tensor(z32, dtype=torch.float64, requires_grad=True)
    mu = torch.tensor(mu32, dtype=torch.float64, requires_grad=True)
    d2 = ((z[:, None, :] - mu[None])**2).sum(2)
    q = (1.0 / ((1.0 + d2 / alpha) + 1e-8))**(alpha + 1.0) / 2.0
    q = q / q.sum(1, keepdim=True)
    p = port.spagcn_target(q).detach()
    p32 = p.float().double()       # the kernels read p in float32, and so does the restatement
    loss = port.spagcn_kl(p32, q)
    loss.backward()
    out = ref.dec_reference(torch.from_numpy(z32), torch.from_numpy(mu32), p.float(), alpha, max_elems=7 * K * h)  # 9 chunks
    assert abs(out["loss"] - loss.item()) <= 1e-13 * max(1.0, abs(loss.item()))
    assert torch.allclose(out["q"], q.detach(), rtol=1e-13, atol=0)
    assert torch.allclose(ref.dec_target(q.detach()), p, rtol=1e-13, atol=0)
    assert bool(((out["dz"] - z.grad).abs() <= 1e-10 * out["scale_dz"]).all())
    assert bool(((out["dmu"] - mu.grad).abs() <= 1e-10 * out["scale_dmu"]).all())
    d2l = d2.detach().requires_grad_()
    ql = (1.0 / ((1.0 + d2l / alpha) + 1e-8))**(alpha + 1.0) / 2.0
    c_auto, = torch.autograd.grad(port.spagcn_kl(p32, ql / ql.sum(1, keepdim=True)), d2l)
    c, c_abs = ref.dec_dl_dd2(d2.detach(), p32, alpha, n)
    assert bool(((c - c_auto).abs() <= 1e-12 * c_abs).all())
    assert bool((c_abs >= c.abs() * (1 - 1e-12)).all()) and bool((2 * out["scale_dz"] * (1 + 1e-12) >= out["dz"].abs()).all())


def test_lloyd_step_equals_sklearn_one_iteration():
    from sklearn.cluster import KMeans
    rng = np.random.default_rng(3)
    k, d = 6, 4
    centres = rng.normal(scale=10.0, size=(k, d))
    X = (centres[rng.integers(0, k, 3000)] + rng.normal(size=(3000, d))).astype(np.float32)
    C0 = (centres + rng.normal(scale=0.5, size=(k, d))).astype(np.float32)
    km = KMeans(n_clusters=k, init=C0, n_init=1, max_iter=1, algorithm="lloyd").fit(X)
    Xt, Ct = torch.from_numpy(X), torch.from_numpy(C0)
    D = ref.sq_dist(Xt, Ct)
    best, second, lab = ref.nearest_two(D)
    new, counts = ref.lloyd_update(Xt, Ct, lab)
    assert int(counts.sum()) == 3000 and int((counts > 0).sum()) == k
    assert np.allclose(new.numpy(), km.cluster_centers_, rtol=1e-5, atol=1e-5)
    inertia, shift2, changed = ref.lloyd_stats(D, lab, torch.full((3000, ), -1), Ct, new)
    assert changed == 3000 and shift2 > 0
    assert abs(inertia - float(((X.astype(np.float64) - C0.astype(np.float64)[lab.numpy()])**2).sum())) < 1e-9 * inertia
    # ties go to the lowest index; an empty cluster keeps its centre
    Cd = torch.tensor([[0.0, 0.0], [2.0, 0.0], [0.0, 0.0], [50.0, 50.0]])
    Xd = torch.tensor([[1.0, 0.0], [0.0, 0.0], [2.0, 1.0]])
    _, _, lab = ref.nearest_two(ref.sq_dist(Xd, Cd))
    assert lab.tolist() == [0, 0, 1]
    new, counts = ref.lloyd_update(Xd, Cd, lab)
    assert counts.tolist() == [2, 1, 0, 0] and torch.equal(new[2:], Cd[2:].double())


def _dense_cluster_colsums(A, labels, n_clusters):
    """The reference's np.matrix route: normalize_cell_cell_matrix's row factor 1/rowsum (masked where the sum is 0, then 0),
    tiled into an N × N np.matrix and multiplied — a MATRIX product — with the adjacency; then each cell's column sum inside its
    own cluster, and 0 for a label outside [0, n_clusters)."""
    x = np.matrix(A)
    avg_factor = np.ma.filled(1 / np.ma.masked_equal(np.asarray(x.sum(axis=1)), 0), fill_value=0)
    adjdense = np.asarray(np.matrix(np.tile(avg_factor, [1, len(x)])) * x)
    w = np.zeros(len(labels))
    for j, c in enumerate(labels):
        if 0 <= c < n_clusters:
            w[j] = adjdense[labels == c, j].sum()
    return w


def _graph(n, rng, weighted):
    import scipy.sparse as sp
    deg = rng.integers(0, 6, n)
    deg[:7] = 0                                               # isolated cells
    rows = np.repeat(np.arange(n), deg)
    cols = rng.integers(0, n, len(rows))
    vals = rng.uniform(0.1, 2.0, len(rows)) if weighted else np.ones(len(rows))
    A = sp.coo_matrix((vals, (rows, cols)), shape=(n, n)).tocsr()
    A.sum_duplicates()
    if not weighted:
        A = ((A + A.T) > 0).astype(np.float64).tocsr()
    keep = np.ones(n)
    keep[:8] = 0.0                                             # cells 0..7 have no edge (undirected: none in or out)
    A = (sp.diags(keep) @ A @ (sp.diags(keep) if not weighted else sp.eye(n))).tocsr()
    A.setdiag(0)
    A.eliminate_zeros()
    loop = (rng.random(n) < 0.3).astype(np.float64) * 3.0     # self-loops in some rows only: the weights skip them
    loop[7] = 3.0                                              # a row holding nothing but its self-loop has degree 0 as well
    Aw = (A + sp.diags(loop)).tocsr()
    if weighted:                                               # stored zeros: a row whose entries sum to 0
        c = Aw.tocoo()
        keep6 = c.row != 6
        Aw = sp.csr_matrix((np.r_[c.data[keep6], 0.0, 0.0], (np.r_[c.row[keep6], 6, 6], np.r_[c.col[keep6], 9, 10])), shape=(n, n))
        assert Aw.indptr[7] - Aw.indptr[6] == 2 and not Aw[6].data.any()
    Aw.sort_indices()
    return A, Aw


@pytest.mark.filterwarnings("ignore::PendingDeprecationWarning")     # np.matrix is the definition under test
@pytest.mark.parametrize("weighted", [False, True])
def test_regulariser_weights_equal_dense_definition(weighted):
    rng = np.random.default_rng(11 + weighted)
    n, n_clusters = 300, 5
    A, Aw = _graph(n, rng, weighted)
    labels = rng.integers(-1, n_clusters + 1, n)             # includes −1 and n_clusters: outside every cluster
    labels[:3] = [-1, n_clusters, 0]
    A_off = Aw.toarray()
    np.fill_diagonal(A_off, 0.0)
    dense = _dense_cluster_colsums(A_off, labels, n_clusters)
    if weighted:
        w = ref.regu_weights_weighted(Aw.indptr, Aw.indices, Aw.data, labels, n_clusters)
    else:
        w = ref.regu_weights(Aw.indptr, Aw.indices, labels, n_clusters)
        deg = A_off.sum(1)
        assert (deg == 0).sum() >= 7 and np.array_equal(A_off, A_off.T)
    assert np.allclose(w, dense, rtol=1e-12, atol=0)
    assert w[0] == 0 and w[1] == 0 and (w[labels < 0] == 0).all() and (w[labels >= n_clusters] == 0).all()


def test_celltype_and_l1_restatements_equal_autograd():
    rng = np.random.default_rng(4)
    rows, cols, co = 20, 12, 9
    r = torch.tensor(rng.normal(size=(rows, cols)))
    r[0, :4] = 0.0
    x = torch.tensor(rng.normal(size=(rows, cols)))
    xd = torch.tensor(rng.normal(size=(rows, co)) * (rng.random((rows, co)) < 0.5))
    w = torch.tensor(rng.uniform(0.1, 1.0, rows))
    rr = r.clone().requires_grad_()
    lt = (w[:, None] * (rr - x)**2).sum() + torch.sqrt((((xd - rr[:, :co]) * (xd != 0))**2).sum())
    lt.backward()
    loss, grad, grad_abs = ref.celltype_loss_grad(r, x, xd, w, relu_mask=False)
    assert abs(loss - lt.item()) < 1e-12 * lt.item()
    assert torch.allclose(grad, rr.grad, rtol=1e-12, atol=1e-15) and bool((grad_abs >= grad.abs()).all())
    _, gm, _ = ref.celltype_loss_grad(r, x, xd, w, relu_mask=True)
    assert torch.equal(gm, torch.where(r > 0, grad, 0.0))
    _, g0, _ = ref.celltype_loss_grad(r, x, torch.zeros_like(xd), w, relu_mask=False)
    assert torch.isfinite(g0).all() and torch.allclose(g0, 2 * w[:, None] * (r - x))
    p = torch.tensor([1.5, -2.0, 0.0, -0.0, 3e-39], dtype=torch.float32)
    g, l1 = ref.l1_grad_add(p, torch.ones(5), 0.5)
    assert g.tolist() == [1.5, 0.5, 1.0, 1.0, 1.5] and abs(l1 - 1.75) < 1e-12
