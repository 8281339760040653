"""graph_AE_retain_weights on the GPU: the weighted, directed graph builder, the decoder with real-valued asymmetric labels, the
engines and the module, against the reference fixture (tests/make_golden_retain_weights.py), the numpy restatement
(tests/retain_weights_ref.py) and fp64 closed forms."""
import argparse

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from conftest import rel_err
from retain_weights_ref import decoder_loss_grad, weighted_graph

pytestmark = pytest.mark.gpu


def _fixture_csr(g, key):
    n = len(g[key + ".indptr"]) - 1
    return sp.csr_matrix((g[key + ".data"], g[key + ".indices"], g[key + ".indptr"]), shape=(n, n))


def _host(A):
    return sp.csr_matrix((A.vals.cpu().numpy(), A.colidx.cpu().numpy(), A.rowptr.cpu().numpy()), shape=A.shape)


def _same_structure(mine: sp.csr_matrix, ref: sp.csr_matrix):
    ref = ref.tocsr()
    ref.sort_indices()
    return np.array_equal(mine.indptr, ref.indptr) and np.array_equal(mine.indices, ref.indices)


def _within_ulp(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return bool(np.all(np.abs(a.astype(np.float64) - b) <= np.spacing(np.abs(b)).astype(np.float64)))


def _check_graph(wg, ahat_ref, labels_ref, sum_w_ref):
    assert _same_structure(_host(wg.adj), ahat_ref) and _within_ulp(_host(wg.adj).data, ahat_ref.tocsr().data)
    ahat_t = ahat_ref.T.tocsr()
    ahat_t.sort_indices()
    assert _same_structure(_host(wg.adj_t), ahat_t) and _within_ulp(_host(wg.adj_t).data, ahat_t.data)
    lt = labels_ref.T.tocsr()
    lt.sort_indices()
    assert _same_structure(_host(wg.labels), labels_ref) and np.array_equal(_host(wg.labels).data, labels_ref.tocsr().data)
    assert _same_structure(_host(wg.labels_t), lt) and np.array_equal(_host(wg.labels_t).data, lt.data)
    assert abs(wg.sum_w.item() - sum_w_ref) <= 1e-12 * abs(sum_w_ref)


@pytest.mark.parametrize("tag", ["k5", "k15"])
def test_builder_matches_reference_fixture(cuda, golden, tag):
    """Structure bit-exact, Â within 1 fp32 ulp, labels exact, ΣW within 1e-12 (k5 holds a self-listed neighbour and a 1e16)."""
    from dance_b200 import ops
    g = golden("scgnn_retain_weights")
    wg = ops.knn_graph_weighted_build(torch.from_numpy(g[f"{tag}.knn_idx"]).to(cuda), torch.from_numpy(g[f"{tag}.knn_dist"]).to(cuda))
    _check_graph(wg, _fixture_csr(g, f"{tag}.ahat"), _fixture_csr(g, f"{tag}.labels"), float(g[f"{tag}.sum_w"]))


def test_builder_at_200k_cells_matches_restatement(cuda):
    from dance_b200 import ops
    gen = torch.Generator(device=cuda).manual_seed(4)
    n, k = 200_000, 15
    X = torch.randn(n, 32, device=cuda, generator=gen) + 3 * torch.randn(8, 32, device=cuda, generator=gen)[
        torch.randint(0, 8, (n, ), device=cuda, generator=gen)]
    idx, dist = ops.knn(X, k)
    wg = ops.knn_graph_weighted_build(idx, dist)
    _, _, ahat, labels, sum_w = weighted_graph(idx.cpu().numpy(), dist.cpu().numpy())
    _check_graph(wg, ahat, labels, sum_w)


def test_builder_rejects_bad_lists(cuda):
    from dance_b200 import ops
    from dance_b200._lib import B2Error
    idx = torch.tensor([[1, 2], [0, 2], [0, 0]], dtype=torch.int32, device=cuda)
    dist = torch.ones(3, 2, dtype=torch.float64, device=cuda)
    with pytest.raises(B2Error, match="twice"):
        ops.knn_graph_weighted_build(idx, dist)
    with pytest.raises(B2Error, match="outside"):
        ops.knn_graph_weighted_build(torch.tensor([[1], [3], [0]], dtype=torch.int32, device=cuda), dist[:, :1].contiguous())


# ---- decoder ---------------------------------------------------------------------------------------------------------
def _random_labels(n, k, seed, device):
    """A random directed pattern (k out-entries per row) plus the unit diagonal, values in [0.05, 3]: L and Lᵀ as CSRs."""
    from dance_b200 import ops
    rng = np.random.default_rng(seed)
    cols = np.stack([rng.choice(n - 1, k, replace=False) for _ in range(n)])
    cols = cols + (cols >= np.arange(n)[:, None])                   # skip the diagonal
    vals = rng.uniform(0.05, 3.0, (n, k))
    L = sp.csr_matrix((vals.reshape(-1), cols.reshape(-1), np.arange(0, n * k + 1, k)), shape=(n, n)) + sp.eye(n)
    L = L.tocsr().astype(np.float32)
    L.sort_indices()
    Lt = L.T.tocsr()
    Lt.sort_indices()
    return L, ops.CSR.from_scipy(L, device), ops.CSR.from_scipy(Lt, device)


def _rows(A, r0, r1):
    from dance_b200 import ops
    return ops.CSR(A.rowptr[r0:r1 + 1].contiguous(), A.colidx, A.vals, (r1 - r0, A.shape[1]))


CASES = [(1000, d, "cuda") for d in (8, 16, 32, 64)] + [(4096, d, "auto") for d in (8, 16, 32, 64)]


@pytest.mark.parametrize("n,d,path", CASES, ids=[f"n{c[0]}-d{c[1]}-{c[2]}" for c in CASES])
@pytest.mark.parametrize("use_pw", [True, False], ids=["posweight", "plain"])
def test_decoder_matches_fp64_closed_form(cuda, n, d, path, use_pw):
    """Loss ≤ 2e-6 and dz ≤ 2e-5 relative to fp64 autograd, full rows and a partial row range (n = 4096, d ≤ 32: tensor cores)."""
    from dance_b200 import ops
    L_sp, L, Lt = _random_labels(n, 12, seed=n + d, device=cuda)
    gen = torch.Generator(device=cuda).manual_seed(d)
    z = torch.randn(n, d, device=cuda, generator=gen) * (0.6 / d**0.5)
    dense = torch.from_numpy(L_sp.toarray()).to(cuda).double()
    sum_w = float(L_sp.sum()) - n
    pw, norm = float(n * n - sum_w) / sum_w, n * n / float((n * n - sum_w) * 2)
    ref_loss, ref_dz = decoder_loss_grad(z.double(), dense, norm, pw, use_pw)
    ops.set_path("gae", path)
    try:
        loss, dz, _, _ = ops.gae_loss_grad(z, L, norm, pw, use_pos_weight=use_pw, labels_t=Lt)
        assert abs(loss.item() - ref_loss) <= 2e-6 * abs(ref_loss)
        assert rel_err(dz, ref_dz) < 2e-5
        # rows [r0, r1): the loss share and dz of those rows
        r0, r1 = n // 4 + 3, (3 * n) // 4
        zr = z.double().requires_grad_()
        x = zr[r0:r1] @ zr.t()
        y = dense[r0:r1]
        part = torch.nn.functional.binary_cross_entropy_with_logits(x, y, pos_weight=y * pw if use_pw else None, reduction="sum")
        part = part * ((norm if use_pw else 1.0) / (n * n))
        loss_r, dz_r, _, _ = ops.gae_loss_grad(z, _rows(L, r0, r1), norm, pw, use_pos_weight=use_pw, labels_t=_rows(Lt, r0, r1),
                                               row_begin=r0, n_rows=r1 - r0)
        assert abs(loss_r.item() - part.item()) <= 2e-6 * abs(part.item())
        assert rel_err(dz_r, ref_dz[r0:r1]) < 2e-5
    finally:
        ops.set_path("gae", "auto")


@pytest.mark.parametrize("use_pw", [True, False], ids=["posweight", "plain"])
def test_pair_sharded_form_sums_to_row_form(cuda, use_pw):
    from dance_b200 import ops
    from dance_b200.parallel import shard_bounds
    n, d, world = 4096, 16, 3
    _, L, Lt = _random_labels(n, 10, seed=5, device=cuda)
    z = torch.randn(n, d, device=cuda, generator=torch.Generator(device=cuda).manual_seed(1)) * 0.15
    loss, dz, _, _ = ops.gae_loss_grad(z, L, 2.0, 30.0, use_pos_weight=use_pw, labels_t=Lt)
    sbs, rows = shard_bounds(ops.gae_sym_super_blocks(n), world), shard_bounds(n, world)
    total, dz_sum = 0.0, torch.zeros_like(dz)
    for r in range(world):
        (s0, s1), (r0, r1) = sbs[r], rows[r]
        ls, dzf, _, _ = ops.gae_loss_grad_sym(z, _rows(L, r0, r1), 2.0, 30.0, s0, s1, use_pos_weight=use_pw, row_begin=r0,
                                              n_rows=r1 - r0, labels_t=_rows(Lt, r0, r1))
        total += ls.item()
        dz_sum += dzf
    assert abs(total - loss.item()) <= 1e-6 * abs(loss.item())
    assert rel_err(dz_sum, dz) < 1e-6


@pytest.mark.parametrize("use_pw", [True, False], ids=["posweight", "plain"])
@pytest.mark.parametrize("n", [1000, 4096])
def test_unit_symmetric_labels_match_existing_entry(cuda, n, use_pw):
    from dance_b200 import ops
    gen = torch.Generator(device=cuda).manual_seed(n)
    X = torch.randn(n, 16, device=cuda, generator=gen)
    A = ops.knn_graph_build(ops.knn(X, 10)[0])                      # union-symmetrised: L = Lᵀ
    ones = torch.ones(A.nnz, dtype=torch.float32, device=cuda)
    Lw = ops.CSR(A.rowptr, A.colidx, ones, A.shape)
    z = torch.randn(n, 16, device=cuda, generator=gen) * 0.2
    l0, dz0, _, _ = ops.gae_loss_grad(z, ops.CSR(A.rowptr, A.colidx, None, A.shape), 1.7, 40.0, use_pos_weight=use_pw)
    l1, dz1, _, _ = ops.gae_loss_grad(z, Lw, 1.7, 40.0, use_pos_weight=use_pw, labels_t=Lw)
    assert abs(l1.item() - l0.item()) <= 1e-6 * abs(l0.item()) and rel_err(dz1, dz0) < 1e-6


def test_decoder_refuses_values_without_transpose(cuda):
    from dance_b200 import ops
    from dance_b200._lib import B2Error
    _, L, Lt = _random_labels(64, 4, seed=0, device=cuda)
    z = torch.zeros(64, 8, device=cuda)
    with pytest.raises(B2Error, match="labels_t"):
        ops.gae_loss_grad(z, L, 1.0, 1.0)
    with pytest.raises(B2Error, match="labels_t"):
        ops.gae_loss_grad(z, L, 1.0, 1.0, labels_t=_rows(Lt, 0, 32))


# ---- engines, regulariser, module ------------------------------------------------------------------------------------
def _fixture_graph(g, cuda):
    from dance_b200 import ops
    return ops.knn_graph_weighted_build(torch.from_numpy(g["k15.knn_idx"]).to(cuda), torch.from_numpy(g["k15.knn_dist"]).to(cuda))


def test_graph_ae_engine_step_matches_reference(cuda, golden):
    from dance_b200.engine import GraphAEEngine
    g = golden("scgnn_retain_weights")
    wg = _fixture_graph(g, cuda)
    x = torch.from_numpy(g["k15.X"]).to(cuda)
    eng = GraphAEEngine(x.shape[1], 16, device=cuda, lr=1e-2, precision="tf32x3")
    eng.load_state_dict({f"gc{i}.weight": g[f"k15.gcn.w{i}"] for i in (1, 2, 3)})
    z, _, _ = eng.train_step(x, wg.adj, wg.labels, float(g["k15.norm"]), float(g["k15.pos_weight"]), torch.from_numpy(g["k15.gcn.eps"]).to(cuda),
                             adj_t=wg.adj_t, labels_t=wg.labels_t)
    assert rel_err(z, g["k15.gcn.z"]) < 1e-4
    assert abs(eng.loss.item() - float(g["k15.gcn.loss"])) < 1e-4 * abs(float(g["k15.gcn.loss"]))
    for i in (1, 2, 3):
        assert rel_err(eng.grads()[f"gc{i}.weight"], g[f"k15.gcn.g_w{i}"]) < 1e-4, i
        assert rel_err(eng.state_dict()[f"gc{i}.weight"], g[f"k15.gcn.w{i}_after"]) < 1e-4, i


def test_gat_engine_step_matches_reference(cuda, golden):
    from dance_b200 import ops
    from dance_b200.engine import GATEngine
    g = golden("scgnn_retain_weights")
    wg = _fixture_graph(g, cuda)
    idx = torch.from_numpy(g["k15.knn_idx"]).to(cuda)
    n, k = idx.shape
    T, _ = ops.csr_transpose(ops.CSR(torch.arange(0, n * k + 1, k, dtype=torch.int32, device=cuda), idx.reshape(-1).contiguous(), None, (n, n)))
    Tt, t_perm = ops.csr_transpose(T)
    x = torch.from_numpy(g["k15.X"]).to(cuda)
    eng = GATEngine(x.shape[1], 64, 16, 2, device=cuda, lr=1e-2, precision="tf32x3")
    pre = "k15.gat.init."
    eng.load_state_dict({key[len(pre):]: g[key] for key in g.files if key.startswith(pre)})
    z = eng.train_step(x, T, Tt, t_perm, wg.labels, wg.labels_t)
    assert rel_err(z, g["k15.gat.z"]) < 1e-4
    assert abs(eng.loss.item() - float(g["k15.gat.loss"])) < 1e-4 * abs(float(g["k15.gat.loss"]))
    for key, gt in eng.grads().items():
        want = g["k15.gat.grad." + key]
        assert rel_err(gt.cpu().numpy().reshape(want.shape), want) < 1e-4, key
    # Adam's first step moves each weight by lr·g/(|g| + eps): where the reference gradient is orders of magnitude below the
    # tensor's largest entry (layer 0's scoring_fn_target has entries below 1e-7), the step's size and sign are set by rounding.
    # Those weights are held to one step; every other weight to 1e-4.
    for key, v in eng.state_dict().items():
        want, gref = g["k15.gat.after." + key], np.abs(g["k15.gat.grad." + key])
        got = v.cpu().numpy().reshape(want.shape)
        firm = gref >= 1e-3 * gref.max()
        assert rel_err(got[firm], want[firm]) < 1e-4, key
        assert np.all(np.abs(got - want) <= 2 * 1e-2 + 1e-6), key


def test_regulariser_weights_match_reference(cuda, golden):
    from dance_b200 import ops
    from dance_b200.modules.scgnn2 import graph_celltype_regu_handler
    g = golden("scgnn_retain_weights")
    W, lab, ref = _fixture_csr(g, "k15.W"), g["k15.regu.labels"], g["k15.regu.w"]
    w, ones = graph_celltype_regu_handler(W, lab, cuda)
    assert torch.equal(ones, torch.ones_like(ones))
    assert np.all(np.abs(w.cpu().numpy() - ref) <= 1e-6 * np.abs(ref))
    dev = torch.sparse_csr_tensor(torch.from_numpy(W.indptr).long(), torch.from_numpy(W.indices).long(), torch.from_numpy(W.data), W.shape).to(cuda)
    w_dev, _ = graph_celltype_regu_handler(dev, lab, cuda)
    assert np.all(np.abs(w_dev.cpu().numpy() - ref) <= 1e-6 * np.abs(ref))
    # 0/1 adjacencies keep the degree path, bit for bit
    A01 = sp.csr_matrix((np.ones(W.nnz, np.float32), W.indices, W.indptr), shape=W.shape)
    w01, _ = graph_celltype_regu_handler(A01, lab, cuda)
    want = ops.graph_regu_weights(ops.CSR.from_scipy(A01, cuda, with_values=False), torch.from_numpy(lab).to(cuda))
    assert torch.equal(w01, want)


def _args(**over):
    d = dict(total_epoch=0, feature_AE_epoch=[2, 1], feature_AE_batch_size=128, feature_AE_learning_rate=1e-3, feature_AE_regu_strength=0.9,
             feature_AE_dropout_prob=0, feature_AE_concat_prev_embed=None, graph_AE_epoch=2, graph_AE_use_GAT=False, graph_AE_GAT_dropout=0,
             graph_AE_learning_rate=1e-2, graph_AE_embedding_size=16, graph_AE_concat_prev_embed=False, graph_AE_normalize_embed=None,
             graph_AE_neighborhood_factor=10, graph_AE_retain_weights=True, gat_multi_heads=2, gat_hid_embed=64)
    d.update(over)
    return argparse.Namespace(**d)


@pytest.mark.parametrize("use_gat", [False, True], ids=["gcn", "gat"])
def test_graph_ae_handler_with_retained_weights(cuda, use_gat):
    from dance_b200.modules.scgnn2 import graph_AE_handler
    from oracle import port
    X = np.abs(port.synthetic_embedding(500, d=64, n_clusters=4, seed=9)) * 0.05
    param = {"device": cuda, "epoch_num": 0, "seed": 1}
    embed, recon, (edge_index, edge_w), adj = graph_AE_handler(X, None, _args(graph_AE_use_GAT=use_gat), param)
    assert embed.shape == (500, 16) and np.isfinite(embed).all() and rel_err(recon, embed @ embed.T) < 1e-5
    W = sp.csr_matrix((edge_w, (edge_index[:, 0], edge_index[:, 1])), shape=(500, 500))
    assert adj.dtype == np.float64 and (adj != W).nnz == 0 and (adj != adj.T).nnz > 0       # W itself: directed, weighted


def test_graph_ae_handler_locality_order_with_retained_weights(cuda):
    from dance_b200.modules.scgnn2 import graph_AE_handler
    from oracle import port
    emb = np.abs(port.synthetic_embedding(3000, d=128, n_clusters=6, seed=3)) * 0.05
    outs = []
    for order in (None, "locality"):
        param = {"device": cuda, "epoch_num": 0, "seed": 0, "precision": "fp32", "cell_order": order, "cell_order_anchors": 16}
        outs.append(graph_AE_handler(emb, None, _args(), param))
    (z0, _, e0, a0), (z1, _, e1, a1) = outs
    assert np.isfinite(z0).all() and np.linalg.norm(z0 - z1) / np.linalg.norm(z0) < 1e-5
    assert np.array_equal(e0[0], e1[0]) and (a0 != a1).nnz == 0


def test_graph_cache_is_keyed_by_the_flag(cuda):
    from dance_b200.modules.scgnn2 import graph_AE_handler
    from oracle import port
    X = port.synthetic_embedding(300, d=32, n_clusters=3, seed=2)
    cache = {}
    _, _, _, a_w = graph_AE_handler(X, None, _args(graph_AE_epoch=1), {"device": cuda, "epoch_num": 0, "seed": 0, "graph_cache": cache})
    _, _, _, a_u = graph_AE_handler(X, None, _args(graph_AE_epoch=1, graph_AE_retain_weights=False),
                                    {"device": cuda, "epoch_num": 0, "seed": 0, "graph_cache": cache})
    assert a_w.dtype == np.float64 and np.all(a_u.data == 1) and (a_u != a_u.T).nnz == 0


def test_scgnn2_fit_with_retained_weights(cuda):
    from dance_b200.modules.scgnn2 import ScGNN2
    from oracle import port
    X = port.synthetic_expression(256, 48, density=0.3, seed=1)
    em = ScGNN2(_args(total_epoch=1, clustering_louvain_only=False, clustering_embed="graph", clustering_method="KMeans", seed=0,
                      cluster_AE_batch_size=12800, cluster_AE_epoch=2, cluster_AE_learning_rate=1e-3, cluster_AE_regu_strength=0.9,
                      cluster_AE_dropout_prob=0), device="cuda", seed=0)
    em.fit(X)
    assert em.predict().shape == X.shape and np.isfinite(em.predict()).all() and len(em.cluster_labels) == 256


# ---- 1 M cells ---------------------------------------------------------------------------------------------------------
def test_one_million_cells_build_and_step(cuda):
    """k = 15, d = 16: build the weighted graph, take one Graph-AE step, and check sampled decoder gradient rows against the fp64
    closed form over all 1 M columns."""
    from dance_b200 import ops
    from dance_b200.engine import GraphAEEngine
    n, k, e = 1_000_000, 15, 16
    gen = torch.Generator(device=cuda).manual_seed(0)
    centres = torch.randn(10, 16, device=cuda, generator=gen) * 3
    X = torch.randn(n, 16, device=cuda, generator=gen) + centres[torch.randint(0, 10, (n, ), device=cuda, generator=gen)]
    idx, dist = ops.knn(X, k)
    wg = ops.knn_graph_weighted_build(idx, dist)
    assert wg.labels.nnz == n * (k + 1) and torch.equal(wg.adj.rowptr[-1:], wg.adj_t.rowptr[-1:])
    sum_w = wg.sum_w.item()
    pw, norm = float(n * n - sum_w) / sum_w, n * n / float((n * n - sum_w) * 2)
    # Â is normalised by out-weights only, so a hub's row sums its many in-edges: a small input keeps logvar (and exp(logvar))
    # in range
    xin = (X.abs() * 1e-3).contiguous()
    eng = GraphAEEngine(16, e, device=cuda, seed=0)
    eps = torch.randn(n, e, device=cuda, generator=gen)
    z, _, _ = eng.train_step(xin, wg.adj, wg.labels, norm, pw, eps, adj_t=wg.adj_t, labels_t=wg.labels_t)
    assert np.isfinite(eng.loss.item())
    # the decoder alone on this z, then the closed form on sampled rows
    _, dz, _, _ = ops.gae_loss_grad(z, wg.labels, norm, pw, labels_t=wg.labels_t)
    rows = torch.tensor([0, 1, 4242, 500_000, 777_777, n - 1], device=cuda)
    zd = z.double()
    coef = norm / (float(n) * n)
    for r in rows.tolist():
        x = zd @ zd[r]
        g = 2 * torch.sigmoid(x)
        for A in (wg.labels, wg.labels_t):                              # row r of L (y_rj) and of Lᵀ (y_jr)
            s, t = A.rowptr[r].item(), A.rowptr[r + 1].item()
            j, y = A.colidx[s:t].long(), A.vals[s:t].double()
            g[j] += -y * y * pw * torch.sigmoid(-x[j]) - y * torch.sigmoid(x[j])
        want = coef * (g @ zd)
        assert rel_err(dz[r], want) < 1e-4, r
