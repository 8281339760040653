"""Pin the oracle (oracle/port.py): against the reference's own known-answer tests and against the
committed fixtures generated from the reference's code (tests/golden, oracle/make_golden.py)."""
import itertools

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.spatial
import torch

from oracle import port

from conftest import rel_err


# ---- the reference's own golden vectors ------------------------------------------------------
def test_matrix_normalize_known_answers():
    # reference tests/utils/test_matrix.py:9-29
    mat = np.array([[1, 1], [4, 4]])
    assert port.matrix_normalize(mat, mode="normalize", axis=0).tolist() == [[0.2, 0.2], [0.8, 0.8]]
    assert port.matrix_normalize(mat, mode="normalize", axis=1).tolist() == [[0.5, 0.5], [0.5, 0.5]]
    assert port.matrix_normalize(mat, mode="standardize", axis=0).tolist() == [[-1, -1], [1, 1]]
    assert port.matrix_normalize(mat, mode="standardize", axis=1).tolist() == [[0, 0], [0, 0]]
    assert port.matrix_normalize(mat, mode="minmax", axis=0).tolist() == [[0, 0], [1, 1]]
    assert port.matrix_normalize(mat, mode="minmax", axis=1).tolist() == [[0, 0], [0, 0]]
    assert port.matrix_normalize(mat, mode="l2", axis=0).tolist() == (mat / np.sqrt((mat**2).sum(0))).tolist()
    assert port.matrix_normalize(mat, mode="l2", axis=1).tolist() == (mat / np.sqrt((mat**2).sum(1, keepdims=True))).tolist()


REF_DIST_MAT = np.array([[0, 1, 2], [2, 2, 4], [5, 3, 5], [3, 2, 1], [5, 6, 3]], dtype=np.float32)


def test_pairwise_euclidean_known_answers():
    # reference tests/utils/test_matrix.py:32-52
    n = REF_DIST_MAT.shape[0]
    ans = np.zeros((n, n), dtype=np.float32)
    for i, j in itertools.product(range(n), range(n)):
        ans[i, j] = scipy.spatial.distance.euclidean(REF_DIST_MAT[i], REF_DIST_MAT[j])
    assert np.allclose(ans, port.pairwise_euclidean(REF_DIST_MAT))


def test_normalize_total_known_answers(assert_ary_isclose):
    # reference tests/transforms/test_normalize.py:8-30 (NormalizeTotal → exclude_highly_expressed=True)
    x = np.array([[1, 1, 1], [1, 1, 1], [3, 0, 0]], dtype=np.float32)
    out = port.normalize_total(x, target_sum=30, exclude_highly_expressed=True, max_fraction=0.99)
    assert_ary_isclose(out, np.array([[15.0, 15.0, 15.0], [15.0, 15.0, 15.0], [3.0, 0.0, 0.0]]))
    out = port.normalize_total(out, target_sum=30, exclude_highly_expressed=True, max_fraction=1.0)
    assert_ary_isclose(out, np.array([[10.0, 10.0, 10.0], [10.0, 10.0, 10.0], [30.0, 0.0, 0.0]]))


def test_log1p_known_answers(assert_ary_isclose):
    # reference tests/transforms/test_normalize.py:33-43
    x = np.array([[1, 1, 1], [1, 1, 1], [3, 0, 0]])
    assert_ary_isclose(port.log1p(x), np.log1p(x))


# ---- committed fixtures generated from the reference --------------------------------------------
def test_pairwise_golden(golden):
    g = golden("pairwise")
    assert np.array_equal(port.pairwise_euclidean(g["X"]), g["D"])  # bit-exact vs the numba kernel


def test_knn_graph_golden(golden):
    g = golden("knn_graph")
    X, k = g["X"], int(g["k"])
    idx, dist = port.knn_indices(X, k, return_dist=True)
    assert np.array_equal(idx, g["knn_idx"])                      # neighbour indices: bit-exact
    assert np.array_equal(1 / (dist + 1e-16), g["knn_w"])         # fp64 weights 1/(d+1e-16): bit-exact
    adj, _ = port.feature2adj(X, k)
    assert np.array_equal(adj.indptr, g["adj_indptr"]) and np.array_equal(adj.indices, g["adj_indices"])
    an = port.preprocess_graph(adj)
    assert np.array_equal(an.indptr, g["norm_indptr"]) and np.array_equal(an.indices, g["norm_indices"])
    assert np.array_equal(an.data, g["norm_data"])
    pw, norm = port.gae_norm_constants(adj)
    assert pw == float(g["pos_weight"]) and norm == float(g["norm"])


def _graph_inputs(golden):
    g = golden("knn_graph")
    adj = sp.csr_matrix((np.ones(len(g["adj_indices"])), g["adj_indices"], g["adj_indptr"]), shape=(len(g["X"]),) * 2)
    an = sp.csr_matrix((g["norm_data"], g["norm_indices"], g["norm_indptr"]), shape=adj.shape)
    return g["X"], adj, an


def test_graph_ae_golden(golden):
    X, adj, an = _graph_inputs(golden)
    g = golden("graph_ae_gcn")
    x = torch.from_numpy(X)
    w = [torch.from_numpy(g[k]).requires_grad_() for k in ("w1", "w2", "w3")]
    loss, z, mu, logvar, hidden1 = port.graph_ae_gcn_loss(x, *w, an, adj, eps=torch.from_numpy(g["eps"]))
    loss.backward()
    assert rel_err(hidden1.detach().numpy(), g["hidden1"]) < 1e-6
    assert rel_err(z.detach().numpy(), g["train_z"]) < 1e-6
    assert abs(loss.item() - float(g["loss"])) < 1e-6 * abs(float(g["loss"]))
    for wi, key in zip(w, ("g_w1", "g_w2", "g_w3")):
        assert rel_err(wi.grad.numpy(), g[key]) < 1e-5
    _, z_eval, mu_eval, lv_eval, _ = port.graph_ae_gcn_loss(x, *[wi.detach() for wi in w], an, adj, eps=None)
    assert rel_err(z_eval.numpy(), g["eval_z"]) < 1e-6 and rel_err(lv_eval.numpy(), g["eval_logvar"]) < 1e-6


def _load_feature_ae(g):
    dim = g["X"].shape[1]
    model = port.FeatureAE(dim)
    model.load_state_dict({k[len("init."):]: torch.from_numpy(g[k]) for k in g.files if k.startswith("init.")})
    return model


def test_feature_ae_golden(golden):
    from oracle.make_golden import sample_index
    g = golden("feature_ae")
    X = torch.from_numpy(g["X"])
    bs = int(g["batch_size"])
    model = _load_feature_ae(g)
    z, recon = model(X[:bs])
    loss = port.feature_ae_loss(recon, X[:bs], "LTMG", float(g["regu_strength"]), torch.zeros(bs, X.shape[1]))
    loss.backward()
    assert rel_err(z.detach().numpy(), g["b0_z"]) < 1e-6 and rel_err(recon.detach().numpy(), g["b0_recon"]) < 1e-6
    assert abs(loss.item() - float(g["b0_loss_ltmg"])) <= 1e-6 * abs(float(g["b0_loss_ltmg"]))
    for k, p in model.named_parameters():
        gnp = p.grad.numpy()
        assert np.allclose(gnp.reshape(-1)[sample_index(gnp.size)], g[f"b0_grad.{k}.sample"], rtol=1e-4, atol=1e-6)
        assert abs(np.linalg.norm(gnp.astype(np.float64)) - float(g[f"b0_grad.{k}.norm"])) < 1e-5 * float(g[f"b0_grad.{k}.norm"])
    # one full epoch (two optimiser steps) of train_handler
    model = _load_feature_ae(g)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    _, z_all, recon_all = port.feature_ae_epoch(model, opt, X, bs, "LTMG", float(g["regu_strength"]))
    assert rel_err(z_all.numpy(), g["z_all"]) < 1e-5 and rel_err(recon_all.numpy(), g["recon_all"]) < 1e-5
    for k, v in model.state_dict().items():
        v = v.numpy()
        assert np.allclose(v.reshape(-1)[sample_index(v.size)], g[f"after.{k}.sample"], rtol=1e-4, atol=1e-6)


# ---- against the reference's feature2adj / preprocess_graph (fixture: oracle/make_golden.py::_feature2adj_fixture) --------------
def _csr(g, key, n):
    return sp.csr_matrix((g[f"{key}.adj_data"], g[f"{key}.adj_indices"], g[f"{key}.adj_indptr"]), shape=(n, n))


def test_port_vs_live_reference_knn_graph(golden):
    g = golden("scgnn_feature2adj")
    X = port.synthetic_embedding(257, d=24, n_clusters=5, seed=3)
    for k in (3, 15):
        adj, idx = port.feature2adj(X, k)
        assert np.array_equal(idx.reshape(-1), g[f"k{k}.edges_dst"])
        assert (_csr(g, f"k{k}", len(X)) != adj).nnz == 0
        an = port.preprocess_graph(adj).tocoo()
        assert np.array_equal(g[f"k{k}.norm_values"], an.data)
        assert np.array_equal(g[f"k{k}.norm_indices"], np.vstack((an.row, an.col)))


def test_port_vs_live_reference_fractional_neighbourhood(golden):
    # neighborhood_factor <= 1 means a fraction of N (scgnn2.py:651-654); default 0.05
    g = golden("scgnn_feature2adj")
    X = port.synthetic_embedding(120, d=8, n_clusters=3, seed=9)
    adj, idx = port.feature2adj(X, 0.05)
    assert idx.shape[1] == 6 and (_csr(g, "frac", len(X)) != adj).nnz == 0


def test_graph_ae_gat_golden(golden):
    """oracle.port GAT restatement vs the fixture generated from the reference's Graph_AE(use_GAT=True)."""
    g = golden("knn_graph")
    gg = golden("graph_ae_gat")
    n, k = g["knn_idx"].shape
    X = torch.from_numpy(g["X"])
    edge_index = torch.from_numpy(np.stack([np.repeat(np.arange(n), k), g["knn_idx"].reshape(-1)]).astype(np.int64))
    sd = {k_[len("init."):]: torch.from_numpy(gg[k_]).requires_grad_() for k_ in gg.files if k_.startswith("init.")}
    z = port.graph_ae_gat_forward(X, edge_index, sd)
    assert rel_err(z.detach().numpy(), gg["z"]) < 1e-6
    adj = sp.csr_matrix((np.ones(len(g["adj_indices"])), g["adj_indices"], g["adj_indptr"]), shape=(n, n))
    labels = torch.from_numpy((adj + sp.eye(n)).toarray()).float()
    loss = torch.nn.functional.binary_cross_entropy_with_logits(z @ z.t(), labels)
    loss.backward()
    assert abs(loss.item() - float(gg["loss"])) < 1e-6 * float(gg["loss"])
    for k_, v in sd.items():
        assert rel_err(v.grad.numpy(), gg["grad." + k_]) < 1e-5, k_


def test_spagcn_golden(golden):
    """The SpaGCN restatement against the reference's own search_l / forward / autograd / fit outputs."""
    g = golden("spagcn_dec")
    X, D, adj = g["X"], g["D"], g["adj_exp"]
    assert abs(port.spagcn_calculate_p(D, float(g["l"])) - float(g["p_at_l"])) < 1e-6
    assert port.spagcn_search_l(0.5, D) == float(g["l"])
    assert np.array_equal(np.exp(-1 * (D**2) / (2 * (float(g["l"])**2))), adj)
    mu = torch.tensor(g["mu"], requires_grad=True)
    W = torch.tensor(g["W0"], requires_grad=True)
    b = torch.tensor(g["b0"], requires_grad=True)
    z, q = port.spagcn_forward(torch.tensor(X), torch.tensor(adj), W, b, mu)
    p = port.spagcn_target(q).detach()
    loss = port.spagcn_kl(p, q)
    loss.backward()
    for name, val in (("s_z", z), ("s_q", q), ("s_p", p), ("s_dW", W.grad), ("s_db", b.grad), ("s_dmu", mu.grad)):
        assert np.allclose(val.detach().numpy(), g[name], rtol=1e-5, atol=1e-7), name
    assert abs(loss.item() - float(g["s_loss"])) < 1e-7
    assert np.allclose(port.spagcn_group_means(g["s_z"], g["init_y"]), g["mu"], rtol=1e-5, atol=1e-6)
    # whole training runs: Adam with frozen mu (A), Adam + weight decay + stop rule (B), SGD (C), fit_with_init (D)
    Wa, ba, mua, _ = port.spagcn_fit(X, adj, g["W0"], g["b0"], g["init_y"], 0.005, 25, tol=-1.0)
    assert np.allclose(Wa, g["A_W"], rtol=1e-4, atol=1e-6) and np.allclose(ba, g["A_b"], rtol=1e-4, atol=1e-6)
    assert np.allclose(mua, g["mu"], rtol=1e-5, atol=1e-6)
    Wb, bb, _, n_b = port.spagcn_fit(X, adj, g["W0"], g["b0"], g["init_y"], 0.005, 40, weight_decay=5e-4, tol=1e-3)
    assert np.allclose(Wb, g["B_W"], rtol=1e-4, atol=1e-6) and np.allclose(bb, g["B_b"], rtol=1e-4, atol=1e-6)
    Wc, bc, _, _ = port.spagcn_fit(X, adj, g["W0"], g["b0"], g["init_y"], 0.01, 12, opt="sgd", tol=-1.0)
    assert np.allclose(Wc, g["C_W"], rtol=1e-4, atol=1e-6) and np.allclose(bc, g["C_b"], rtol=1e-4, atol=1e-6)
    Wd, bd, mud, _ = port.spagcn_fit(X, adj, g["W0"], g["b0"], g["init_y"], 0.01, 8, update_interval=1, opt="sgd", train_mu=True)
    assert np.allclose(Wd, g["D_W"], rtol=1e-4, atol=1e-6) and np.allclose(mud, g["D_mu"], rtol=1e-4, atol=1e-6)


def test_pyg_lite_primitives_against_dense_formulas():
    """The restated torch_geometric pieces (oracle/pyg_lite.py) against dense per-target formulas."""
    from oracle import pyg_lite
    rng = np.random.default_rng(0)
    n, e = 23, 140
    src, dst = torch.from_numpy(rng.integers(0, n, e)), torch.from_numpy(rng.integers(0, n, e))
    ei = torch.stack([src, dst])
    sc = torch.from_numpy(rng.normal(size=(e, 1)).astype(np.float32))
    a = pyg_lite.softmax(sc, dst, None, n)
    for v in range(n):
        m = dst == v
        if m.any():
            ref = torch.softmax(sc[m, 0], 0)
            assert torch.allclose(a[m, 0], ref, atol=1e-6)
    x = torch.from_numpy(rng.normal(size=(n, 5)).astype(np.float32))

    class Sum(pyg_lite.MessagePassing):

        def message(self, x_j, w_i):
            return x_j * w_i

    w = torch.from_numpy(rng.normal(size=(n, 1)).astype(np.float32))
    out = Sum().propagate(ei, x=x, w=(None, w))
    dense = torch.zeros(n, n)
    dense.index_put_((dst, src), torch.ones(e), accumulate=True)          # row = target, column = source
    assert torch.allclose(out, (dense @ x) * w, atol=1e-5)
    ei2, _ = pyg_lite.remove_self_loops(torch.tensor([[0, 1, 2], [0, 2, 2]]))
    assert ei2.tolist() == [[1], [2]]
    ei3, _ = pyg_lite.add_self_loops(ei2, num_nodes=3)
    assert ei3.tolist() == [[1, 0, 1, 2], [2, 0, 1, 2]]


def test_dgl_lite_graphconv_against_dense_formula():
    """oracle/dgl_lite.GraphConv(norm="both") = D_in^-1/2 A D_out^-1/2 applied on the side dgl chooses."""
    from oracle import dgl_lite
    rng = np.random.default_rng(1)
    n = 17
    A = (rng.random((n, n)) < 0.25)
    np.fill_diagonal(A, True)
    src, dst = np.nonzero(A)                                             # edge u → v for A[u, v]
    g = dgl_lite.Graph(src, dst, n)
    Ad = torch.from_numpy(A.T.astype(np.float32))                        # aggregation matrix: row = destination
    din = Ad.sum(1).clamp(min=1).pow(-0.5)
    dout = Ad.sum(0).clamp(min=1).pow(-0.5)
    for fin, fout in ((9, 4), (4, 9)):
        conv = dgl_lite.GraphConv(fin, fout, activation=torch.tanh)
        x = torch.from_numpy(rng.normal(size=(n, fin)).astype(np.float32))
        if fin <= fout:      # aggregate first, then W
            ref = torch.tanh(din[:, None] * (Ad @ (dout[:, None] * x)) @ conv.weight + conv.bias)
        else:                # W first
            ref = torch.tanh(din[:, None] * (Ad @ ((dout[:, None] * x) @ conv.weight)) + conv.bias)
        assert torch.allclose(conv(g, x), ref, atol=1e-5)
    with pytest.raises(RuntimeError):
        dgl_lite.GraphConv(3, 3)(dgl_lite.Graph([0], [1], 3), torch.zeros(3, 3))


def test_stagate_and_graphsci_fixtures_are_self_consistent(golden):
    """Cheap invariants of the committed fixtures: tied / aliased STAGATE weights, GraphSCI loss bookkeeping."""
    g = golden("stagate")
    assert np.array_equal(g["fit.conv3.lin_src"], g["fit.conv2.lin_src"].T) and np.array_equal(g["fit.conv4.lin_src"], g["fit.conv1.lin_src"].T)
    assert np.array_equal(g["fit.conv2.att_src"], g["init.conv2.att_src"])          # never receives a gradient
    gn = np.sqrt(sum((g[k].astype(np.float64)**2).sum() for k in g.files if k.startswith("grad.")))
    assert abs(gn - float(g["grad_norm"])) < 1e-4 * gn
    s = golden("graphsci")
    la, le, kl, tr, va = s["e1.losses"]
    assert abs((la + le - kl) - tr) < 1e-6 * abs(tr)                                # loss = log_lik − kl  (graphsci.py:482-483)
    assert "grad.gnnmodel.dec_log_std.weight" not in s.files                        # dec_log_std never runs (:129)


def test_cellgene_and_adaptive_sage_golden(golden):
    """port.cell_feature_graph / adaptive_sage_neighbour_mean / ScDeepSortNet against the reference's own CellFeatureGraph
    and AdaptiveSAGE code (run on oracle/dgl_lite.py by make_golden) — the restatements the GPU tests compare with."""
    g = golden("cellgene")
    X = g["X"]
    n, G = X.shape
    for norm, tag in ((True, "norm"), (False, "raw")):
        src, dst, w = port.cell_feature_graph(X, normalize_edges=norm)
        assert np.array_equal(src.numpy(), g[f"{tag}.src"]) and np.array_equal(dst.numpy(), g[f"{tag}.dst"])      # edge list + order
        assert np.allclose(w.numpy(), g[f"{tag}.w"], rtol=1e-6, atol=0)
    assert np.array_equal(g["cell_id"], np.concatenate([np.arange(G), -np.ones(n)]).astype(np.int32))          # the naming quirk (:56-59)
    assert np.array_equal(g["feat_id"], np.concatenate([-np.ones(G), np.arange(n)]).astype(np.int32))
    assert np.array_equal(g["features"], np.vstack([g["gene_feat"], g["cell_feat"]]))
    src, dst, w = (torch.from_numpy(g[f"norm.{k}"]) for k in ("src", "dst", "w"))
    neigh = port.adaptive_sage_neighbour_mean(src, dst, w, torch.from_numpy(g["features"]), torch.from_numpy(g["alpha"]), G)
    assert np.allclose(neigh.numpy(), g["neigh"], rtol=1e-5, atol=1e-6)
    # the layer output ignores the aggregate (SURVEY App. B): Linear → ReLU on the destination features only
    z = torch.relu(torch.from_numpy(g["features"]) @ torch.from_numpy(g["sage_weight"]).T + torch.from_numpy(g["sage_bias"]))
    assert np.allclose(z.numpy(), g["sage_out"], rtol=1e-5, atol=1e-6)


def test_scdeepsort_training_golden(golden):
    """port.ScDeepSortNet / scdeepsort_epoch replaying the batches the reference's own ScDeepSort.fit saw (run on
    oracle/dgl_lite.py by make_golden): per-epoch loss and weights, the alpha that never trains, final probabilities."""
    g = golden("scdeepsort")
    feats, lab = torch.from_numpy(g["feats"]), g["labels"]
    n, G = g["X"].shape
    c, hid, n_lab = feats.shape[1], int(g["hid"]), int(lab.max()) + 1
    net = port.ScDeepSortNet(c, hid, n_lab, G)
    with torch.no_grad():
        net.sage_linear.weight.copy_(torch.from_numpy(g["init.layers.0.layers.1.weight"]))
        net.sage_linear.bias.copy_(torch.from_numpy(g["init.layers.0.layers.1.bias"]))
        net.linear.weight.copy_(torch.from_numpy(g["init.linear.weight"]))
        net.linear.bias.copy_(torch.from_numpy(g["init.linear.bias"]))
    assert np.array_equal(g["init.alpha"], np.ones((G + 2, 1), np.float32))
    full_labels = torch.cat([-torch.ones(G, dtype=torch.long), torch.from_numpy(lab).long()])
    # Adam over the parameters that receive gradients (alpha has none: torch skips it; weight decay never touches it either)
    opt = torch.optim.Adam([net.sage_linear.weight, net.sage_linear.bias, net.linear.weight, net.linear.bias], lr=1e-2, weight_decay=1e-4)
    for e in range(3):
        batches = [g[f"e{e}.batch{b}"] for b in range(int(g[f"e{e}.n_batches"]))]
        loss = port.scdeepsort_epoch(net, opt, feats, full_labels, batches)
        assert abs(loss - float(g["losses"][e])) < 1e-5 * abs(float(g["losses"][e]))
        assert np.allclose(net.sage_linear.weight.detach().numpy(), g[f"e{e}.layers.0.layers.1.weight"], rtol=1e-4, atol=1e-6)
        assert np.allclose(net.linear.weight.detach().numpy(), g[f"e{e}.linear.weight"], rtol=1e-4, atol=1e-6)
        assert np.array_equal(g[f"e{e}.alpha"], g["init.alpha"])                     # the aggregate is discarded → no gradient
    # the reference reloads its best-validation state; with the restatement's weights at that epoch the probabilities agree
    best = [e for e in range(3) if np.array_equal(g[f"e{e}.linear.weight"], g["best.linear.weight"])]
    assert best, "best state must be one of the epoch snapshots"
    with torch.no_grad():
        w1, b1 = torch.from_numpy(g["best.layers.0.layers.1.weight"]), torch.from_numpy(g["best.layers.0.layers.1.bias"])
        w2, b2 = torch.from_numpy(g["best.linear.weight"]), torch.from_numpy(g["best.linear.bias"])
        logits = torch.relu(feats[G:] @ w1.T + b1) @ w2.T + b2
        prob = torch.softmax(logits, -1).numpy()
    assert np.allclose(prob, g["prob"], rtol=1e-5, atol=1e-6) and np.array_equal(prob.argmax(1), g["pred"])


def test_weighted_graphconv_golden(golden):
    """port.weighted_graphconv against the reference's own WeightedGraphConv class (graph-sc) for every norm / agg mode."""
    g = golden("graphsc_conv")
    src, dst = torch.from_numpy(g["src"]).long(), torch.from_numpy(g["dst"]).long()
    x, w_e = torch.from_numpy(g["x"]), torch.from_numpy(g["w_e"])
    for norm in ("both", "right", "none"):
        for agg in ("sum", "mean"):
            out = port.weighted_graphconv(x, src, dst, w_e, torch.from_numpy(g[f"{norm}.W"]), torch.from_numpy(g[f"{norm}.b"]), norm=norm,
                                          agg=agg, act=torch.relu)
            assert np.allclose(out.numpy(), g[f"{norm}.{agg}"], rtol=1e-5, atol=1e-6), (norm, agg)


def test_umap_connectivities_against_closed_forms():
    """Independent checks of the loop-level UMAP restatement (scanpy/umap are absent, so there is no fixture): a vectorised
    re-derivation of the smooth-kNN bisection, the fuzzy-union identity on the dense matrices, and analytically known cases."""
    rng = np.random.default_rng(4)
    n, d, k = 120, 6, 10
    X = rng.normal(size=(n, d)).astype(np.float32)
    X[9] = X[2]                                                  # a zero distance to a non-self neighbour
    d2 = ((X[:, None, :].astype(np.float64) - X[None, :, :])**2).sum(-1)
    idx = np.argsort(d2, axis=1, kind="stable")[:, :k].astype(np.int32)
    dist = np.sqrt(np.take_along_axis(d2, idx, 1)).astype(np.float32)
    C = port.umap_connectivities(idx, dist)
    # (1) vectorised smooth_knn_dist: rho = first positive distance, sigma solves Σ_{j>=1} exp(-max(d-rho,0)/sigma) = log2(k)
    pos = np.where(dist > 0, dist, np.inf)
    rho = pos.min(1).astype(np.float32)
    lo, hi, mid = np.zeros(n), np.full(n, np.inf), np.ones(n)
    done = np.zeros(n, bool)
    target = np.log2(k)
    for _ in range(64):
        dd = (dist[:, 1:] - rho[:, None]).astype(np.float32).astype(np.float64)
        psum = np.where(dd > 0, np.exp(-dd / mid[:, None]), 1.0).sum(1)
        done |= np.abs(psum - target) < 1e-5
        up = (psum > target) & ~done
        dn = (psum <= target) & ~done
        hi = np.where(up, mid, hi)
        lo = np.where(dn, mid, lo)
        mid = np.where(up, (lo + hi) / 2, np.where(dn, np.where(np.isinf(hi), mid * 2, (lo + hi) / 2), mid))
    sigma = np.maximum(mid.astype(np.float32), (1e-3 * dist.mean(1)).astype(np.float32))
    # (2) membership strengths and the fuzzy union A + Aᵀ - A∘Aᵀ on dense matrices
    val = np.where(idx == np.arange(n)[:, None], 0.0, np.where((dist - rho[:, None] <= 0) | (sigma[:, None] == 0), 1.0,
                                                                np.exp(-((dist - rho[:, None]) / sigma[:, None])))).astype(np.float32)
    A = np.zeros((n, n), np.float32)
    np.add.at(A, (np.repeat(np.arange(n), k), idx.reshape(-1)), val.reshape(-1))
    dense = A + A.T - A * A.T
    assert np.allclose(C.toarray(), dense, rtol=1e-5, atol=1e-7)
    assert np.array_equal(C.toarray() != 0, dense != 0)
    # (3) analytic cases: every non-self neighbour at the SAME distance → d - rho = 0 → strength 1 for all of them
    idx2 = np.stack([np.arange(6), (np.arange(6) + 1) % 6, (np.arange(6) + 2) % 6], 1).astype(np.int32)
    dist2 = np.tile(np.array([0.0, 2.0, 2.0], np.float32), (6, 1))
    C2 = port.umap_connectivities(idx2, dist2).toarray()
    expect = np.zeros((6, 6), np.float32)
    for i in range(6):
        for j in ((i + 1) % 6, (i + 2) % 6):
            expect[i, j] = expect[j, i] = 1.0                   # 1 + 1 - 1·1 = 1 when both directions exist, 1 + 0 - 0 otherwise
    assert np.array_equal(C2, expect)


def _trunc32(x):
    """Round a float64 array toward zero to fp32 precision (the worst case assumed for the tensor-core accumulate)."""
    y = x.astype(np.float32)
    over = np.abs(y.astype(np.float64)) > np.abs(x)
    return np.where(over, np.nextafter(y, np.float32(0)), y).astype(np.float32)


@pytest.mark.parametrize("d,scale", [(128, 1.0), (50, 1.0), (128, 300.0), (16, 1e-3)])
def test_knn_tensor_core_filter_error_bound_is_sound(d, scale):
    """Host emulation of the fp16 hi/lo-split filter estimate of knn_tc.cu (operands 2^e·x split into fp16 pairs, the three
    products per 16-feature step accumulated in fp32 with TRUNCATING adds, fp32 norms and final fma) against the exact fp64
    squared distance: the bound `tc_err_rel` used by the refine proof (csrc/knn_tc.cu) must dominate the error — this is
    what makes the tensor-core kNN exact.  Includes vectors of very different norms."""
    rng = np.random.default_rng(d)
    n = 400
    X = (rng.normal(size=(n, d)) * scale + rng.normal(size=(1, d)) * 3 * scale).astype(np.float32)
    X[:7] *= 40.0
    dp = (d + 63) // 64 * 64
    e = 9 - int(np.frexp(np.abs(X).max())[1])
    s = np.float32(2.0**e)
    Xs = np.zeros((n, dp), np.float32)
    Xs[:, :d] = X * s
    hi = Xs.astype(np.float16)
    lo = (Xs - hi.astype(np.float32)).astype(np.float16)
    hi64, lo64 = hi.astype(np.float64), lo.astype(np.float64)
    q = slice(0, 60)
    acc = np.zeros((60, n), np.float32)
    for k0 in range(0, dp, 16):                                  # one MMA per product and 16-feature step
        ks = slice(k0, k0 + 16)
        for a, b in ((lo64, hi64), (hi64, lo64), (hi64, hi64)):
            acc = _trunc32(acc.astype(np.float64) + a[q, ks] @ b[:, ks].T)
    sqn = np.array([np.float32(np.sum(np.float32(r) * np.float32(r), dtype=np.float32)) for r in X], np.float32)   # row_sqnorm_kernel (fp32)
    inv_s2 = np.float32(2.0**(-2 * e))
    est = (np.float32(-2.0) * inv_s2 * acc + (sqn[q, None] + sqn[None, :])).astype(np.float32)
    true = ((X[q, None, :].astype(np.float64) - X[None, :, :].astype(np.float64))**2).sum(-1)
    err_rel = 7.62939453125e-06 + 1.1920928955078125e-07 * (d + 8)           # ktc::tc_err_rel
    rmax = float(sqn.max())
    bound = err_rel * (sqn[q, None].astype(np.float64) + rmax + 2.0 * np.sqrt(sqn[q, None].astype(np.float64) * rmax))
    worst = np.abs(est.astype(np.float64) - true) / bound
    assert worst.max() < 1.0, worst.max()
    assert worst.max() < 0.5                                                 # comfortable margin, not a knife edge


def _tf32(x):
    """Truncate fp32 values to tf32 (the operand precision of the tensor-core MMA: top 19 bits of the fp32 container)."""
    return (np.ascontiguousarray(x, dtype=np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def test_decoder_tf32_split_scheme_precision_on_host():
    """Host emulation of the arithmetic of gae_tc.cu (the tf32 hi/lo-split tensor-core decoder): logits from the three products
    lo·hi + hi·lo + hi·hi of hi = x & 0xFFFFE000 and lo = x − hi (lo truncated to tf32 by the MMA), per-tile accumulation with
    truncating adds; σ split the same way for the gradient product against Z_J, tiles summed in fp32 — against fp64.  Shows the
    scheme carries fp32-grade precision (what lets the GPU tests hold 2e-6 on the loss and 2e-5 on dz)."""
    rng = np.random.default_rng(3)
    n, d, bt = 512, 16, 128
    z = (rng.normal(size=(n, d)) * 0.4).astype(np.float32)

    def split(x):
        h = _tf32(x)
        return h, _tf32(x - h)

    zh, zl = split(z)
    acc = np.zeros((n, n), np.float32)
    for k0 in range(0, d, 8):                       # K = 8 per instruction, three products, truncating adds
        ks = slice(k0, k0 + 8)
        for a, b in ((zl, zh), (zh, zl), (zh, zh)):
            acc = _trunc32(acc.astype(np.float64) + a[:, ks].astype(np.float64) @ b[:, ks].astype(np.float64).T)
    x_true = z.astype(np.float64) @ z.astype(np.float64).T
    assert np.abs(acc - x_true).max() < 4e-6 * np.abs(x_true).max()            # logits: ≈ 2^-18 relative to the largest logit
    g = (1.0 / (1.0 + np.exp(-acc.astype(np.float64)))).astype(np.float32)
    gh, gl = split(g)
    dz = np.zeros((n, d), np.float32)
    for j0 in range(0, n, bt):                      # one J tile: 16 k-steps of 8 columns accumulate in the MMA registers
        big = np.zeros((n, d), np.float32)
        small = np.zeros((n, d), np.float32)
        for k0 in range(j0, j0 + bt, 8):
            ks = slice(k0, k0 + 8)
            big = _trunc32(big.astype(np.float64) + gh[:, ks].astype(np.float64) @ zh[ks].astype(np.float64))
            small = _trunc32(small.astype(np.float64) + gl[:, ks].astype(np.float64) @ zh[ks].astype(np.float64))
            small = _trunc32(small.astype(np.float64) + gh[:, ks].astype(np.float64) @ zl[ks].astype(np.float64))
        dz = (dz + (big + small)).astype(np.float32)  # the tile's sum joins the fp32 total (round to nearest)
    sig = 1.0 / (1.0 + np.exp(-x_true))
    dz_true = sig @ z.astype(np.float64)
    assert np.linalg.norm(dz - dz_true) / np.linalg.norm(dz_true) < 2e-6


def test_plain_c_restatements_agree_with_the_port(golden):
    """oracle/c (plain C, built by oracle/Makefile) as an independent checker: CSR aggregate, fp64 kNN ranking and the
    Graph-AE decoder loss + gradient against oracle/port.py and the reference fixtures."""
    from oracle import c_oracle
    g = golden("knn_graph")
    X, k = g["X"], int(g["k"])
    for qi in (0, 17, len(X) - 1):
        idx, dist = c_oracle.knn_rank(X, qi, k)
        assert np.array_equal(idx, g["knn_idx"][qi]) and np.array_equal(1 / (dist + 1e-16), g["knn_w"][qi])       # bit-exact vs the reference
    rng = np.random.default_rng(0)
    S = rng.normal(size=(len(X), 12)).astype(np.float32)
    A = sp.csr_matrix((g["norm_data"], g["norm_indices"], g["norm_indptr"]), shape=(len(X), len(X)))
    assert np.allclose(c_oracle.csr_spmm(A.indptr, A.indices, A.data, S), A @ S, rtol=1e-5, atol=1e-6)
    # decoder: dense torch formula of the port (scgnn2.py:603-609) vs the C loops
    n, d = 150, 16
    z = torch.tensor((rng.normal(size=(n, d)) * 0.4).astype(np.float32), requires_grad=True)
    adj, _ = port.feature2adj(port.synthetic_embedding(n, d=8, seed=2), 5)
    L = (adj + sp.eye(n)).tocsr()
    L.sort_indices()
    pw, norm = port.gae_norm_constants(adj)
    loss = port.gae_loss(torch.mm(z, z.t()), torch.from_numpy(L.toarray()).float(), None, None, n, norm, pw)
    loss.backward()
    c_loss, c_dz = c_oracle.gae_loss_grad(z.detach().numpy(), L.indptr, L.indices, norm, pw)
    assert abs(c_loss - loss.item()) < 1e-5 * abs(loss.item())
    assert np.linalg.norm(c_dz - z.grad.numpy()) / np.linalg.norm(z.grad.numpy()) < 1e-4      # torch side is fp32
