"""SpaGCN path (BASELINE config 4): exp-adjacency / search_l, the DEC head kernels, and the SimpleGCDEC training loops
against fixtures produced by the REFERENCE's own ``fit`` / ``fit_with_init`` (oracle/make_golden.py::_spagcn_fixture)."""
import numpy as np
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu

TOL = 1e-4   # fp32 layer outputs / trained weights, relative (north_star)


def _t(a, cuda):
    return torch.as_tensor(np.ascontiguousarray(a)).to(cuda)


def test_exp_adj_and_search_l(cuda, golden):
    from dance_b200 import ops
    from dance_b200.modules import spagcn
    g = golden("spagcn_dec")
    D = _t(g["D"], cuda)
    l = float(g["l"])
    A, acc = ops.exp_adj(D, l, want_matrix=True, want_sum=True)
    assert np.allclose(A.cpu().numpy(), g["adj_exp"], rtol=5e-7, atol=1e-30)
    assert abs(acc.item() - g["adj_exp"].astype(np.float64).sum()) < 1e-3
    assert abs(spagcn.calculate_p(D, l) - float(g["p_at_l"])) < 1e-5
    assert spagcn.search_l(0.5, g["D"]) == l                      # same bisection path → the identical float
    assert spagcn.search_l(0.5, g["D"], start=50.0) is None       # "try smaller start point"
    assert spagcn.search_l(500.0, g["D"]) is None                 # "try bigger end point"


def test_dec_kernels_match_reference_autograd(cuda, golden):
    from dance_b200 import ops
    g = golden("spagcn_dec")
    z, mu = _t(g["s_z"], cuda), _t(g["mu"], cuda)
    q = ops.dec_q(z, mu, 0.2)
    assert rel_err(q, g["s_q"]) < 1e-5
    p = ops.dec_target(q)
    assert rel_err(p, g["s_p"]) < 1e-5
    q_out = torch.empty_like(q)
    labels = torch.empty(z.shape[0], dtype=torch.int32, device=cuda)
    loss, dz, dmu = ops.dec_kl_grad(z, mu, _t(g["s_p"], cuda), 0.2, q_out=q_out, labels_out=labels)
    assert abs(loss.item() - float(g["s_loss"])) < 1e-6
    assert rel_err(dz, g["s_dz"]) < TOL
    assert rel_err(dmu, g["s_dmu"]) < TOL
    assert torch.equal(q_out, q)
    assert np.array_equal(labels.cpu().numpy(), g["s_q"].argmax(1))


def test_dec_kernels_wide_cluster_count(cuda):
    """K > 32 exercises the second cluster slot of each lane; checked against the torch restatement + autograd."""
    from dance_b200 import ops
    from oracle import port
    rng = np.random.default_rng(5)
    n, h, K = 333, 50, 47
    z = torch.tensor(rng.normal(size=(n, h)).astype(np.float32), requires_grad=True)
    mu = torch.tensor(rng.normal(size=(K, h)).astype(np.float32), requires_grad=True)
    d2 = torch.sum((z.unsqueeze(1) - mu)**2, dim=2)
    q = (1.0 / ((1.0 + d2 / 0.2) + 1e-8))**1.2 / 2.0
    q = q / q.sum(1, keepdim=True)
    p = port.spagcn_target(q).detach()
    loss = port.spagcn_kl(p, q)
    loss.backward()
    zc, muc = z.detach().to(cuda), mu.detach().to(cuda)
    qg = ops.dec_q(zc, muc, 0.2)
    assert rel_err(qg, q.detach().numpy()) < 1e-5
    assert rel_err(ops.dec_target(qg), p.numpy()) < 1e-5
    labels = torch.empty(n, dtype=torch.int32, device=cuda)
    lg, dz, dmu = ops.dec_kl_grad(zc, muc, p.to(cuda), 0.2, labels_out=labels)
    assert abs(lg.item() - loss.item()) < 1e-5 * max(1.0, abs(loss.item()))
    assert rel_err(dz, z.grad.numpy()) < TOL and rel_err(dmu, mu.grad.numpy()) < TOL
    assert np.array_equal(labels.cpu().numpy(), q.detach().numpy().argmax(1))


def test_sgd_momentum_matches_torch(cuda):
    from dance_b200 import ops
    rng = np.random.default_rng(2)
    w0 = rng.normal(size=1001).astype(np.float32)
    grads = [rng.normal(size=1001).astype(np.float32) for _ in range(5)]
    ref = torch.nn.Parameter(torch.tensor(w0))
    opt = torch.optim.SGD([ref], lr=0.01, momentum=0.9, weight_decay=1e-3)
    w, buf = _t(w0, cuda), torch.zeros(1001, device=cuda)
    for step, gr in enumerate(grads, 1):
        ref.grad = torch.tensor(gr)
        opt.step()
        ops.sgd_momentum_step(w, _t(gr, cuda), buf, step, 0.01, 0.9, 1e-3)
    assert np.allclose(w.cpu().numpy(), ref.detach().numpy(), rtol=1e-6, atol=1e-7)


def _model(g, cuda):
    from dance_b200.modules.spagcn import SimpleGCDEC
    m = SimpleGCDEC(g["X"].shape[1], g["X"].shape[1], device=cuda)
    m.load_state_dict({"gc.weight": g["W0"], "gc.bias": g["b0"]})
    return m


def test_fit_adam_matches_reference_fit(cuda, golden):
    g = golden("spagcn_dec")
    m = _model(g, cuda)
    m.fit(g["X"], g["adj_exp"], lr=0.005, epochs=25, weight_decay=0, opt="admin", init="kmeans", n_clusters=3, tol=-1.0,
          init_labels=g["init_y"])
    assert m.epochs_run == 25
    assert rel_err(m.mu, g["mu"]) < 1e-5                       # cluster centres; frozen during fit (reference quirk)
    assert rel_err(m.params.p["gc.weight"], g["A_W"]) < TOL
    assert rel_err(m.params.p["gc.bias"], g["A_b"]) < TOL
    z, q = m.predict(g["X"], g["adj_exp"])
    assert rel_err(z, g["A_z"]) < TOL and rel_err(q, g["A_q"]) < TOL
    assert np.array_equal(m.trajectory[0], g["init_y"])


def test_fit_weight_decay_and_stop_rule(cuda, golden):
    from oracle import port
    g = golden("spagcn_dec")
    m = _model(g, cuda)
    m.fit(g["X"], g["adj_exp"], lr=0.005, epochs=40, weight_decay=5e-4, opt="admin", tol=1e-3, init_labels=g["init_y"])
    *_, n_ref = port.spagcn_fit(g["X"], g["adj_exp"], g["W0"], g["b0"], g["init_y"], 0.005, 40, weight_decay=5e-4, tol=1e-3)
    assert m.epochs_run == n_ref                               # stopped at the same epoch as the reference loop
    assert rel_err(m.params.p["gc.weight"], g["B_W"]) < TOL
    assert rel_err(m.params.p["gc.bias"], g["B_b"]) < TOL


def test_fit_sgd_and_fit_with_init(cuda, golden):
    g = golden("spagcn_dec")
    m = _model(g, cuda)
    m.fit(g["X"], g["adj_exp"], lr=0.01, epochs=12, opt="sgd", tol=-1.0, init_labels=g["init_y"])
    assert rel_err(m.params.p["gc.weight"], g["C_W"]) < TOL and rel_err(m.params.p["gc.bias"], g["C_b"]) < TOL
    m2 = _model(g, cuda)
    with pytest.raises(AttributeError):
        m2.fit_with_init(g["X"], g["adj_exp"], g["init_y"])     # no mu yet — the reference raises too
    m2.set_mu(np.zeros((3, g["X"].shape[1]), np.float32))
    m2.fit_with_init(g["X"], g["adj_exp"], g["init_y"], lr=0.01, epochs=8, update_interval=1, opt="sgd")
    assert rel_err(m2.params.p["gc.weight"], g["D_W"]) < TOL
    assert rel_err(m2.mu, g["D_mu"]) < TOL                      # mu IS trained here


def test_spagcn_module_end_to_end_larger(cuda):
    """N large enough for the tensor-core GEMM to build adj·X; compared with the torch restatement of the reference loop."""
    from dance_b200.modules.spagcn import SpaGCN
    from dance_b200 import ops
    from oracle import port
    rng = np.random.default_rng(21)
    n, h, K = 1536, 48, 5
    xy = rng.uniform(0, 400, size=(n, 2)).astype(np.float32)
    dom = np.minimum((xy[:, 0] // 80).astype(int), K - 1)
    X = (rng.normal(scale=2.0, size=(K, h))[dom] + rng.normal(size=(n, h))).astype(np.float32)
    D = port.pairwise_euclidean(xy)
    model = SpaGCN(device=cuda, seed=0)
    l = model.search_l(0.5, D)
    assert l == port.spagcn_search_l(0.5, D)
    model.set_l(l)
    with pytest.raises(ValueError):
        SpaGCN(device=cuda).fit((X, D))                          # l must be set first
    ops.reset_counters()
    pred = model.fit_predict((X, D), lr=0.005, epochs=20, opt="admin", init="kmeans", n_clusters=K, tol=-1.0, init_labels=dom)
    assert ops.counters()["launches"] > 0
    adj_exp = np.exp(-1 * (D**2) / (2 * (l**2)))
    sd0 = SpaGCN(device=cuda, seed=0)
    sd0.set_l(l)
    from dance_b200.modules.spagcn import SimpleGCDEC
    init = SimpleGCDEC(h, h, device=cuda, seed=0).state_dict()
    W, b, mu, _ = port.spagcn_fit(X, adj_exp, init["gc.weight"].cpu().numpy(), init["gc.bias"].cpu().numpy(), dom, 0.005, 20, tol=-1.0)
    assert rel_err(model.model.params.p["gc.weight"], W) < TOL
    assert rel_err(model.model.params.p["gc.bias"], b) < TOL
    z_ref, q_ref = port.spagcn_forward(torch.tensor(X), torch.tensor(adj_exp), torch.tensor(W), torch.tensor(b), torch.tensor(mu))
    q = model.predict_proba((X, D))
    assert rel_err(q, q_ref.numpy()) < TOL
    assert (pred == q_ref.numpy().argmax(1)).mean() > 0.999
    assert model.score((X, D), dom) > 0.8                        # ARI against the planted domains


def test_spagcn_graph_transforms(cuda):
    from dance_b200.data import AnnDataLite, Data
    from dance_b200.transforms import SpaGCNGraph, SpaGCNGraph2D
    from oracle import port
    rng = np.random.default_rng(8)
    n = 90
    xy = rng.integers(0, 60, size=(n, 2))
    xy_pixel = xy * 5 + rng.integers(0, 3, size=(n, 2))
    img = rng.integers(0, 255, size=(320, 310, 3)).astype(np.uint8)
    ad = AnnDataLite(np.zeros((n, 4), np.float32), obsm={"spatial": xy, "spatial_pixel": xy_pixel}, uns={"image": img})
    data = Data(ad)
    SpaGCNGraph(alpha=1, beta=49)(data)
    SpaGCNGraph2D()(data)
    # restatement of spagcn.py:81-116 (calculate_adj_matrix, histology=True)
    bh = round(49 / 2)
    g = np.array([np.mean(np.mean(img[max(0, px - bh):min(320, px + bh + 1), max(0, py - bh):min(310, py + bh + 1)], axis=0), axis=0)
                  for px, py in xy_pixel])
    v = g.var(0)
    c3 = (g * v).sum(1) / v.sum()
    z = (c3 - c3.mean()) / c3.std() * max(xy[:, 0].std(), xy[:, 1].std())
    ref3 = port.pairwise_euclidean(np.column_stack([xy, z]).astype(np.float32))
    ref2 = port.pairwise_euclidean(xy_pixel.astype(np.float32))
    assert np.allclose(ad.obsp["SpaGCNGraph"], ref3, rtol=1e-5, atol=1e-4)
    assert np.allclose(ad.obsp["SpaGCNGraph2D"], ref2, rtol=1e-5, atol=1e-4)
    assert ad.obsp["SpaGCNGraph"].dtype == np.float32
