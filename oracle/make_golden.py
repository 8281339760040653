"""Generate the golden fixtures in ``tests/golden/`` by running the REFERENCE's own code
(through ``oracle.ref_loader``) on small seeded inputs.  TEST INFRASTRUCTURE.

Run in the build container (needs ``/root/reference``):  ``python -m oracle.make_golden``
The fixtures are committed; the GPU box never runs this script.
"""
from __future__ import annotations

import warnings
from pathlib import Path

import numpy as np
import scipy.sparse as sp
import torch

from . import port, ref_loader

OUT = Path(__file__).resolve().parent.parent / "tests" / "golden"


def _knn_graph_fixture(ref):
    """feature2adj + preprocess_graph + gae constants (scgnn2.py:650-689,1191-1209,567-569)."""
    X = port.synthetic_embedding(300, d=16, n_clusters=4, seed=11)
    k = 10
    adj, adj_train, edge_list = ref.feature2adj(X, k, False)
    adj_train = sp.csr_matrix(adj_train)
    adj_train.sort_indices()
    knn_idx = np.array([e[1] for e in edge_list], dtype=np.int64).reshape(X.shape[0], k)
    knn_w = np.array([e[2] for e in edge_list], dtype=np.float64).reshape(X.shape[0], k)
    adj_norm = ref.preprocess_graph(adj_train).coalesce()
    an = sp.csr_matrix((adj_norm.values().numpy(), adj_norm.indices().numpy()), shape=tuple(adj_norm.shape))
    an.sort_indices()
    n = X.shape[0]
    pos_weight = float(n * n - adj_train.sum()) / adj_train.sum()
    norm = n * n / float((n * n - adj_train.sum()) * 2)
    global _KNN_IDX
    _KNN_IDX = knn_idx
    np.savez_compressed(OUT / "knn_graph.npz", X=X, k=k, knn_idx=knn_idx, knn_w=knn_w,
                        adj_indptr=adj_train.indptr, adj_indices=adj_train.indices,
                        norm_indptr=an.indptr, norm_indices=an.indices, norm_data=an.data.astype(np.float32),
                        pos_weight=pos_weight, norm=norm)
    return X, adj_train, an, pos_weight, norm


def _graph_ae_fixture(ref, X, adj_train, an, pos_weight, norm):
    """Graph_AE GCN branch: forward, loss, gradients, one Adam step (scgnn2.py:373-412,479-502,555-595,603-615)."""
    torch.manual_seed(3)
    n = X.shape[0]
    model = ref.Graph_AE(X.shape[1], 16, 0, 2, 64)
    x = torch.from_numpy(X)
    adj_t = ref.sparse_mx_to_torch_sparse_tensor(an)
    labels = torch.from_numpy((adj_train + sp.eye(n)).toarray()).float()
    w = {k: v.detach().clone().numpy() for k, v in model.state_dict().items() if k.startswith("gc")}
    out = dict(w1=w["gc1.weight"], w2=w["gc2.weight"], w3=w["gc3.weight"])

    # eval mode: z = mu
    model.eval()
    z, info, recon = model(x, adj_t, use_GAT=False)
    out.update(eval_z=z.detach().numpy(), eval_mu=info[0].detach().numpy(), eval_logvar=info[1].detach().numpy())

    # training mode with recorded noise
    model.train()
    opt = torch.optim.Adam(model.parameters(), lr=1e-2)
    torch.manual_seed(5)
    eps = torch.randn(n, 16)
    torch.manual_seed(5)  # reparameterize draws randn_like(std) first thing → identical eps
    opt.zero_grad()
    z, info, recon = model(x, adj_t, use_GAT=False)
    assert torch.allclose(z, eps * torch.exp(info[1]) + info[0])
    loss = ref.gae_loss_function(preds=recon, labels=labels, mu=info[0], logvar=info[1], n_nodes=n, norm=norm,
                                 pos_weight=pos_weight)
    loss.backward()
    out.update(eps=eps.numpy(), train_z=z.detach().numpy(), loss=np.float64(loss.item()),
               g_w1=model.gc1.weight.grad.numpy().copy(), g_w2=model.gc2.weight.grad.numpy().copy(),
               g_w3=model.gc3.weight.grad.numpy().copy())
    opt.step()
    out.update(w1_after=model.gc1.weight.detach().numpy().copy(), w2_after=model.gc2.weight.detach().numpy().copy(),
               w3_after=model.gc3.weight.detach().numpy().copy())
    # hidden1 for the layer-level check
    hidden1 = ref.GraphConvolution(X.shape[1], 32, 0.)
    with torch.no_grad():
        hidden1.weight.copy_(torch.from_numpy(out["w1"]))
        out["hidden1"] = hidden1(x, adj_t).numpy()
    np.savez_compressed(OUT / "graph_ae_gcn.npz", **out)


def _gat_fixture(ref, X, knn_idx, adj_train):
    """Graph_AE with use_GAT=True (scgnn2.py:376-378, 883-1215, 560-563, 618-619): forward, plain-BCE loss,
    gradients of every GAT parameter, one Adam step."""
    torch.manual_seed(13)
    n, k = knn_idx.shape
    model = ref.Graph_AE(X.shape[1], 16, 0, 2, 64)
    # non-zero biases so that the bias path is exercised (the reference initialises them to zero)
    with torch.no_grad():
        for layer in model.gat.gat_net:
            layer.bias.normal_(0, 0.1)
    sd = {k_: v.detach().clone().numpy() for k_, v in model.state_dict().items() if k_.startswith("gat.")}
    edge_index = torch.from_numpy(np.stack([np.repeat(np.arange(n), k), knn_idx.reshape(-1)]).astype(np.int64))
    labels = torch.from_numpy((adj_train + sp.eye(n)).toarray()).float()
    model.train()
    opt = torch.optim.Adam(model.parameters(), lr=1e-2)
    opt.zero_grad()
    x = torch.from_numpy(X)
    embed, _, recon = model(x, edge_index, use_GAT=True)
    loss = ref.loss_function(preds=recon, labels=labels)
    loss.backward()
    out = {"init." + k_: v for k_, v in sd.items()}
    out.update(z=embed.detach().numpy(), loss=np.float64(loss.item()))
    for k_, p in model.named_parameters():
        if k_.startswith("gat."):
            out["grad." + k_] = p.grad.numpy().copy()
    # layer-1 output for a layer-level check
    with torch.no_grad():
        out["layer0_out"] = model.gat.gat_net[0]((x, edge_index))[0].numpy()
    opt.step()
    out.update({"after." + k_: v.detach().numpy().copy() for k_, v in model.state_dict().items() if k_.startswith("gat.")})
    np.savez_compressed(OUT / "graph_ae_gat.npz", **out)


def sample_index(size: int) -> np.ndarray:
    """Fixed pseudo-random sample of flat indices used to spot-check large tensors."""
    return np.sort(np.random.default_rng(size).choice(size, size=min(2000, size), replace=False))


def _sample(a: np.ndarray) -> np.ndarray:
    return a.reshape(-1)[sample_index(a.size)].copy()


def _feature_ae_fixture(ref):
    """Feature_AE + train_handler/loss_function_graph: two optimiser steps on two batches
    (scgnn2.py:338-370,1217-1315).  dim kept small (32) and post-step weights / gradients stored as
    a fixed 2000-element sample + Frobenius norm per tensor so the fixture stays small."""
    torch.manual_seed(7)
    n, g, bs = 160, 32, 80
    X = port.synthetic_expression(n, g, density=0.3, seed=2)
    model = ref.Feature_AE(dim=g)
    init = {k: v.detach().clone().numpy() for k, v in model.state_dict().items()}
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    loader = torch.utils.data.DataLoader(ref.ExpressionDataset(X), batch_size=bs)
    trs = torch.zeros(n, g)
    param = {"device": "cpu", "epoch_num": 0, "total_epoch": 1, "n_feature_orig": g}
    import logging
    logging.getLogger("dance-ref-stub").setLevel(logging.WARNING)
    _, z_all, recon_all = ref.train_handler(model=model, train_loader=loader, optimizer=opt, TRS=trs, total_epoch=1,
                                            impute_regu=None, regu_type=["LTMG", "noregu"], regu_strength=0.9,
                                            masked_prob=0, param=param)
    after = {k: v.detach().clone().numpy() for k, v in model.state_dict().items()}
    out = {"X": X, "batch_size": bs, "regu_strength": 0.9, "z_all": z_all.detach().numpy(),
           "recon_all": recon_all.detach().numpy()}
    out.update({f"init.{k}": v for k, v in init.items()})
    for k, v in after.items():
        out[f"after.{k}.sample"], out[f"after.{k}.norm"] = _sample(v), np.float64(np.linalg.norm(v.astype(np.float64)))
    # single-batch forward/loss/grad snapshot ("noregu" and "LTMG") from the initial weights
    m2 = ref.Feature_AE(dim=g)
    m2.load_state_dict({k: torch.from_numpy(v) for k, v in init.items()})
    xb = torch.from_numpy(X[:bs])
    z, recon = m2(xb)
    loss = ref.loss_function_graph(recon, xb.clone(), regulationMatrix={"LTMG_regu": trs[:bs]}, regu_strength=0.9,
                                   regularizer_type="LTMG", param=param)
    loss.backward()
    out.update(b0_z=z.detach().numpy(), b0_recon=recon.detach().numpy(), b0_loss_ltmg=np.float64(loss.item()))
    for k, p in m2.named_parameters():
        gnp = p.grad.numpy()
        out[f"b0_grad.{k}.sample"], out[f"b0_grad.{k}.norm"] = _sample(gnp), np.float64(np.linalg.norm(gnp.astype(np.float64)))
    np.savez_compressed(OUT / "feature_ae.npz", **out)


def _matrix_fixture():
    """utils/matrix.py pairwise_distance (numba) on a seeded 40×7 matrix."""
    mx = ref_loader.matrix()
    X = np.random.default_rng(4).normal(size=(40, 7)).astype(np.float32)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        D = mx.pairwise_distance(X, 0)
    np.savez_compressed(OUT / "pairwise.npz", X=X, D=D)


def _spagcn_fixture():
    """SpaGCN (spagcn.py): search_l / calculate_p, SimpleGCDEC forward / target / KL loss / autograd gradients, and the
    reference's own ``fit`` (Adam, mu frozen because the optimiser is created before ``self.mu`` exists, spagcn.py:464-495),
    ``fit`` with SGD, the early-stop rule, and ``fit_with_init`` (mu trained)."""
    import copy
    import logging
    logging.getLogger("dance").setLevel(logging.WARNING)
    ref = ref_loader.spagcn()
    mx = ref_loader.matrix()
    rng = np.random.default_rng(11)
    side, h, K = 16, 12, 3
    gx, gy = np.meshgrid(np.arange(side), np.arange(side), indexing="ij")
    xy = np.stack([gx.ravel() * 10 + rng.integers(-2, 3, side * side), gy.ravel() * 10 + rng.integers(-2, 3, side * side)], 1)
    n = xy.shape[0]
    domain = (xy[:, 0] > 55).astype(int) + (xy[:, 1] > 95).astype(int)
    centers = rng.normal(scale=2.0, size=(K, h))
    X = (centers[domain] + rng.normal(scale=1.0, size=(n, h))).astype(np.float32)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        D = mx.pairwise_distance(xy.astype(np.float32), 0)
    l = ref.search_l(0.5, D, start=0.01, end=1000, tol=0.01, max_run=100)
    p_at_l = ref.calculate_p(D, l)
    adj_exp = np.exp(-1 * (D**2) / (2 * (l**2)))
    out = dict(xy=xy, X=X, D=D, l=np.float64(l), p_at_l=np.float64(p_at_l), adj_exp=adj_exp, K=K)

    def fresh():
        torch.manual_seed(3)
        return ref.SimpleGCDEC(h, h)

    m0 = fresh()
    out["W0"] = m0.gc.weight.detach().numpy().copy()
    out["b0"] = m0.gc.bias.detach().numpy().copy()

    # run A: reference fit, Adam, never stops early (tol < 0)
    np.random.seed(0)
    mA = fresh()
    mA.fit(X, adj_exp, lr=0.005, epochs=25, weight_decay=0, opt="admin", init="kmeans", n_clusters=K, init_spa=True, tol=-1.0)
    init_y = np.asarray(mA.trajectory[0]).astype(np.int64)
    out.update(init_y=init_y, mu=mA.mu.detach().numpy().copy(), A_W=mA.gc.weight.detach().numpy().copy(),
               A_b=mA.gc.bias.detach().numpy().copy())
    zA, qA = mA.predict(X, adj_exp)
    out.update(A_z=zA.detach().numpy(), A_q=qA.detach().numpy())

    # one restated step at the initial state for kernel-level checks (reference forward / target / loss + autograd)
    m1 = fresh()
    m1.mu = torch.nn.Parameter(torch.tensor(out["mu"]))
    z, q = m1(torch.FloatTensor(X), torch.FloatTensor(adj_exp))
    p = m1.target_distribution(q).data
    loss = m1.loss_function(p, q)
    z.retain_grad()
    loss.backward()
    out.update(s_z=z.detach().numpy(), s_q=q.detach().numpy(), s_p=p.numpy(), s_loss=np.float64(loss.item()),
               s_dz=z.grad.numpy(), s_dW=m1.gc.weight.grad.numpy(), s_db=m1.gc.bias.grad.numpy(), s_dmu=m1.mu.grad.numpy())

    # run B: Adam with weight decay and the default stopping tolerance
    np.random.seed(0)
    mB = fresh()
    mB.fit(X, adj_exp, lr=0.005, epochs=40, weight_decay=5e-4, opt="admin", init="kmeans", n_clusters=K, init_spa=True, tol=1e-3)
    assert np.array_equal(np.asarray(mB.trajectory[0]), init_y)
    out.update(B_W=mB.gc.weight.detach().numpy().copy(), B_b=mB.gc.bias.detach().numpy().copy())

    # run C: SGD with momentum
    np.random.seed(0)
    mC = fresh()
    mC.fit(X, adj_exp, lr=0.01, epochs=12, opt="sgd", init="kmeans", n_clusters=K, init_spa=True, tol=-1.0)
    assert np.array_equal(np.asarray(mC.trajectory[0]), init_y)
    out.update(C_W=mC.gc.weight.detach().numpy().copy(), C_b=mC.gc.bias.detach().numpy().copy())

    # run D: fit_with_init on top of a fresh model that already owns mu (so mu is in the optimiser)
    mD = fresh()
    mD.mu = torch.nn.Parameter(torch.zeros(K, h))
    mD.fit_with_init(X, adj_exp, init_y, lr=0.01, epochs=8, update_interval=1, opt="sgd")
    out.update(D_W=mD.gc.weight.detach().numpy().copy(), D_b=mD.gc.bias.detach().numpy().copy(),
               D_mu=mD.mu.detach().numpy().copy())
    np.savez_compressed(OUT / "spagcn_dec.npz", **out)


def _stagate_fixture():
    """STAGATE (stagate.py): the reference's GATConv / Stagate.forward / pretrain executed on oracle/pyg_lite.py, plus
    sklearn's radius / kNN graphs as used by StagateGraph (spatial_graph.py:143-151)."""
    from sklearn.neighbors import NearestNeighbors
    ref = ref_loader.stagate()
    rng = np.random.default_rng(17)
    side = 14
    gx, gy = np.meshgrid(np.arange(side), np.arange(side), indexing="ij")
    xy = np.stack([gx.ravel() * 100 + (gy.ravel() % 2) * 50 + rng.integers(-3, 4, side * side),
                   gy.ravel() * 87 + rng.integers(-3, 4, side * side)], 1).astype(np.int64)
    n = xy.shape[0]
    dims = [36, 24, 8]
    dom = (xy[:, 0] > 650).astype(int) + (xy[:, 1] > 600).astype(int)
    X = (rng.normal(scale=1.5, size=(3, dims[0]))[dom] + rng.normal(size=(n, dims[0]))).astype(np.float32)
    adj_r = NearestNeighbors(radius=150).fit(xy).radius_neighbors_graph(xy).tocsr()
    adj_r.sort_indices()
    adj_k = NearestNeighbors(n_neighbors=5).fit(xy).kneighbors_graph(xy).tocsr()
    adj_k.sort_indices()
    out = dict(xy=xy, X=X, dims=np.array(dims), radius=np.float64(150), r_indptr=adj_r.indptr, r_indices=adj_r.indices,
               k_indptr=adj_k.indptr, k_indices=adj_k.indices)
    edge = np.vstack(np.nonzero(adj_r))
    out["edge_index"] = edge

    torch.manual_seed(5)
    m = ref.Stagate(dims, device="cpu")
    for k, v in m.state_dict().items():
        out["init." + k] = v.numpy().copy()
    xt, et = torch.from_numpy(X), torch.from_numpy(edge.astype(np.int64))
    z, rec = m(xt, et)
    loss = torch.nn.functional.mse_loss(xt, rec)
    loss.backward()
    out.update(f_z=z.detach().numpy(), f_rec=rec.detach().numpy(), f_loss=np.float64(loss.item()))
    for k, p in m.named_parameters():
        if p.grad is not None:
            out["grad." + k] = p.grad.numpy().copy()
    total = torch.nn.utils.clip_grad_norm_(m.parameters(), 5)
    out["grad_norm"] = np.float64(total.item())
    m.zero_grad()

    # pretrain with a clipping threshold small enough to be active
    m.pretrain(X, edge, lr=1e-3, weight_decay=1e-4, epochs=8, gradient_clipping=0.05)
    for k, v in m.state_dict().items():
        out["fit." + k] = v.numpy().copy()
    out["fit_rep"] = m.rep.copy()
    np.savez_compressed(OUT / "stagate.npz", **out)


def _graphsci_fixture():
    """GraphSCI (graphsci.py): the reference's own GNNModel / AEModel / get_loss / fit running on oracle/dgl_lite.py, with
    dropout = 0 and ``torch.normal`` replaced by mean + std·ε for a recorded ε sequence (train, eval, train, eval, …)."""
    import contextlib
    import io
    import os
    import tempfile
    from . import dgl_lite
    ref = ref_loader.graphsci()
    rng = np.random.default_rng(23)
    n, g = 260, 48
    lat = rng.gamma(2.0, 1.0, size=(n, 5))
    load = rng.gamma(1.0, 0.6, size=(5, g))
    X = rng.poisson(lat @ load * rng.lognormal(0, 0.3, size=(n, 1))).astype(np.float32)
    X[X.sum(1) == 0, 0] = 1
    Xl = np.log1p(X)
    src, dst, w, _ = port.feature_feature_graph(Xl, 0.2, False, True)
    mask = rng.random((n, g)) < 0.9
    train_idx = np.arange(n)[: int(0.9 * n)]
    n_eps = 9
    eps = rng.normal(size=(n_eps, g, g)).astype(np.float32)
    out = dict(X=X, Xl=Xl, src=src, dst=dst, w=w, mask=mask, train_idx=train_idx, eps=eps)

    def graph():
        gr = dgl_lite.Graph(src, dst, g)
        gr.edata["weight"] = torch.tensor(w)
        gr.ndata["feat"] = torch.tensor(Xl.T.copy())
        return gr

    def fresh():
        torch.manual_seed(7)
        return ref.GraphSCI(num_cells=n, num_genes=g, dataset="fixture", dropout=0.0)

    real_normal = torch.normal
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        try:
            m = fresh()
            for scope, sd in (("aemodel", m.aemodel.state_dict()), ("gnnmodel", m.gnnmodel.state_dict())):
                for k, v in sd.items():
                    out[f"init.{scope}.{k}"] = v.numpy().copy()
            for n_epochs, tag in ((1, "e1"), (4, "e4")):
                m = fresh()
                it = iter(eps)
                torch.normal = lambda mean, std: mean + std * torch.from_numpy(next(it))
                with contextlib.redirect_stdout(io.StringIO()):
                    m.fit(torch.tensor(Xl), torch.tensor(X), graph(), mask=mask.copy(), n_epochs=n_epochs, lr=1e-3, weight_decay=1e-5,
                          train_idx=train_idx)
                out[f"{tag}.losses"] = np.array([m.loss_adj, m.loss_exp, m.kl, m.train_loss, m.valid_loss], dtype=np.float64)
                for scope, mod in (("aemodel", m.aemodel), ("gnnmodel", m.gnnmodel)):
                    for k, v in mod.state_dict().items():
                        out[f"{tag}.{scope}.{k}"] = v.numpy().copy()
                    if tag == "e1":
                        for k, prm in mod.named_parameters():
                            if prm.grad is not None:
                                out[f"grad.{scope}.{k}"] = prm.grad.numpy().copy()
                if tag == "e4":
                    with torch.no_grad():
                        pred = m.predict(torch.tensor(Xl), torch.tensor(X), graph(), mask=mask.copy())
                    out["e4.predict"] = pred.numpy().copy()
        finally:
            torch.normal = real_normal
            os.chdir(cwd)
    np.savez_compressed(OUT / "graphsci.npz", **out)


def _cellgene_fixture():
    """scDeepSort front end: the reference's own CellFeatureGraph.__call__ (cell_feature_graph.py:34-79) and
    AdaptiveSAGE.message_func / forward (models/nn/gnn.py:62-96) running on oracle/dgl_lite.py (dgl itself is absent)."""
    from dance_b200.data import AnnDataLite, Data       # host-side stand-ins for AnnData / dance.data.Data (no kernels involved)
    from . import dgl_lite
    cfg = ref_loader.cell_feature_graph()
    gnn = ref_loader.gnn()
    rng = np.random.default_rng(31)
    n, g, c = 37, 19, 6
    X = (rng.random((n, g)) < 0.3) * rng.gamma(2.0, 1.5, size=(n, g))
    X[5] = 0            # a cell without expressed genes
    X[:, 7] = 0         # a gene nobody expresses
    X = X.astype(np.float32)
    gene_feat = rng.normal(size=(g, c)).astype(np.float32)
    cell_feat = rng.normal(size=(n, c)).astype(np.float32)
    out = dict(X=X, gene_feat=gene_feat, cell_feat=cell_feat)
    for norm, tag in ((True, "norm"), (False, "raw")):
        data = Data(AnnDataLite(X.copy(), obsm={"f": cell_feat}, varm={"f": gene_feat}))
        cfg.CellFeatureGraph(cell_feature_channel="f", normalize_edges=norm)(data)
        gr = data.data.uns["CellFeatureGraph"]
        out.update({f"{tag}.src": gr.src.numpy(), f"{tag}.dst": gr.dst.numpy(), f"{tag}.w": gr.edata["weight"].numpy()})
        if norm:
            out.update(cell_id=gr.ndata["cell_id"].numpy(), feat_id=gr.ndata["feat_id"].numpy(), features=gr.ndata["features"].numpy())
            graph = gr
    # AdaptiveSAGE on the full graph (every node is a destination): message_func + fn.mean, then the layer output
    torch.manual_seed(3)
    alpha = torch.nn.Parameter(torch.rand(g + 2, 1) + 0.5)
    layer = gnn.AdaptiveSAGE(c, 5, alpha, torch.nn.Dropout(0.0), torch.nn.ReLU(), torch.nn.Identity())
    h = graph.ndata["features"]
    graph.ndata["h"] = h
    graph.update_all(layer.message_func, dgl_lite.function.mean("m", "neigh"))
    out.update(alpha=alpha.detach().numpy(), neigh=graph.ndata["neigh"].detach().numpy(), sage_weight=layer.layers[1].weight.detach().numpy(),
               sage_bias=layer.layers[1].bias.detach().numpy(), sage_out=layer(graph, h).detach().numpy())
    np.savez_compressed(OUT / "cellgene.npz", **out)


def _scdeepsort_fixture():
    """scDeepSort training: the reference's own ScDeepSort.fit / cal_loss / evaluate / predict_proba (scdeepsort.py:142-349) with
    its GNN + AdaptiveSAGE, running on oracle/dgl_lite.py (graph, full-neighbourhood blocks, dataloader).  The batches the
    reference saw are recorded so that the restatement / the GPU module can replay them."""
    import contextlib
    import io
    import os
    import tempfile
    from . import dgl_lite
    ref = ref_loader.scdeepsort()
    rng = np.random.default_rng(41)
    n, g, c, hid, n_lab, bs = 90, 30, 8, 7, 4, 16
    lab = rng.integers(0, n_lab, n)
    X = ((rng.random((n, g)) < 0.3) * rng.gamma(2.0, 1.5, size=(n, g))).astype(np.float32)
    X[np.arange(n), lab * 5] += 3.0                                   # a label-specific marker gene: something to learn
    src, dst, w = port.cell_feature_graph(X, True)
    feats = rng.normal(size=(n + g, c)).astype(np.float32)
    feats[g:] += np.eye(n_lab, c, dtype=np.float32)[lab] * 2.0
    out = dict(X=X, feats=feats, labels=lab, src=src.numpy(), dst=dst.numpy(), w=w.numpy(), hid=hid, batch_size=bs)

    def graph():
        gr = dgl_lite.Graph(src, dst, n + g)
        gr.edata["weight"] = w.clone()
        gr.ndata["cell_id"] = torch.cat([torch.arange(g, dtype=torch.int32), -torch.ones(n, dtype=torch.int32)])
        gr.ndata["features"] = torch.from_numpy(feats)
        return gr

    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        try:
            with contextlib.redirect_stdout(io.StringIO()):
                torch.manual_seed(9)
                m0 = ref.ScDeepSort(c, hid, 1, "sp", "ti", batch_size=bs)
                try:
                    m0.fit(graph(), torch.from_numpy(lab), epochs=0, lr=1e-2)         # builds the model: initial weights …
                except UnboundLocalError:
                    pass                                                              # … then trips over its own summary print (:204-207)
                for k, v in m0.model.state_dict().items():
                    out["init." + k] = v.numpy().copy()
                torch.manual_seed(9)
                dgl_lite.DataLoader.history = []
                m = ref.ScDeepSort(c, hid, 1, "sp", "ti", batch_size=bs)
                snaps, losses = [], []
                orig = m.cal_loss

                def cal_loss(graph_, idx):
                    start = len(dgl_lite.DataLoader.history)
                    loss = orig(graph_, idx)
                    snaps.append(([b.numpy().copy() for b in dgl_lite.DataLoader.history[start:]],
                                  {k: v.numpy().copy() for k, v in m.model.state_dict().items()}))
                    losses.append(loss)
                    return loss

                m.cal_loss = cal_loss
                m.fit(graph(), torch.from_numpy(lab), epochs=3, lr=1e-2, weight_decay=1e-4, val_ratio=0.2)
                prob = m.predict_proba(graph())
                pred, unsure = m.predict(graph(), unsure_rate=1.2, return_unsure=True)
        finally:
            os.chdir(cwd)
    out["losses"] = np.array(losses)
    for e, (batches, sd) in enumerate(snaps):
        out[f"e{e}.n_batches"] = len(batches)
        for b, idx in enumerate(batches):
            out[f"e{e}.batch{b}"] = idx
        for k, v in sd.items():
            out[f"e{e}.{k}"] = v
    for k, v in m.model.state_dict().items():
        out["best." + k] = v.numpy().copy()
    out.update(prob=prob, pred=pred, unsure=unsure)
    np.savez_compressed(OUT / "scdeepsort.npz", **out)


def _graphsc_conv_fixture():
    """graph-sc's in-tree WeightedGraphConv (graphsc.py:414-484) — the reference class itself, on oracle/dgl_lite.py."""
    from . import dgl_lite
    ref = ref_loader.graphsc()
    rng = np.random.default_rng(51)
    n, fin, fout = 40, 9, 5
    src = np.concatenate([rng.integers(0, n, 150), np.arange(n)])
    dst = np.concatenate([rng.integers(0, n, 150), np.arange(n)])
    w_e = rng.uniform(0.1, 2.0, size=(len(src), 1)).astype(np.float32)
    x = rng.normal(size=(n, fin)).astype(np.float32)
    out = dict(src=src, dst=dst, w_e=w_e, x=x)
    for norm in ("both", "right", "none"):
        torch.manual_seed(1)
        conv = ref.WeightedGraphConv(fin, fout, norm=norm, activation=torch.relu)
        with torch.no_grad():
            conv.bias.copy_(torch.linspace(-0.2, 0.2, fout))
        gr = dgl_lite.Graph(src, dst, n)
        gr.edata["weight"] = torch.from_numpy(w_e)
        out[f"{norm}.W"], out[f"{norm}.b"] = conv.weight.detach().numpy().copy(), conv.bias.detach().numpy().copy()
        for agg in ("sum", "mean"):
            out[f"{norm}.{agg}"] = conv(gr, torch.from_numpy(x), agg=agg).detach().numpy()
    np.savez_compressed(OUT / "graphsc_conv.npz", **out)


def _feature2adj_fixture(ref):
    """The reference's feature2adj / preprocess_graph on two seeded embeddings: integer k (3, 15) and a fractional
    neighbourhood (0.05 of N, scgnn2.py:651-654)."""
    out = {}
    X = port.synthetic_embedding(257, d=24, n_clusters=5, seed=3)
    for k in (3, 15):
        _, adj_train, edges = ref.feature2adj(X, k, False)
        a = sp.csr_matrix(adj_train)
        a.sort_indices()
        out[f"k{k}.edges_dst"] = np.array([e[1] for e in edges], dtype=np.int64)
        out[f"k{k}.adj_indptr"], out[f"k{k}.adj_indices"], out[f"k{k}.adj_data"] = a.indptr.astype(np.int64), a.indices.astype(np.int64), a.data
        an = ref.preprocess_graph(adj_train).coalesce()
        out[f"k{k}.norm_values"], out[f"k{k}.norm_indices"] = an.values().numpy(), an.indices().numpy()
    X2 = port.synthetic_embedding(120, d=8, n_clusters=3, seed=9)
    _, adj_train, _ = ref.feature2adj(X2, 0.05, False)
    a = sp.csr_matrix(adj_train)
    a.sort_indices()
    out["frac.adj_indptr"], out["frac.adj_indices"], out["frac.adj_data"] = a.indptr.astype(np.int64), a.indices.astype(np.int64), a.data
    np.savez_compressed(OUT / "scgnn_feature2adj.npz", **out)


def main():
    import sys
    OUT.mkdir(parents=True, exist_ok=True)
    only = [a for a in sys.argv[1:] if a in ("spagcn", "stagate", "graphsci", "cellgene", "scdeepsort", "graphsc_conv")]
    if only:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            for a in only:
                {"spagcn": _spagcn_fixture, "stagate": _stagate_fixture, "graphsci": _graphsci_fixture, "cellgene": _cellgene_fixture, "scdeepsort": _scdeepsort_fixture, "graphsc_conv": _graphsc_conv_fixture}[a]()
        return
    ref = ref_loader.scgnn2()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        X, adj_train, an, pw, norm = _knn_graph_fixture(ref)
        _feature2adj_fixture(ref)
        _graph_ae_fixture(ref, X, adj_train, an, pw, norm)
        _gat_fixture(ref, X, _KNN_IDX, adj_train)
        _feature_ae_fixture(ref)
        _matrix_fixture()
        _spagcn_fixture()
        _stagate_fixture()
        _graphsci_fixture()
        _cellgene_fixture()
        _scdeepsort_fixture()
        _graphsc_conv_fixture()
    for f in sorted(OUT.glob("*.npz")):
        print(f.name, f.stat().st_size)


if __name__ == "__main__":
    main()
