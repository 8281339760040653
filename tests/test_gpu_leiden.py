"""Leiden on the device (csrc/leiden.cu through dance_b200.leiden): its quality against a host fp64 recomputation, node
optimality and connectivity of its communities, the float64 restatement (tests/leiden_ref.py) and the host Louvain as
yardsticks, the exact cases, its labels, and SpaGCN's init="louvain" path that it completes."""
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.csgraph as csgraph
import torch

from leiden_ref import canonical, leiden_ref, quality

pytestmark = pytest.mark.gpu


def run(A, gamma, **kw):
    from dance_b200 import ops
    from dance_b200.leiden import leiden
    A = sp.csr_matrix(A, dtype=np.float32)
    res = leiden(ops.CSR.from_scipy(A), resolution=gamma, **kw)
    return res, res.labels.cpu().numpy()


def check_invariants(A, gamma, res, labels):
    """Reported quality = host fp64 Q/W; no single-vertex move gains more than 1e-9·W; communities connected; canonical labels."""
    A = sp.csr_matrix(A, dtype=np.float64)
    n = A.shape[0]
    assert labels.min() >= 0 and labels.max() == res.n_communities - 1
    assert np.array_equal(labels, canonical(labels))
    q = quality(A, labels, gamma)
    assert abs(res.quality - q) <= 1e-9 * max(abs(q), 1e-300), (res.quality, q)
    W = A.sum()
    k = np.asarray(A.sum(axis=1)).ravel()
    K = np.bincount(labels, weights=k, minlength=n)
    size = np.bincount(labels, minlength=n)
    Ad = sp.csr_matrix(A - sp.diags(A.diagonal()))
    M = sp.csr_matrix(Ad @ sp.csr_matrix((np.ones(n), (np.arange(n), labels)), shape=(n, n)))   # M[v, c] = w(v, c∖v)
    ad = Ad.tocoo()
    inside = labels[ad.row] == labels[ad.col]
    own = np.bincount(ad.row[inside], weights=ad.data[inside], minlength=n)
    Ka = K[labels] - k
    coo = M.tocoo()
    gain = 2 * (coo.data - own[coo.row] - gamma * k[coo.row] * (K[coo.col] - Ka[coo.row]) / W)
    gain[coo.col == labels[coo.row]] = 0
    worst = gain.max(initial=0.0)
    empty = np.where(size[labels] > 1, 2 * (-own + gamma * k * Ka / W), 0.0)
    worst = max(worst, empty.max(initial=0.0))
    assert worst <= 1e-9 * W, worst
    for c in range(res.n_communities):
        idx = np.flatnonzero(labels == c)
        if len(idx) > 1:
            assert csgraph.connected_components(A[idx][:, idx], directed=False)[0] == 1, c


def sbm(sizes, p_in, p_out, seed):
    import networkx as nx
    g = nx.random_partition_graph(sizes, p_in, p_out, seed=seed)
    A = nx.to_scipy_sparse_array(g, nodelist=range(sum(sizes)), format="csr").astype(np.float32)
    rng = np.random.default_rng(seed)
    U = sp.triu(A, k=1)
    U.data = rng.uniform(0.2, 1.0, U.nnz).astype(np.float32)
    return sp.csr_matrix(U + U.T), np.repeat(np.arange(len(sizes)), sizes)


def mixture(n, d=50, clusters=10, seed=0):
    rng = np.random.default_rng(seed)
    centres = rng.normal(scale=4.0, size=(clusters, d))
    return (centres[rng.integers(0, clusters, n)] + rng.normal(size=(n, d))).astype(np.float32)


def umap_graph(n, seed=0, n_neighbors=10):
    from dance_b200.leiden import neighbor_graph
    return neighbor_graph(torch.from_numpy(mixture(n, seed=seed)).cuda(), n_neighbors).to_scipy()


@pytest.mark.parametrize("gamma", [0.4, 1.0, 2.0])
def test_sbm_invariants_and_reference(cuda, gamma):
    A, _ = sbm([300, 200, 200, 150, 100, 50], 0.08, 0.01, seed=3)
    res, labels = run(A, gamma)
    check_invariants(A, gamma, res, labels)
    ref, _ = leiden_ref(A, gamma)
    assert res.quality >= quality(A, ref, gamma) - 0.005
    assert res.iterations >= 1 and res.levels >= 1


@pytest.mark.parametrize("gamma", [0.4, 1.0])
def test_umap_mixture_against_reference(cuda, gamma):
    A = umap_graph(20_000)
    res, labels = run(A, gamma)
    check_invariants(A, gamma, res, labels)
    ref, _ = leiden_ref(A, gamma)
    assert res.quality >= quality(A, ref, gamma) - 0.005


def test_large_graph_against_host_louvain(cuda):
    from dance_b200 import ops
    A = umap_graph(200_000, seed=1)
    res, labels = run(A, 1.0)
    check_invariants(A, 1.0, res, labels)
    _, _, mod = ops.louvain_host(A.indptr, A.indices, A.data)
    assert res.quality >= mod - 0.005, (res.quality, mod)


def test_planted_partition_is_recovered(cuda):
    from sklearn.metrics import adjusted_rand_score
    A, truth = sbm([120, 100, 80, 60], 0.5, 0.002, seed=5)
    res, labels = run(A, 1.0)
    assert adjusted_rand_score(truth, labels) == 1.0
    assert np.array_equal(labels, canonical(truth))


def test_isolated_vertices_and_edgeless_graphs_give_singletons(cuda):
    res, labels = run(sp.csr_matrix((50, 50), dtype=np.float32), 1.0)
    assert res.n_communities == 50 and np.array_equal(labels, np.arange(50)) and res.quality == 0.0
    A, _ = sbm([40, 40], 0.5, 0.0, seed=1)
    A = sp.block_diag([A, sp.csr_matrix((10, 10))]).tocsr()         # vertices 80..89 isolated
    res, labels = run(A, 1.0)
    assert res.n_communities == 12
    assert len(set(labels[80:])) == 10 and not set(labels[80:]) & set(labels[:80])
    check_invariants(A, 1.0, res, labels)


def test_tiny_resolution_gives_connected_components(cuda):
    blocks = [sbm([30, 30], 0.3, 0.05, seed=s)[0] for s in range(4)]
    A = sp.block_diag(blocks).tocsr()
    res, labels = run(A, 1e-6)
    _, comp = csgraph.connected_components(A, directed=False)
    assert res.n_communities == len(np.unique(comp))
    assert np.array_equal(labels, canonical(comp))


def test_large_resolution_gives_singletons(cuda):
    A, _ = sbm([50, 50], 0.2, 0.05, seed=2)
    A = sp.csr_matrix(A, dtype=np.float64)
    k = np.asarray(A.sum(axis=1)).ravel()
    coo = A.tocoo()
    bound = (coo.data * A.sum() / (k[coo.row] * k[coo.col])).max()
    res, labels = run(A, bound * 1.01)
    assert res.n_communities == 100 and np.array_equal(labels, np.arange(100))


def test_star_hub_with_100000_leaves(cuda):
    n = 100_001
    rows = np.zeros(n - 1, dtype=np.int64)
    cols = np.arange(1, n)
    U = sp.csr_matrix((np.ones(n - 1, dtype=np.float32), (rows, cols)), shape=(n, n))
    A = sp.csr_matrix(U + U.T)
    for gamma in (0.5, 1.0):
        res, labels = run(A, gamma)
        check_invariants(A, gamma, res, labels)


def test_aggregate_vertex_wider_than_4096(cuda):
    """5000 triangles, each tied to one hub vertex: after the first aggregation the hub has 5000 neighbour communities."""
    t = 5000
    hub = 3 * t
    tri = np.arange(3 * t).reshape(t, 3)
    r = np.concatenate([tri[:, 0], tri[:, 1], tri[:, 2], np.full(t, hub)])
    c = np.concatenate([tri[:, 1], tri[:, 2], tri[:, 0], tri[:, 0]])
    w = np.concatenate([np.ones(3 * t), np.full(t, 0.2)]).astype(np.float32)
    U = sp.csr_matrix((w, (r, c)), shape=(hub + 1, hub + 1))
    A = sp.csr_matrix(U + U.T)
    res, labels = run(A, 1.0)
    assert res.levels >= 2
    check_invariants(A, 1.0, res, labels)
    ref, _ = leiden_ref(A, 1.0)
    assert res.quality >= quality(A, ref, 1.0) - 0.005


def test_two_calls_give_identical_labels(cuda):
    A = umap_graph(30_000, seed=4)
    a, la = run(A, 0.7)
    b, lb = run(A, 0.7)
    assert np.array_equal(la, lb) and a.quality == b.quality and a.n_communities == b.n_communities
    assert np.all(np.diff(np.bincount(la)) <= 0)


def test_max_iterations_one_is_one_iteration(cuda):
    A, _ = sbm([100, 100, 100], 0.1, 0.02, seed=9)
    res, labels = run(A, 1.0, max_iterations=1)
    assert res.iterations == 1
    assert np.array_equal(labels, canonical(labels))


def test_neighbor_graph_is_what_neighborgraph_stores(cuda):
    from dance_b200 import ops
    from dance_b200.leiden import neighbor_graph
    X = torch.from_numpy(mixture(500)).cuda()
    idx, dist = ops.knn(X, 10, include_rank0=True)
    want = ops.umap_connectivities(idx, dist.float()).to_scipy()
    got = neighbor_graph(X, 10).to_scipy()
    assert (want != got).nnz == 0


# ---- SpaGCN -------------------------------------------------------------------------------------------------------------------
def _spatial(n=900, h=30, K=4, seed=11):
    rng = np.random.default_rng(seed)
    xy = rng.uniform(0, 300, size=(n, 2)).astype(np.float32)
    dom = np.minimum((xy[:, 0] // 75).astype(int), K - 1)
    X = (rng.normal(scale=2.0, size=(K, h))[dom] + rng.normal(size=(n, h))).astype(np.float32)
    D = np.sqrt(((xy[:, None, :] - xy[None, :, :])**2).sum(-1)).astype(np.float32)
    return X, D, dom


def test_simplegcdec_louvain_init_equals_init_labels(cuda):
    from dance_b200.leiden import leiden, neighbor_graph
    from dance_b200.modules.spagcn import SimpleGCDEC
    X, D, _ = _spatial()
    adj = np.exp(-(D**2) / (2 * 40.0**2)).astype(np.float32)
    kw = dict(lr=0.005, epochs=30, opt="admin", tol=-1.0, n_neighbors=10, res=0.4)
    a = SimpleGCDEC(X.shape[1], X.shape[1], device=cuda, seed=0).fit(X, adj, init="louvain", **kw)
    b = SimpleGCDEC(X.shape[1], X.shape[1], device=cuda, seed=0)
    b.bind(X, adj)
    labels = leiden(neighbor_graph(b._features().clone(), 10), resolution=0.4).labels.cpu().numpy()
    b.fit(X, adj, init_labels=labels, **kw)
    assert len(np.unique(labels)) > 1
    assert np.array_equal(a.trajectory[0], labels)
    for k, v in a.state_dict().items():
        assert torch.equal(v, b.state_dict()[k]), k


def test_spagcn_fit_with_default_arguments(cuda):
    from dance_b200.modules.spagcn import SpaGCN
    X, D, dom = _spatial()
    model = SpaGCN(l=40.0, device=cuda, seed=0)
    model.fit((X, D))
    pred = model.predict((X, D))
    assert pred.shape == (len(X), ) and model.model.n_clusters >= 2
    assert 0.0 <= model.default_score_func(dom, pred) <= 1.0
    assert model.score((X, D), dom) == model.default_score_func(dom, pred)


_SPAGCN_FLOW = '''
import argparse
import numpy as np
from dance.datasets.spatial import SpatialLIBDDataset
from dance.modules.spatial.spatial_domain.spagcn import SpaGCN, refine
from dance.utils import set_seed
if __name__ == "__main__":
    parser = argparse.ArgumentParser()
    parser.add_argument("--cache", action="store_true", help="Cache processed data.")
    parser.add_argument("--sample_number", type=str, default="151673")
    parser.add_argument("--beta", type=int, default=49, help="")
    parser.add_argument("--alpha", type=int, default=1, help="")
    parser.add_argument("--p", type=float, default=0.05)
    parser.add_argument("--l", type=float, default=0.5)
    parser.add_argument("--start", type=float, default=0.01)
    parser.add_argument("--end", type=float, default=1000)
    parser.add_argument("--tol", type=float, default=5e-3)
    parser.add_argument("--max_run", type=int, default=200)
    parser.add_argument("--epochs", type=int, default=200)
    parser.add_argument("--n_clusters", type=int, default=7)
    parser.add_argument("--step", type=float, default=0.1)
    parser.add_argument("--lr", type=float, default=0.05)
    parser.add_argument("--device", default="cpu")
    parser.add_argument("--seed", type=int, default=100)
    parser.add_argument("--num_runs", type=int, default=1)
    args = parser.parse_args()
    scores = []
    for seed in range(args.seed, args.seed + args.num_runs):
        set_seed(seed)
        model = SpaGCN(device=args.device)
        preprocessing_pipeline = model.preprocessing_pipeline(alpha=args.alpha, beta=args.beta)
        dataloader = SpatialLIBDDataset(data_id=args.sample_number)
        data = dataloader.load_data(transform=preprocessing_pipeline, cache=args.cache)
        (x, adj, adj_2d), y = data.get_train_data()
        l = model.search_l(args.p, adj, start=args.start, end=args.end, tol=args.tol, max_run=args.max_run)
        model.set_l(l)
        res = model.search_set_res((x, adj), l=l, target_num=args.n_clusters, start=0.4, step=args.step, tol=args.tol,
                                   lr=args.lr, epochs=args.epochs, max_run=args.max_run)
        pred = model.fit_predict((x, adj), init_spa=True, init="louvain", tol=args.tol, lr=args.lr, epochs=args.epochs,
                                 res=res)
        score = model.default_score_func(y, pred)
        print(f"ARI: {score:.4f}")
        refined_pred = refine(sample_id=data.data.obs_names.tolist(), pred=pred.tolist(), dis=adj_2d, shape="hexagon")
        score_refined = model.default_score_func(y, refined_pred)
        scores.append(score_refined)
        print(f"ARI (refined): {score_refined:.4f}")
    print(f"SpaGCN {args.sample_number}:")
    print(f"{scores}\\n{np.mean(scores):.5f} +/- {np.std(scores):.5f}")
'''


@pytest.fixture
def spatial_env(tmp_path, monkeypatch):
    monkeypatch.setenv("DANCE_B200_SYNTH", "cells=800,genes=300,types=5,density=0.5")
    monkeypatch.chdir(tmp_path)
    from dance_b200 import dropin
    assert set(dropin.install()) == {"dance", "scanpy"}
    yield tmp_path
    for k in [k for k in sys.modules if k == "dance" or k.startswith("dance.") or k == "scanpy" or k.startswith("scanpy.")]:
        del sys.modules[k]


def test_spagcn_example_script_runs_unchanged(cuda, spatial_env, capsys):
    """examples/spatial/spatial_domain/spagcn.py:33-61 (search_l, search_set_res, fit_predict with init="louvain", refine) at
    reduced epochs and max_run; only CLI arguments differ from the defaults (``--device cuda``: there is no CPU path)."""
    from dance_b200 import dropin
    script = spatial_env / "spagcn.py"
    script.write_text(_SPAGCN_FLOW)
    ns = dropin.run_example(script, ["--device", "cuda", "--epochs", "20", "--max_run", "30"])
    out = capsys.readouterr().out
    assert "ARI: " in out and "ARI (refined): " in out
    assert len(ns["scores"]) == 1 and -1.0 <= ns["scores"][0] <= 1.0
