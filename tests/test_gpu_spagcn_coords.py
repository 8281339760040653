"""SpaGCN from the spot coordinates (``matrix.SpotDistance`` and the ``spatial_ops.spatial_*`` sweeps) against the dense path: the same
bits for every pair's distance and weight, AX against float64, and the SpaGCN API run end to end on either form."""
import pickle

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return "cuda"


def _dense(P):
    from dance_b200 import ops, spatial_ops
    return ops.pairwise_l2_dense(torch.as_tensor(P).cuda())


def _weights64(rows, cols, l):
    """The fp32 weights of the dense path for the pairs rows × cols (bit-identical by construction), as float64."""
    from dance_b200 import ops, spatial_ops
    n = rows.shape[0]
    D = _dense(np.concatenate([rows, cols]))[:n, n:].contiguous()
    return ops.exp_adj(D, l)[0].double()


def test_spot_distance_materialises_the_dense_matrices(cuda):
    from dance_b200 import ops, spatial_ops
    from dance_b200.matrix import SpotDistance
    from dance_b200.modules.spagcn import SpaGCN
    rng = np.random.default_rng(0)
    for P in (rng.uniform(0, 1e4, size=(300, 2)).astype(np.float32), rng.normal(size=(257, 3)).astype(np.float32)):
        m = SpotDistance(P)
        assert m.shape == (P.shape[0], P.shape[0]) and m.dtype == np.float32
        D = _dense(P)
        assert np.array_equal(m.toarray(), D.cpu().numpy()) and np.array_equal(np.asarray(m), D.cpu().numpy())
        model = SpaGCN(l=float(np.median(D.cpu().numpy())) / 3)
        assert np.array_equal(model.calc_adj_exp(m).toarray(), model.calc_adj_exp(D).cpu().numpy())
        idx = rng.permutation(P.shape[0])[:100]
        assert np.array_equal(m[idx][:, idx].toarray(), D.cpu().numpy()[idx][:, idx])
        assert np.array_equal(m[:, idx[:7]].toarray(), D.cpu().numpy()[:, idx[:7]])
        back = pickle.loads(pickle.dumps(m))
        assert back._dev == {} and np.array_equal(back.toarray(), D.cpu().numpy())
    # rows and cols from different sets: the block of the joint matrix
    A, B = rng.normal(size=(33, 2)).astype(np.float32), rng.normal(size=(70, 2)).astype(np.float32)
    assert np.array_equal(SpotDistance(A, B).toarray(), _dense(np.concatenate([A, B])).cpu().numpy()[:33, 33:])
    with pytest.raises(IndexError):
        m[3]


def test_graph_transforms_coordinate_form(cuda):
    from dance_b200.data import AnnDataLite, Data
    from dance_b200.matrix import SpotDistance
    from dance_b200.transforms import SpaGCNGraph, SpaGCNGraph2D
    rng = np.random.default_rng(8)
    n = 90
    xy = rng.integers(0, 60, size=(n, 2))
    xy_pixel = xy * 5 + rng.integers(0, 3, size=(n, 2))
    img = rng.integers(0, 255, size=(320, 310, 3)).astype(np.uint8)
    make = lambda: Data(AnnDataLite(np.zeros((n, 4), np.float32), obsm={"spatial": xy, "spatial_pixel": xy_pixel}, uns={"image": img}))
    dense, coords = make(), make()
    SpaGCNGraph(alpha=1, beta=49)(dense)
    SpaGCNGraph2D()(dense)
    SpaGCNGraph(alpha=1, beta=49, dense=False)(coords)
    SpaGCNGraph2D(dense=False)(coords)
    for ch in ("SpaGCNGraph", "SpaGCNGraph2D"):
        m = coords.data.obsp[ch]
        assert isinstance(m, SpotDistance)
        assert np.array_equal(m.toarray(), dense.data.obsp[ch])
    assert repr(SpaGCNGraph(alpha=1, beta=49)) == "SpaGCNGraph(alpha=1, beta=49)"
    assert repr(SpaGCNGraph2D()) == "SpaGCNGraph2D()"
    assert repr(SpaGCNGraph(alpha=1, beta=49, dense=False)) == "SpaGCNGraph(alpha=1, beta=49, dense=False)"
    assert SpaGCNGraph2D(dense=False).hexdigest() != SpaGCNGraph2D().hexdigest()
    back = pickle.loads(pickle.dumps(coords))
    assert np.array_equal(back.data.obsp["SpaGCNGraph2D"].toarray(), dense.data.obsp["SpaGCNGraph2D"])
    # get_feature: unmaterialised for numpy / default, split indices applied; torch / sparse materialise
    got = coords.get_feature(return_type="numpy", channel="SpaGCNGraph2D", channel_type="obsp")
    assert isinstance(got, SpotDistance)
    assert coords.get_feature(return_type="default", channel="SpaGCNGraph2D", channel_type="obsp") is coords.data.obsp["SpaGCNGraph2D"]
    t = coords.get_feature(return_type="torch", channel="SpaGCNGraph2D", channel_type="obsp")
    assert isinstance(t, torch.Tensor) and np.array_equal(t.cpu().numpy(), dense.data.obsp["SpaGCNGraph2D"])
    sp_ = coords.get_feature(return_type="sparse", channel="SpaGCNGraph2D", channel_type="obsp")
    assert np.array_equal(sp_.toarray(), dense.data.obsp["SpaGCNGraph2D"])


def test_get_feature_split_subsets_the_coordinates(cuda):
    from dance_b200.data import AnnDataLite, Data
    from dance_b200.matrix import SpotDistance
    rng = np.random.default_rng(3)
    n = 40
    P = rng.normal(size=(n, 2)).astype(np.float32)
    data = Data(AnnDataLite(np.zeros((n, 3), np.float32)), train_size=25)
    data.data.obsp["g"] = SpotDistance(P)
    got = data.get_feature(split_name="train", return_type="numpy", channel="g", channel_type="obsp")
    idx = data.get_split_idx("train")
    assert isinstance(got, SpotDistance) and got.shape == (len(idx), len(idx))
    assert np.array_equal(got.toarray(), _dense(P).cpu().numpy()[idx][:, idx])


@pytest.mark.parametrize("n", [1, 2, 129, 1536, 5000])
@pytest.mark.parametrize("d", [2, 3])
def test_weight_total_matches_dense(cuda, n, d):
    from dance_b200 import ops, spatial_ops
    rng = np.random.default_rng(n * 10 + d)
    P = rng.uniform(0, 100, size=(n, d)).astype(np.float32)
    Pt = torch.as_tensor(P).cuda()
    D = ops.pairwise_l2_dense(Pt)
    for l in (1e-3, 0.5, 5.0, 1e4):    # from "the diagonal only" to "every weight ≈ 1"
        want = ops.exp_adj(D, l, want_matrix=False, want_sum=True)[1].item()
        got = spatial_ops.spatial_exp_adj_sum(Pt, Pt, l).item()
        assert abs(got - want) <= 1e-12 * abs(want), (l, got, want)


def test_search_l_same_on_both_forms(cuda):
    from dance_b200.matrix import SpotDistance
    from dance_b200.modules.spagcn import calculate_p, search_l
    rng = np.random.default_rng(5)
    P = rng.uniform(0, 400, size=(1536, 2)).astype(np.float32)
    D = _dense(P)
    m = SpotDistance(P)
    assert search_l(0.5, m) == search_l(0.5, D)
    assert abs(calculate_p(m, 37.0) - calculate_p(D, 37.0)) <= 1e-12 * (abs(calculate_p(D, 37.0)) + 1)


def _check_ax(rows, cols, l, X, worst):
    from dance_b200 import ops, spatial_ops
    Rt, Ct, Xt = (torch.as_tensor(a).cuda() for a in (rows, cols, X))
    AX = spatial_ops.spatial_exp_adj_matmul(Rt, Ct, l, Xt).double()
    W = _weights64(rows, cols, l)
    ref = W @ Xt.double()
    scale = W @ Xt.double().abs()
    err = (AX - ref).abs()
    # a floor of 2⁻¹⁴⁹ (the smallest subnormal) per column's |x|: products of subnormal weights may be flushed by the tensor core
    bound = scale * 2.0**-21 + Xt.double().abs().sum(0, keepdim=True) * 2.0**-149
    ratio = float((err / bound).max())
    worst[0] = max(worst[0], ratio)
    assert ratio < 4.0, ratio
    return AX


@pytest.mark.parametrize("n", [1, 7, 64, 128, 129, 1000, 4099])
@pytest.mark.parametrize("F", [1, 8, 50, 64, 130])
def test_ax_against_float64(cuda, n, F):
    rng = np.random.default_rng(n * 1000 + F)
    P = rng.uniform(0, 50, size=(n, 3)).astype(np.float32)
    X = rng.normal(size=(n, F)).astype(np.float32)
    worst = [0.0]
    _check_ax(P, P, 4.0, X, worst)
    # rectangular: a row subset against a different column set
    C = rng.uniform(0, 50, size=(n + 37, 3)).astype(np.float32)
    Xc = rng.normal(size=(n + 37, F)).astype(np.float32)
    _check_ax(P[: max(1, n // 2)], C, 6.0, Xc, worst)
    print(f"n={n} F={F}: largest |AX - fp64| / (2^-21 W|X|) = {worst[0]:.3f}")


def test_ax_edge_cases(cuda):
    rng = np.random.default_rng(11)
    worst = [0.0]
    # duplicate spots: d = 0 and weight exactly 1
    P = np.repeat(rng.uniform(0, 10, size=(150, 2)).astype(np.float32), 3, axis=0)
    X = rng.normal(size=(450, 50)).astype(np.float32)
    _check_ax(P, P, 1.0, X, worst)
    # pixel-scale coordinates
    P = rng.uniform(0, 2e4, size=(1200, 2)).astype(np.float32)
    X = rng.normal(size=(1200, 64)).astype(np.float32)
    _check_ax(P, P, 300.0, X, worst)
    # l so small that most weights underflow to zero or to subnormals
    P = rng.uniform(0, 40, size=(700, 2)).astype(np.float32)
    X = rng.normal(size=(700, 16)).astype(np.float32)
    for l in (0.05, 0.15):
        _check_ax(P, P, l, X, worst)
    print(f"edge cases: largest |AX - fp64| / (2^-21 W|X|) = {worst[0]:.3f}")


def test_ax_matches_dense_tf32x3_gemm(cuda):
    from dance_b200 import ops, spatial_ops
    from dance_b200.matrix import SpotDistance
    rng = np.random.default_rng(2)
    n = 3000
    P = rng.uniform(0, 300, size=(n, 2)).astype(np.float32)
    X = torch.as_tensor(rng.normal(size=(n, 50)).astype(np.float32)).cuda()
    m = SpotDistance(P).exp(20.0)
    dense = ops.gemm(m.to_device(), X, precision="tf32x3")
    coords = spatial_ops.spatial_exp_adj_matmul(*m.device_coords(), 20.0, X)
    scale = m.to_device().double() @ X.double().abs()
    assert float(((coords.double() - dense.double()).abs() / scale).max()) < 2.0**-18


def test_ax_full_size_sampled_rows(cuda):
    """200 k spots (the BASELINE configuration-5 size): 64 sampled rows of AX against an fp64 sum over all columns."""
    from dance_b200 import ops, spatial_ops
    n, F = 200_000, 50
    g = torch.Generator(device="cuda").manual_seed(0)
    P = torch.rand((n, 2), generator=g, device="cuda") * 20_000
    X = torch.randn((n, F), generator=g, device="cuda")
    l = 150.0
    AX = spatial_ops.spatial_exp_adj_matmul(P, P, l, X)
    rows = torch.randperm(n, device="cuda", generator=g)[:64]
    ref = torch.zeros((64, F), dtype=torch.float64, device="cuda")
    scale = torch.zeros_like(ref)
    for c0 in range(0, n, 8192):     # the fp32 weights of the dense path, a block of columns at a time
        D = ops.pairwise_l2_dense(torch.cat([P[rows], P[c0:c0 + 8192]]))[:64, 64:].contiguous()
        W = ops.exp_adj(D, l)[0].double()
        ref += W @ X[c0:c0 + 8192].double()
        scale += W @ X[c0:c0 + 8192].double().abs()
    ratio = float(((AX[rows].double() - ref).abs() / (scale * 2.0**-21)).max())
    print(f"200k: largest |AX - fp64| / (2^-21 W|X|) = {ratio:.3f}")
    assert ratio < 8.0


def _planted(n=1536, h=48, K=5, seed=21):
    rng = np.random.default_rng(seed)
    xy = rng.uniform(0, 400, size=(n, 2)).astype(np.float32)
    dom = np.minimum((xy[:, 0] // 80).astype(int), K - 1)
    X = (rng.normal(scale=2.0, size=(K, h))[dom] + rng.normal(size=(n, h))).astype(np.float32)
    return xy, dom, X


def test_spagcn_fit_predict_on_coordinates(cuda):
    from dance_b200.matrix import SpotDistance
    from dance_b200.modules.spagcn import SpaGCN
    xy, dom, X = _planted()
    D, m = _dense(xy).cpu().numpy(), SpotDistance(xy)
    runs = []
    for adj in (D, m):
        model = SpaGCN(device=cuda, seed=0)
        model.set_l(model.search_l(0.5, adj))
        pred = model.fit_predict((X, adj), lr=0.005, epochs=20, opt="admin", init="kmeans", n_clusters=5, tol=-1.0, init_labels=dom)
        runs.append((model, pred, model.predict_proba((X, adj))))
    (md, pd_, qd), (mc, pc, qc) = runs
    assert md.l == mc.l
    rel = lambda a, b: float((a - b).abs().max() / b.abs().max())
    assert rel(mc.model.params.p["gc.weight"], md.model.params.p["gc.weight"]) < 1e-4
    assert rel(qc, qd) < 1e-4
    assert (pc == pd_).mean() > 0.999


def test_spagcn_louvain_search_set_res_on_coordinates(cuda):
    from sklearn.metrics import adjusted_rand_score
    from dance_b200.matrix import SpotDistance
    from dance_b200.modules.spagcn import SpaGCN
    xy, dom, X = _planted(seed=4)
    m = SpotDistance(xy)
    model = SpaGCN(device=cuda, seed=0)
    l = model.search_l(0.5, m)
    res = model.search_set_res((X, m), l, target_num=5, start=0.4, step=0.1, tol=5e-3, lr=0.05, epochs=10, max_run=10)
    clf = SpaGCN(l, device=cuda, seed=0)
    pred = clf.fit_predict((X, m), init_spa=True, init="louvain", res=res, tol=5e-3, lr=0.05, epochs=200)
    assert adjusted_rand_score(dom, pred) > 0.8


def _hex_grid(r, c):
    pts = [(j + 0.5 * (i % 2), i * np.sqrt(3) / 2) for i in range(r) for j in range(c)]
    return np.array(pts, dtype=np.float32) * 100


def _pair_l2_np(P):
    """numpy restatement of pair_l2: fp32 differences and squares, fp64 sum in coordinate order; returns (sum, fp32 distance)."""
    diff = P[:, None, :] - P[None, :, :]
    sq = diff * diff
    s = np.zeros(sq.shape[:2])
    for c in range(P.shape[1]):
        s = s + sq[..., c].astype(np.float64)
    return s, np.sqrt(s).astype(np.float32)


def _spaced_grid(side=40, seed=0):
    """Spots 10⁴ pixels apart with integer jitter of up to 3: the near neighbours of a spot have distinct squared distances
    that round to the same fp32 distance (the fp32 spacing there is 2⁻¹⁰, the distances differ by ~10⁻⁴)."""
    rng = np.random.default_rng(seed)
    g = np.stack(np.meshgrid(np.arange(side), np.arange(side)), -1).reshape(-1, 2) * 10_000
    return (g + rng.integers(-3, 4, size=g.shape) + 50_000).astype(np.float32)


def _rank_by_sum_differs(s, D32, m):
    """Rows whose first m columns by (fp32 distance, index) differ from those by (fp64 squared sum, index): there a kernel
    ranking by the sum would return other spots.  Each such row holds a pair with equal fp32 distance whose higher index has
    the smaller sum."""
    by_d = np.argsort(D32, axis=1, kind="stable")[:, :m]
    by_s = np.argsort(s, axis=1, kind="stable")[:, :m]
    return np.nonzero((by_d != by_s).any(1))[0]


def _set_differs(s, D32, m):
    by_d = np.sort(np.argsort(D32, axis=1, kind="stable")[:, :m], 1)
    by_s = np.sort(np.argsort(s, axis=1, kind="stable")[:, :m], 1)
    return np.nonzero((by_d != by_s).any(1))[0]


def test_spaced_grid_has_fp32_collisions_in_the_top_ranks(cuda):
    P = _spaced_grid()
    s, D32 = _pair_l2_np(P)
    assert np.array_equal(D32, _dense(P).cpu().numpy())       # the restatement is the dense kernel's bits
    for m in (1, 5, 7, 8):
        rows = _rank_by_sum_differs(s, D32, m)
        if m > 1:
            assert len(rows) > 0, m
            i = rows[0]
            by_d = np.argsort(D32[i], kind="stable")[:m]
            assert any(D32[i, j] == D32[i, k] and s[i, j] > s[i, k] for a, j in enumerate(by_d) for k in by_d[a + 1:])
    assert len(_set_differs(s, D32, 7)) > 0 and len(_set_differs(s, D32, 5)) > 0


@pytest.mark.parametrize("shape", ["hexagon", "square"])
def test_refine_matches_dense(cuda, shape):
    from dance_b200.matrix import SpotDistance
    from dance_b200.modules.spagcn import refine
    rng = np.random.default_rng(9)
    grids = [_hex_grid(30, 40),                                                                       # exact ties
             _spaced_grid(),                                                                          # fp32 collisions
             np.round(rng.uniform(0, 2e4, size=(3000, 2))).astype(np.float32),                         # pixel scale
             (np.stack(np.meshgrid(np.arange(50), np.arange(50)), -1).reshape(-1, 2) * 137 + 9000).astype(np.float32)]
    for P in grids:
        n = P.shape[0]
        pred = rng.integers(0, 3, n)
        D = _dense(P).cpu().numpy()
        ids = [f"s{i}" for i in range(n)]
        assert refine(ids, pred, SpotDistance(P), shape=shape) == refine(ids, pred, D, shape=shape)


def test_nearest_matches_stable_sort(cuda):
    from dance_b200 import ops, spatial_ops
    rng = np.random.default_rng(1)
    for P in (_hex_grid(20, 20), _spaced_grid(), np.round(rng.uniform(0, 3e4, size=(2000, 2))).astype(np.float32)):
        Pt = torch.as_tensor(P).cuda()
        D = ops.pairwise_l2_dense(Pt)
        for m in (1, 5, 7, 8):
            want = torch.sort(D, dim=1, stable=True).indices[:, :m].int()
            assert torch.equal(spatial_ops.spatial_nearest(Pt, Pt, m), want)


def test_nearest_and_refine_with_nan_coordinates(cuda):
    """NaN distances rank after every number, ties by index, as torch.sort(stable=True) orders them: every index returned is
    a real column, and refine agrees with the dense refine (a uniform histology image makes SpaGCNGraph's z NaN everywhere)."""
    from dance_b200 import ops, spatial_ops
    from dance_b200.data import AnnDataLite, Data
    from dance_b200.matrix import SpotDistance
    from dance_b200.modules.spagcn import refine
    from dance_b200.transforms import SpaGCNGraph
    rng = np.random.default_rng(12)
    some = rng.uniform(0, 100, size=(300, 3)).astype(np.float32)
    some[rng.random(300) < 0.3, 2] = np.nan
    every = some.copy()
    every[:, 2] = np.nan
    for P in (some, every):
        Pt = torch.as_tensor(P).cuda()
        D = ops.pairwise_l2_dense(Pt)
        for m in (1, 7, 8):
            want = torch.sort(D, dim=1, stable=True).indices[:, :m].int()
            assert torch.equal(spatial_ops.spatial_nearest(Pt, Pt, m), want)
        pred = rng.integers(0, 3, P.shape[0])
        ids = list(range(P.shape[0]))
        assert refine(ids, pred, SpotDistance(P)) == refine(ids, pred, D.cpu().numpy())
    n = 120
    xy = rng.integers(0, 40, size=(n, 2))
    ad = AnnDataLite(np.zeros((n, 4), np.float32), obsm={"spatial": xy, "spatial_pixel": xy * 5 + 30},
                     uns={"image": np.full((300, 300, 3), 128, np.uint8)})
    data = Data(ad)
    with np.errstate(invalid="ignore"):                          # the colour variances are all zero
        SpaGCNGraph(alpha=1, beta=49, dense=False)(data)
    m = data.data.obsp["SpaGCNGraph"]
    assert np.isnan(m.rows[:, 2]).all()
    pred = rng.integers(0, 3, n)
    assert refine(list(range(n)), pred, m) == refine(list(range(n)), pred, m.toarray())


def test_spot_distance_owns_its_coordinates(cuda):
    from dance_b200.matrix import SpotDistance
    from dance_b200.modules.spagcn import SimpleGCDEC
    rng = np.random.default_rng(13)
    P = rng.uniform(0, 50, size=(200, 2)).astype(np.float32)
    m = SpotDistance(P)
    before = m.toarray()
    P[:] = 0                                                     # the caller's array is not the object's
    assert np.array_equal(m.toarray(), before)
    with pytest.raises(ValueError):
        m.rows[0, 0] = 1.0                                       # and the object's cannot be edited in place
    assert m.device_coords("cuda")[0] is m.device_coords(torch.device("cuda", torch.cuda.current_device()))[0]
    X = rng.normal(size=(200, 8)).astype(np.float32)
    model = SimpleGCDEC(8, 8, device="cuda:0", seed=0)
    model.bind(X, m.exp(5.0))
    assert model.AX.device == torch.device("cuda", 0)


@pytest.fixture
def spatial_env(tmp_path, monkeypatch):
    monkeypatch.setenv("DANCE_B200_SYNTH", "cells=1200,genes=400,types=5,density=0.5")
    monkeypatch.chdir(tmp_path)
    import sys
    from dance_b200 import dropin
    assert set(dropin.install()) == {"dance", "scanpy"}
    yield tmp_path
    for k in [k for k in sys.modules if k == "dance" or k.startswith("dance.") or k == "scanpy" or k.startswith("scanpy.")]:
        del sys.modules[k]


def _example_flow(dense):
    """examples/spatial/spatial_domain/spagcn.py:31-65 at its defaults (p 0.05, tol 5e-3, max_run 200, epochs 200, lr 0.05,
    seed 100, one run), restated line by line; ``dense`` goes to the pipeline and n_clusters is the synthetic data's 5."""
    from dance.datasets.spatial import SpatialLIBDDataset
    from dance.modules.spatial.spatial_domain.spagcn import SpaGCN, refine
    from dance.utils import set_seed
    set_seed(100)
    model = SpaGCN(device="cuda")
    preprocessing_pipeline = model.preprocessing_pipeline(alpha=1, beta=49, dense=dense)
    dataloader = SpatialLIBDDataset(data_id="151673")
    data = dataloader.load_data(transform=preprocessing_pipeline, cache=False)
    (x, adj, adj_2d), y = data.get_train_data()
    l = model.search_l(0.05, adj, start=0.01, end=1000, tol=5e-3, max_run=200)
    model.set_l(l)
    res = model.search_set_res((x, adj), l=l, target_num=5, start=0.4, step=0.1, tol=5e-3, lr=0.05, epochs=200, max_run=200)
    pred = model.fit_predict((x, adj), init_spa=True, init="louvain", tol=5e-3, lr=0.05, epochs=200, res=res)
    score = model.default_score_func(y, pred)
    refined_pred = refine(sample_id=data.data.obs_names.tolist(), pred=pred.tolist(), dis=adj_2d, shape="hexagon")
    score_refined = model.default_score_func(y, refined_pred)
    return adj, adj_2d, l, res, pred, refined_pred, score, score_refined


def test_example_flow_on_coordinates(cuda, spatial_env):
    from sklearn.metrics import adjusted_rand_score
    from dance_b200.matrix import SpotDistance
    dense = _example_flow(True)
    coords = _example_flow(False)
    assert isinstance(dense[0], np.ndarray) and isinstance(coords[0], SpotDistance) and isinstance(coords[1], SpotDistance)
    assert np.array_equal(coords[0].toarray(), dense[0]) and np.array_equal(coords[1].toarray(), dense[1])
    assert coords[2] == dense[2] and coords[3] == dense[3]                # the same l and resolution
    agree, agree_refined = adjusted_rand_score(dense[4], coords[4]), adjusted_rand_score(dense[5], coords[5])
    print(f"example flow: ARI dense {dense[6]:.4f} / {dense[7]:.4f} refined, coordinates {coords[6]:.4f} / {coords[7]:.4f}; "
          f"dense vs coordinates {agree:.4f} / {agree_refined:.4f}")
    assert agree > 0.95 and agree_refined > 0.95
