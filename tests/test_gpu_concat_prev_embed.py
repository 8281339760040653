"""feature_AE_concat_prev_embed / graph_AE_concat_prev_embed and the device normalizer on the GPU: ``ops.quantiles`` and
``ops.concat_normalized`` bit for bit against numpy / the float32 restatement, the handlers against the reference's own recorded
inputs (tests/golden/scgnn_concat_prev_embed.npz), one widened Feature-AE epoch against the oracle, and ScGNN2.fit end to end.

Bit patterns are compared after adding +0.0 (see tests/test_normalizer_cpu.py): −0.0 and +0.0 are one value to numpy's partition."""
import argparse

import numpy as np
import pytest
import torch

import normalizer_ref as nr
from conftest import rel_err

pytestmark = pytest.mark.gpu
f32 = np.float32
QS = (0.0, 0.1, 0.5, 0.9, 1.0)


def bits(a):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a
    return (np.asarray(a, dtype=np.float32) + f32(0)).view(np.uint32)


def _padded(host, pitch, dev):
    """host [r, c] as a row-padded device view with the given pitch (NaN in the padding, which must never be read)."""
    r, c = host.shape
    buf = torch.full((r, pitch), float("nan"), dtype=torch.float32, device=dev)
    buf[:, :c] = torch.from_numpy(host).to(dev)
    return buf[:, :c]


def _data(rng, rows, cols):
    x = rng.standard_normal((rows, cols)).astype(np.float32)
    x[rng.random((rows, cols)) < 0.3] = 0.0                                  # ties at zero, some of them −0.0
    x[rng.random((rows, cols)) < 0.05] = -0.0
    x[rng.random((rows, cols)) < 0.1] = f32(1.5)                            # more ties
    return x


@pytest.mark.parametrize("rows,cols,pitch", [(1, 1, 1), (1, 2, 2), (2, 1, 4), (3, 3, 3), (7, 1, 1), (13, 7, 8), (101, 10, 12),
                                             (1000, 33, 33), (1000, 33, 36), (257, 128, 128), (4097, 16, 20)])
def test_quantiles_match_numpy(cuda, rows, cols, pitch):
    from dance_b200 import ops
    host = _data(np.random.default_rng(rows * 1000 + cols), rows, cols)
    got = ops.quantiles(_padded(host, pitch, cuda), QS)
    want = np.array([np.quantile(host, q) for q in QS], dtype=np.float32)
    assert np.array_equal(bits(got), bits(want)), (got, want)


@pytest.mark.parametrize("pitch", [60, 64])
def test_quantiles_above_2_24_values(cuda, pitch):
    from dance_b200 import ops
    rows, cols = (1 << 24) // 60 + 7, 60
    host = np.random.default_rng(pitch).standard_normal((rows, cols)).astype(np.float32)
    host[::3, ::7] = 0.0
    got = ops.quantiles(_padded(host, pitch, cuda), QS)
    want = np.array([np.quantile(host, q) for q in QS], dtype=np.float32)
    assert np.array_equal(bits(got), bits(want)), (got, want)


def test_quantiles_above_2_31_values(cuda):
    """2.2·10⁹ values built on the device from x = ((i·7919 + 12345) mod 1009) − 504 over the flat index i: value class r is hit
    by the indices i ≡ j_r (mod 1009), so every order statistic, and with it np.quantile's result, is known in closed form."""
    from dance_b200 import ops
    M, A, B = 1009, 7919, 12345
    rows, cols = 1_100_000, 2000
    n = rows * cols
    assert n > 2**31
    x = torch.empty((rows, cols), dtype=torch.float32, device=cuda)
    step = 50_000
    for r0 in range(0, rows, step):
        r1 = min(rows, r0 + step)
        i = torch.arange(r0 * cols, r1 * cols, dtype=torch.int64, device=cuda)
        x[r0:r1] = (((i * A + B) % M) - 504).to(torch.float32).view(r1 - r0, cols)
        del i
    inv = pow(A, -1, M)
    counts = np.array([(n - 1 - ((v - B) * inv % M)) // M + 1 for v in range(M)], dtype=np.int64)   # class v ↔ value v − 504
    cum = np.cumsum(counts)

    def order_stat(k):
        return f32(int(np.searchsorted(cum, k, side="right")) - 504)

    got = ops.quantiles(x, QS)
    for q, g in zip(QS, got):
        prev, nxt, t = nr.plan(n, q)
        assert bits(g) == bits(nr.lerp(order_stat(prev), order_stat(nxt), t)), q
    del x
    torch.cuda.empty_cache()


def test_quantiles_reject_non_finite(cuda):
    from dance_b200 import ops
    x = torch.randn(100, 8, device=cuda)
    x[17, 3] = float("inf")
    with pytest.raises(ValueError, match="non-finite"):
        ops.quantiles(x, [0.5])
    x[17, 3] = float("nan")
    with pytest.raises(ValueError, match="non-finite"):
        ops.quantiles(x, [0.5])


def _concat_cases():
    rng = np.random.default_rng(77)
    big = np.maximum(rng.standard_normal((3000, 128)) * 2, 0).astype(np.float32)
    ge = rng.standard_normal((3000, 16)).astype(np.float32)
    yield "graph_embed_on_embedding", big, ge, big, 128
    expr = np.log1p(np.where(rng.random((500, 70)) < 0.75, 0, rng.gamma(2.0, 1.0, (500, 70)))).astype(np.float32)
    yield "graph_embed_on_expression", expr, ge[:500], expr, 72
    sparse = np.where(rng.random((500, 70)) < 0.95, f32(0), expr)           # q0.1 == q0.9: falls back to (min, max)
    yield "fallback_range", sparse, ge[:500], sparse, 70
    near = ge[:500].copy()
    near[:, 3] = f32(0.25)                                                  # constant column: scale 1
    yield "constant_column", expr, near, expr, 80
    yield "feature_embed_on_graph_embed", ge, big, ge, 16
    yield "unscaled", expr, big[:500], None, 70


@pytest.mark.parametrize("name,left,right,base,pitch", list(_concat_cases()), ids=[c[0] for c in _concat_cases()])
def test_concat_normalized_matches_restatement(cuda, name, left, right, base, pitch):
    from dance_b200 import ops
    L = _padded(left, pitch, cuda)
    R = torch.from_numpy(right).to(cuda)
    B = None if base is None else (L if base is left else torch.from_numpy(base).to(cuda))
    out = ops.concat_normalized(L, R, base=B)
    a, e = left.shape[1], right.shape[1]
    assert tuple(out.shape) == (left.shape[0], a + e) and out.stride(0) % 4 == 0 and out.stride(0) >= a + e
    assert np.array_equal(bits(out), bits(nr.concat_normalized(left, right, base)))
    full = out.as_strided((out.shape[0], out.stride(0)), (out.stride(0), 1))
    assert torch.all(full[:, a + e:] == 0)                                   # padding columns are zero


def test_concat_normalized_errors(cuda):
    from dance_b200 import ops
    left = torch.full((50, 8), 2.0, device=cuda)
    right = torch.randn(50, 4, device=cuda)
    with pytest.raises(ValueError, match="Minimum of desired feature range must be smaller than maximum"):
        ops.concat_normalized(left, right, base=left)
    base = torch.randn(50, 8, device=cuda)
    base[3, 3] = float("inf")
    with pytest.raises(ValueError, match="non-finite"):
        ops.concat_normalized(left, right, base=base)
    right[0, 0] = float("nan")
    with pytest.raises(ValueError, match="non-finite"):
        ops.concat_normalized(left, right, base=torch.randn(50, 8, device=cuda))


# ---- handlers against the reference's recorded inputs ------------------------------------------------------------------------
def _args(**over):
    d = dict(total_epoch=0, feature_AE_epoch=[1, 1], feature_AE_batch_size=64, feature_AE_learning_rate=1e-3, feature_AE_regu_strength=0.9,
             feature_AE_dropout_prob=0, feature_AE_concat_prev_embed=None, graph_AE_epoch=1, graph_AE_use_GAT=False, graph_AE_GAT_dropout=0,
             graph_AE_learning_rate=1e-2, graph_AE_embedding_size=16, graph_AE_concat_prev_embed=False, graph_AE_normalize_embed=None,
             graph_AE_neighborhood_factor=0.05, graph_AE_retain_weights=False, gat_multi_heads=2, gat_hid_embed=64)
    d.update(over)
    return argparse.Namespace(**d)


@pytest.mark.parametrize("mode", ["graph", "feature"])
def test_feature_ae_handler_matches_reference_contract(cuda, golden, monkeypatch, mode):
    from dance_b200 import ops
    from dance_b200.engine import FeatureAEEngine
    from dance_b200.modules import scgnn2
    g = golden("scgnn_concat_prev_embed")
    seen = {}
    concat = ops.concat_normalized

    def spy_concat(*a, **k):
        seen["X"] = concat(*a, **k)
        return seen["X"]

    load = FeatureAEEngine.load_state_dict

    def spy_load(self, sd):
        seen["loaded"] = sd
        return load(self, sd)

    monkeypatch.setattr(ops, "concat_normalized", spy_concat)
    monkeypatch.setattr(FeatureAEEngine, "load_state_dict", spy_load)
    X = g["X"]
    state = None
    for e in (0, 1, 2):
        seen.clear()
        param = {"device": cuda, "epoch_num": e, "total_epoch": 2, "n_feature_orig": X.shape[1], "seed": 3,
                 "graph_embed": g["graph_embed"], "feature_embed": g["feature_embed"]}
        emb, recon, ckpt = scgnn2.feature_AE_handler(X, None, _args(feature_AE_concat_prev_embed=mode), param, state)
        key = f"fae.{mode}.e{e}"
        want = g[key + ".X"]
        got = seen.get("X", X)
        assert np.array_equal(bits(got), bits(want)), key
        assert param["_feature_AE_engine"].dim == int(g[key + ".dim"])
        assert sorted(ckpt) == sorted(g[key + ".keys"].tolist())
        loaded = str(g[key + ".loaded"])
        sd = seen.get("loaded")
        assert loaded == ("none" if sd is None else ("model_concat" if sd is (state or {}).get("model_concat") else "model")), key
        assert emb.shape == (X.shape[0], 128) and recon.shape == X.shape and np.isfinite(recon).all()
        if e >= 1:
            assert ckpt["model"] is state["model"] and ckpt["optimizer"] is state["optimizer"]
            assert ckpt["model_concat"]["fc1.weight"].shape == (512, int(g[key + ".dim"]))
        state = ckpt


@pytest.mark.parametrize("branch", ["gcn", "gat"])
def test_graph_ae_handler_widened_knn_is_exact(cuda, golden, monkeypatch, branch):
    from dance_b200.modules import scgnn2
    g = golden("scgnn_concat_prev_embed")
    seen = {}
    build = scgnn2.build_knn_graph

    def spy(xe, *a, **k):
        seen["X"] = xe
        out = build(xe, *a, **k)
        seen["knn"] = out[1]
        return out

    monkeypatch.setattr(scgnn2, "build_knn_graph", spy)
    for e in (0, 1):
        seen.clear()
        param = {"device": cuda, "epoch_num": e, "seed": 0, "graph_embed": g["graph_embed"]}
        embed, _, _, _ = scgnn2.graph_AE_handler(g["x_embed"], None, _args(graph_AE_use_GAT=branch == "gat",
                                                                             graph_AE_concat_prev_embed=True), param)
        key = f"gae.{branch}.e{e}"
        assert np.array_equal(bits(seen["X"]), bits(g[key + ".X"])), key
        assert seen["X"].shape[1] == int(g[key + ".dim"])
        assert np.array_equal(seen["knn"].cpu().numpy(), g[key + ".knn"]), key
        if branch == "gcn":
            assert param["_graph_AE_engine"].dim == int(g[key + ".dim"])
        assert embed.shape == (g["x_embed"].shape[0], 16) and np.isfinite(embed).all()


def test_graph_cache_is_keyed_by_width(cuda, golden):
    from dance_b200.modules import scgnn2
    g = golden("scgnn_concat_prev_embed")
    cache = {}
    args = _args(graph_AE_concat_prev_embed=True)
    scgnn2.graph_AE_handler(g["x_embed"], None, args, {"device": cuda, "epoch_num": 0, "seed": 0, "graph_cache": cache})
    assert cache["d"] == 128
    _, _, (edges, _), _ = scgnn2.graph_AE_handler(g["x_embed"], None, args, {"device": cuda, "epoch_num": 1, "seed": 0,
                                                                             "graph_embed": g["graph_embed"], "graph_cache": cache})
    assert cache["d"] == 144
    assert np.array_equal(edges[:, 1].reshape(-1, 10), g["gae.gcn.e1.knn"])


def test_widened_feature_ae_epoch_matches_oracle(cuda, golden):
    from dance_b200.engine import FeatureAEEngine
    from dance_b200.modules.scgnn2 import feature_AE_handler
    from oracle import port
    g = golden("scgnn_concat_prev_embed")
    X, Xw = g["X"], g["fae.graph.e1.X"]
    param = {"device": cuda, "epoch_num": 1, "total_epoch": 1, "n_feature_orig": X.shape[1], "seed": 5,
             "graph_embed": g["graph_embed"]}
    emb, recon, ckpt = feature_AE_handler(X, None, _args(feature_AE_concat_prev_embed="graph"), param, {"model": {}, "optimizer": {}})
    dim = Xw.shape[1]
    init = FeatureAEEngine(dim, device=cuda, seed=5).state_dict()             # epoch 1: a fresh model, same seed
    ref = port.FeatureAE(dim)
    ref.load_state_dict({k: v.cpu() for k, v in init.items()})
    opt = torch.optim.Adam(ref.parameters(), lr=1e-3)
    _, z_ref, r_ref = port.feature_ae_epoch(ref, opt, torch.from_numpy(Xw), 64, "noregu", 0.9)
    assert rel_err(emb, z_ref.numpy()) < 1e-4 and rel_err(recon, r_ref.numpy()[:, :X.shape[1]]) < 1e-4
    for k, v in ckpt["model_concat"].items():
        assert rel_err(v.cpu().numpy(), ref.state_dict()[k].numpy()) < 1e-4, k


def test_unrecognised_feature_concat_value_raises(cuda, golden):
    from dance_b200.modules.scgnn2 import feature_AE_handler
    g = golden("scgnn_concat_prev_embed")
    param = {"device": cuda, "epoch_num": 1, "total_epoch": 1, "n_feature_orig": 64, "graph_embed": g["graph_embed"]}
    with pytest.raises(ValueError, match="'graph' or 'feature'"):
        feature_AE_handler(g["X"], None, _args(feature_AE_concat_prev_embed="both"), param, {"model": {}, "optimizer": {}})


@pytest.mark.parametrize("over", [dict(feature_AE_concat_prev_embed="graph"), dict(feature_AE_concat_prev_embed="feature"),
                                  dict(graph_AE_concat_prev_embed=True), dict(clustering_embed="both"),
                                  dict(feature_AE_concat_prev_embed="graph", graph_AE_concat_prev_embed=True, graph_AE_use_GAT=True)],
                         ids=["feature_graph", "feature_feature", "graph", "clustering_both", "all_gat"])
def test_scgnn2_fit_two_em_iterations(cuda, over):
    from dance_b200.modules.scgnn2 import ScGNN2
    from oracle import port
    X = port.synthetic_expression(256, 48, density=0.3, seed=1)
    kw = dict(total_epoch=2, feature_AE_epoch=[2, 1], graph_AE_epoch=2, graph_AE_neighborhood_factor=10, clustering_louvain_only=False,
              clustering_embed="graph", clustering_method="KMeans", seed=0, cluster_AE_batch_size=12800, cluster_AE_epoch=1,
              cluster_AE_learning_rate=1e-3, cluster_AE_regu_strength=0.9, cluster_AE_dropout_prob=0)
    kw.update(over)
    model = ScGNN2(_args(**kw), device="cuda", seed=0)
    model.fit(X)
    out = model.predict()
    assert out.shape == X.shape and np.isfinite(out).all()
    assert model.x_embed.shape == (256, 128) and model.graph_embed.shape == (256, 16) and np.isfinite(model.graph_embed).all()
    if "feature_AE_concat_prev_embed" in over:
        assert sorted(model.model_state) == ["model", "model_concat", "optimizer", "optimizer_concat"]
        assert model.model_state["model"]["fc1.weight"].shape == (512, 48)
