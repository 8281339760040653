"""graph-sc on the device: the new kernels against float64, GraphSC.fit against the reference's own fit (tests/golden/graphsc_fit.npz,
made by tests/make_golden_graphsc.py), predict against sklearn, and the engine's host-synchronisation and launch-count claims.

The float64 side is tests/graphsc_ref.py, whose restatement is pinned to the reference by tests/test_graphsc_step_ref_cpu.py."""
import numpy as np
import pytest
import torch

import graphsc_ref as R
from conftest import rel_err

pytestmark = pytest.mark.gpu

SEED = 3


def _mask(shape, p, key, dev):
    """The device's scaled keep mask (keep / (1 − p)) over a [rows, cols] grid, float64."""
    from dance_b200 import ops
    return ops.dropout(torch.ones(shape, device=dev), p, SEED, key).double().cpu()


# ---- fused decoder -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 2, 127, 128, 129, 500])
@pytest.mark.parametrize("d", [1, 50, 200, 300, 1024])
def test_batch_decoder_vs_float64(cuda, B, d):
    from dance_b200 import ops
    g = torch.Generator().manual_seed(B * 7 + d)
    z = torch.randn(B, d, generator=g) * (2.0 / d**0.5)
    key = 11
    loss, dz = ops.graphsc_batch_decoder(z.to(cuda), 0.1, SEED, key)
    m = _mask((B, d), 0.1, key, cuda)
    zd = z.double().requires_grad_(True)
    zt = zd * m
    ref = R.batch_loss(zt @ zt.t())
    ref.backward()
    if B == 1:                                  # pos_weight 0: the loss and its gradient vanish
        assert loss.item() == 0.0 and torch.count_nonzero(dz).item() == 0
        return
    assert abs(loss.item() - ref.item()) <= 1e-5 * abs(ref.item())
    assert rel_err(dz, zd.grad) <= 1e-5


def test_batch_decoder_refuses_wide_embeddings(cuda):
    from dance_b200 import ops
    from dance_b200._lib import B2Error
    with pytest.raises(B2Error, match=r"\[1, 1024\]"):
        ops.graphsc_batch_decoder(torch.zeros(4, 1025, device=cuda))


# ---- block degrees and aggregate -----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def block_graph(cuda):
    from dance_b200.ops import CSR
    gd = R.synthetic_graph(300, 100, 24, seed=5)
    cs = R.csr_by_destination(gd)
    A = CSR(torch.from_numpy(cs["indptr"]).int().to(cuda), torch.from_numpy(cs["indices"]).int().to(cuda),
            torch.from_numpy(cs["weights"]).float().to(cuda), (cs["n_nodes"], cs["n_nodes"]))
    batch = np.random.default_rng(1).choice(300, 64, replace=False) + 100
    return cs, A, batch


def _row_err(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return (np.linalg.norm(a - b, axis=1) / np.maximum(np.linalg.norm(b, axis=1), 1e-30)).max()


@pytest.mark.parametrize("agg", ["sum", "mean"])
@pytest.mark.parametrize("p", [0.0, 0.3])
def test_block_aggregate_vs_float64(cuda, block_graph, agg, p):
    from dance_b200 import ops
    cs, A, batch = block_graph
    n, F = cs["n_nodes"], 24
    x = torch.from_numpy(np.random.default_rng(2).standard_normal((n, F)))
    x32 = x.float().to(cuda)
    # layer 2 of a two-layer block: destinations = the batch; its sources = layer 1's destinations
    dst2 = torch.from_numpy(batch).int().to(cuda)
    cap = int((cs["indptr"][batch + 1] - cs["indptr"][batch]).sum())
    deg2, src, pos = ops.graphsc_block_degrees(A, dst2, src_cap=cap)
    assert np.array_equal(deg2.cpu().numpy(), R.block_outdeg(cs["indptr"], cs["indices"], batch, n))
    src_h = src.cpu().numpy()
    nsrc = int((src_h >= 0).sum())
    assert (src_h[nsrc:] == -1).all()
    u, _, _ = R.block_edges(cs["indptr"], cs["indices"], None, batch)
    assert np.array_equal(np.sort(src_h[:nsrc]), np.unique(u))
    assert np.array_equal(pos.cpu().numpy()[src_h[:nsrc]], np.arange(nsrc))
    # layer 1: destinations = the (padded) source list
    deg1 = ops.graphsc_block_degrees(A, src)
    assert np.array_equal(deg1.cpu().numpy(), R.block_outdeg(cs["indptr"], cs["indices"], src_h[:nsrc], n))
    m1 = _mask((n, F), p, 5, cuda) if p else None
    out1 = ops.graphsc_block_aggregate(A, src, deg1, x32, agg, p, SEED, 5)
    ref1 = R.block_aggregate(cs["indptr"], cs["indices"], cs["weights"], src_h[:nsrc], x, n, agg, m1)
    assert _row_err(out1[:nsrc].cpu(), ref1) <= 1e-6
    assert torch.count_nonzero(out1[nsrc:]).item() == 0
    # layer 2 reads layer 1's rows through src_pos
    h1 = torch.from_numpy(np.random.default_rng(3).standard_normal((cap, F)))
    m2 = _mask((n, F), p, 6, cuda) if p else None
    out2 = ops.graphsc_block_aggregate(A, dst2, deg2, h1.float().to(cuda), agg, p, SEED, 6, x_pos=pos)
    h1_global = torch.zeros(n, F, dtype=torch.float64)
    h1_global[torch.from_numpy(src_h[:nsrc]).long()] = h1[:nsrc]
    ref2 = R.block_aggregate(cs["indptr"], cs["indices"], cs["weights"], batch, h1_global, n, agg, m2)
    assert _row_err(out2.cpu(), ref2) <= 1e-6
    # the adjoint of layer 2, into layer 1's rows
    dout = torch.from_numpy(np.random.default_rng(4).standard_normal((batch.size, F)))
    dx = ops.graphsc_block_aggregate(A, dst2, deg2, dout.float().to(cuda), agg, p, SEED, 6, x_pos=pos, transposed=True, out_rows=cap)
    xg = h1_global.clone().requires_grad_(True)
    (R.block_aggregate(cs["indptr"], cs["indices"], cs["weights"], batch, xg, n, agg, m2) * dout).sum().backward()
    assert _row_err(dx[:nsrc].cpu(), xg.grad[torch.from_numpy(src_h[:nsrc]).long()]) <= 1e-6
    assert torch.count_nonzero(dx[nsrc:]).item() == 0


# ---- GraphSC.fit against the reference ---------------------------------------------------------------------------------------
def _graph(gold=None):
    """The fixture's graph as a GraphLite (regenerated; checked against the fixture's checksum)."""
    from dance_b200.graph import GraphLite
    gd = R.fixture_graph()
    if gold is not None:
        assert np.allclose(R.graph_checksum(gd), gold["graph_checksum"], rtol=1e-12, atol=0), "the fixture graph did not regenerate"
    g = GraphLite(torch.from_numpy(gd["src"]).long(), torch.from_numpy(gd["dst"]).long(), gd["n_nodes"])
    g.edata["weight"] = torch.from_numpy(gd["weight"]).float()
    G = gd["n_genes"]
    g.ndata["features"] = torch.from_numpy(gd["features"]).float()
    g.ndata["feat_id"] = torch.cat([-torch.ones(G, dtype=torch.int32), torch.arange(gd["n_nodes"] - G, dtype=torch.int32)])
    return g


def _cfg(gold, tag):
    cfg = {}
    for k in gold.files:
        if k.startswith(f"{tag}.cfg."):
            v = gold[k]
            cfg[k[len(tag) + 5:]] = v.item() if v.dtype.kind != "U" else str(v)
    return cfg


def _fit_recorded(cfg, init, fit_seed, epochs, lr, batch_size, drop_seed, g, cuda):
    """GraphSC(**cfg).fit from the state ``init``, recording every epoch's batch order and per-batch losses."""
    from dance_b200.modules.graphsc import GraphSC
    m = GraphSC(**cfg, device=cuda, drop_seed=drop_seed)
    m.model.load_state_dict(init)
    orders, losses = [], []
    epoch = m.model.train_epoch

    def recorded(*a, **k):
        out = epoch(*a, **k)
        orders.append(m.model.last_order.numpy())
        losses.append(out.cpu().numpy())
        return out

    m.model.train_epoch = recorded
    torch.manual_seed(fit_seed)
    m.fit(g, epochs=epochs, lr=lr, batch_size=batch_size)
    return m, np.concatenate(orders), np.concatenate(losses)


def _fit(gold, tag, cuda):
    cfg = _cfg(gold, tag)
    return _fit_recorded(cfg, R.init_state(cfg, int(gold[f"{tag}.init_seed"])), int(gold[f"{tag}.fit_seed"]), int(gold[f"{tag}.epochs"]),
                         float(gold["lr"]), int(gold[f"{tag}.batch_size"]), int(gold["drop_seed"]), _graph(gold), cuda)


# (per-batch loss, final embedding and weights) relative.  "base" is GraphSC()'s defaults with narrower widths.  "deep" stacks BatchNorm
# over 16 columns, gelu and a short 18-row batch: Adam's steps (close to lr · sign(g)) follow the sign of gradient entries that
# float32 rounding decides, so float32 and float64 part by up to lr per step there and the loss follows them; its weights are
# held to that lr-per-step bound (None) instead of a relative one.
TOL = {"base": (1e-5, 1e-4, 1e-4), "deep": (2e-4, 1e-3, None)}


@pytest.mark.parametrize("tag", ["base", "deep"])
def test_fit_matches_reference(cuda, golden, tag):
    gold = golden("graphsc_fit")
    tol_loss, tol_z, tol_w = TOL[tag]
    m, order, losses = _fit(gold, tag, cuda)
    assert np.array_equal(order, gold[f"{tag}.order"])
    ref_losses = gold[f"{tag}.losses"]
    assert losses.shape == ref_losses.shape
    assert (np.abs(losses - ref_losses) <= tol_loss * np.abs(ref_losses)).all(), np.abs(losses / ref_losses - 1).max()
    assert rel_err(m.get_latent(), gold[f"{tag}.z"]) <= tol_z, rel_err(m.get_latent(), gold[f"{tag}.z"])
    sd = m.model.state_dict()
    final = {k[len(tag) + 7:]: gold[k] for k in gold.files if k.startswith(f"{tag}.final.")}
    assert set(sd) == set(final)
    # A bias in front of a BatchNorm has an exact gradient of 0, so Adam steps it by rounding noise (of order lr once that noise
    # exceeds eps); it changes no output, only the running mean that tracks it.  Those are held to lr-sized bounds.
    pre_bn = {k for k in sd if k.startswith("encoder.") and k.endswith(".bias") and f"encoder.{int(k.split('.')[1]) + 1}.running_mean" in sd}
    tracked = {f"encoder.{int(k.split('.')[1]) + 1}.running_mean" for k in pre_bn}
    n_steps = len(ref_losses)
    for k, v in sd.items():
        if k.endswith("num_batches_tracked"):
            assert int(v) == int(final[k]) == 2 * n_steps
        elif k in pre_bn or k in tracked or tol_w is None:
            assert np.abs(v.cpu().numpy() - final[k]).max() <= 2 * float(gold["lr"]) * n_steps, k
        else:
            assert rel_err(v, final[k]) <= tol_w, (k, rel_err(v, final[k]))


def test_fit_at_default_widths_matches_float64(cuda):
    """GraphSC() exactly as constructed by default (50 → 200 → 300) on the fixture's graph, one epoch at lr 1e-3, against the
    float64 restatement (pinned to the reference's fit by tests/test_graphsc_step_ref_cpu.py) on the batches the module drew."""
    cfg = dict(agg="sum", activation="relu", in_feats=50, n_hidden=1, hidden_dim=200, hidden_1=300, hidden_2=0, dropout=0.1,
               n_layers=1, hidden_relu=False, hidden_bn=False)
    init = R.init_state(cfg, 30)
    lr, bs = 1e-3, 128
    m, order, losses = _fit_recorded(cfg, init, 31, 1, lr, bs, 0, _graph(), cuda)
    graph = R.csr_by_destination(R.fixture_graph())
    G = graph["n_genes"]
    assert np.array_equal(np.sort(order), np.arange(G, graph["n_nodes"]))
    batches = [order[i:i + bs] for i in range(0, order.size, bs)]
    ref_losses, z, sd = R.fit(init, dict(cfg, stride=1), graph, batches, None, lr, R.device_masks(0, cfg["dropout"]))
    assert (np.abs(losses - ref_losses) <= 1e-5 * np.abs(ref_losses)).all(), np.abs(losses / ref_losses - 1).max()
    assert rel_err(m.get_latent(), z) <= 1e-4
    for k, v in m.model.state_dict().items():
        assert rel_err(v, sd[k]) <= 1e-4, (k, rel_err(v, sd[k]))


def test_predict_partitions_as_sklearn(cuda, golden):
    from sklearn.cluster import KMeans
    from sklearn.metrics import adjusted_rand_score

    from dance_b200.modules.graphsc import GraphSC
    gold = golden("graphsc_fit")
    z = gold["base.z"]
    m = GraphSC(n_clusters=8, device=cuda)
    m.z = z
    pred = m.predict()
    ref = KMeans(n_clusters=8, init="k-means++", random_state=5, n_init=10).fit_predict(z)
    assert adjusted_rand_score(ref, pred) == 1.0


# ---- engine: no host synchronisation, fixed launches per batch -----------------------------------------------------------------
LAUNCHES_PER_BATCH = 17       # GraphSCEngine's default configuration, as DESIGN.md §4 counts them


@pytest.mark.parametrize("n_cells,batch", [(300, 64), (700, 128)])
def test_train_epoch_is_sync_free_with_fixed_launches(cuda, n_cells, batch):
    from dance_b200 import ops
    from dance_b200.engine import GraphSCEngine, prepare_graph
    gold_like = R.synthetic_graph(n_cells, 120, 50, seed=n_cells)
    from dance_b200.graph import GraphLite
    g = GraphLite(torch.from_numpy(gold_like["src"]), torch.from_numpy(gold_like["dst"]), gold_like["n_nodes"])
    g.edata["weight"] = torch.from_numpy(gold_like["weight"]).float()
    g.ndata["features"] = torch.from_numpy(gold_like["features"]).float()
    g.ndata["feat_id"] = torch.cat([-torch.ones(120, dtype=torch.int32), torch.arange(n_cells, dtype=torch.int32)])
    graph = prepare_graph(g, cuda)
    eng = GraphSCEngine(device=cuda)
    eng.train_epoch(graph, graph["train_ids"], batch, 1e-3)          # warm-up: buffers, GEMM set-up
    torch.cuda.synchronize()
    nb = (n_cells + batch - 1) // batch
    ops.reset_counters()
    torch.cuda.set_sync_debug_mode("error")
    try:
        losses = eng.train_epoch(graph, graph["train_ids"], batch, 1e-3)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert ops.counters()["launches"] == nb * LAUNCHES_PER_BATCH
    assert losses.is_cuda and losses.shape == (nb, ) and bool(torch.isfinite(losses).all())


# ---- interface ---------------------------------------------------------------------------------------------------------------
def test_state_dict_round_trips_reference_keys(cuda, golden):
    from dance_b200.engine import GraphSCEngine
    gold = golden("graphsc_fit")
    for tag in ("base", "deep"):
        cfg = _cfg(gold, tag)
        init = {k[len(tag) + 7:]: gold[k] for k in gold.files if k.startswith(f"{tag}.final.")}      # the reference's keys
        eng = GraphSCEngine(**cfg, device=cuda)
        sd = eng.state_dict()
        assert {k: tuple(v.shape) for k, v in sd.items()} == {k: tuple(v.shape) for k, v in init.items()}
        eng.load_state_dict({k: torch.from_numpy(v) for k, v in init.items()})
        for k, v in eng.state_dict().items():
            assert np.array_equal(v.cpu().numpy(), init[k]), k


def test_reference_errors(cuda):
    from dance_b200.modules.graphsc import GraphSC
    g = _graph()
    with pytest.raises(TypeError):
        GraphSC(activation="prelu", device=cuda).fit(g, epochs=1)
    with pytest.raises(ValueError, match="hidden_2"):
        GraphSC(n_hidden=2, device=cuda)
    m = GraphSC(hidden_bn=True, device=cuda)
    torch.manual_seed(0)
    with pytest.raises(ValueError, match="more than 1 value per channel"):
        m.fit(g, epochs=1, batch_size=599)                          # 600 cells: the last batch has one


def test_dropin_import():
    from dance_b200 import dropin
    dropin.install()
    from dance.modules.single_modality.clustering.graphsc import GraphSC

    from dance_b200.modules.graphsc import GraphSC as Native
    assert GraphSC is Native
