"""GATLayer's dropout (scgnn2.py:999-1031) and identity skip (scgnn2.py:1167-1171) on the GPU.

* the counter-based draw behind ``ops.dropout`` and the attention mask: values, keep rates, independence across keys, heads,
  rows and columns;
* the ``_drop`` aggregate kernels against fp64 autograd of the masked restatement (masks materialised with ``ops.dropout`` on
  the attention key), on tests/test_gpu_gat.py's graph (empty rows, in-degrees 1/31/32/33/64, a hub), both head paths and both
  softmax shifts; at p = 0 bit-identical to the plain entry points;
* the identity-skip combine kernels against an explicitly broadcast skip;
* ``GATEngine`` with dropout against tests/gat_dropout_ref.py run with the engine's own masks, with projected and identity skips;
* ``graph_AE_handler`` / ``ScGNN2.fit`` with ``graph_AE_GAT_dropout``.

Kernel tolerances start from tests/test_gpu_gat.py's (forward 2e-6 global / 5e-5 per row, gradients 5e-6 / 2e-4 per row) and
are tightened to about 10x the largest errors measured on an H100 80 GB HBM3 (700 W limit) at p = 0.5: forward 1.5e-7 global /
1.5e-6 per row, dH 1.6e-7 global / 3.5e-5 per row (that file's 2e-4 kept), da 3.2e-7.  The errors are printed with ``-s``
(lines ``ERR <name> <value>``).

da_src / da_trg and the global shift's gradient are sums of float atomics, whose order is not fixed: two identical backward
calls can differ in the last bits, so bit-identity is checked where the arithmetic is ordered and a 1e-6 bound elsewhere."""
import argparse

import numpy as np
import pytest
import torch

from conftest import rel_err
from test_gpu_gat import GRAD_FLOOR, GRAD_ROW, _graph, _indeg, _params, row_err

pytestmark = pytest.mark.gpu

SEED = 1234
FWD_REL, FWD_ROW, GRAD_REL = 1.5e-6, 1.5e-5, 3.5e-6


def _log(name, v):
    print(f"ERR {name} {v:.3e}")
    return v


# ---------------------------------------------------------------------------------------------------------- the draw
def test_dropout_values_and_repeatability(cuda):
    from dance_b200 import ops
    ones = torch.ones(1000, 777, device=cuda)
    for p in (0.1, 0.3, 0.5):
        a = ops.dropout(ones, p, SEED, 5)
        b = ops.dropout(ones, p, SEED, 5)
        assert torch.equal(a, b)
        vals = torch.unique(a)
        assert set(vals.tolist()) <= {0.0, float(torch.tensor(1 / (1 - p), dtype=torch.float32))}
        assert not torch.equal(a, ops.dropout(ones, p, SEED, 6)) and not torch.equal(a, ops.dropout(ones, p, SEED + 1, 5))
    # strided input, in place: the kept entries are scaled, the padding is untouched
    buf = torch.randn(300, 70, device=cuda)
    x = buf[:, :64]
    want = x * ops.dropout(torch.ones(300, 64, device=cuda), 0.3, SEED, 9)
    ops.dropout(x, 0.3, SEED, 9, out=x)
    assert torch.allclose(x, want, rtol=1e-7, atol=0)
    assert torch.equal(ops.dropout(ones, 0.0, SEED, 1), ones)
    assert torch.equal(ops.dropout(ones, 1.0, SEED, 1), torch.zeros_like(ones))
    for bad in (-0.1, 1.5, float("nan")):
        with pytest.raises(ValueError):
            ops.dropout(ones, bad, SEED, 1)


@pytest.mark.parametrize("p", [0.1, 0.3, 0.5, 0.9])
def test_dropout_keep_rate_and_independence(cuda, p):
    """≥ 10⁷ draws: the keep rate is within 6σ of 1 − p; pairs from different keys, heads (columns of an [E, NH] mask), adjacent
    rows and adjacent columns are kept together at rate (1 − p)² within 6σ."""
    from dance_b200 import ops
    R, C = 4096, 2560
    ones = torch.ones(R, C, device=cuda)
    k0 = ops.dropout(ones, p, SEED, 100) != 0
    k1 = ops.dropout(ones, p, SEED, 101) != 0
    q = 1 - p

    def within(x, mean, n):
        return abs(x - mean) <= 6 * np.sqrt(mean * (1 - mean) / n)

    assert within(k0.double().mean().item(), q, k0.numel())
    pairs = {"keys": (k0, k1), "rows": (k0[:-1], k0[1:]), "cols": (k0[:, :-1], k0[:, 1:])}
    heads = ops.dropout(torch.ones(R * C // 2, 2, device=cuda), p, SEED, 102) != 0      # an attention mask with 2 heads
    pairs["heads"] = (heads[:, 0], heads[:, 1])
    for name, (a, b) in pairs.items():
        assert within((a & b).double().mean().item(), q * q, a.numel()), name


# ---------------------------------------------------------------------------------------------------------- kernels
HEADS = [(1, 512), (2, 64), (4, 128), (2, 16), (3, 100), (32, 16)]      # wide-head path first, then narrow


def _masked_reference(H, a_src, a_trg, src, trg, nh, shift, M, dOut):
    """fp64 (out, α) of the aggregate with α' = α · M, and autograd (dH, da_src, da_trg) of <out, dOut>."""
    from oracle import gat_ref
    n = H.shape[0]
    leaves = [t.detach().double().requires_grad_() for t in (H, a_src, a_trg)]
    s_src, s_trg = gat_ref.scores(leaves[0], leaves[1], leaves[2], nh)
    e = gat_ref.score_act(s_src.index_select(0, src) + s_trg.index_select(0, trg), "leakyrelu", 0.2)
    alpha = gat_ref.edge_softmax(e, trg, n, shift)
    lifted = leaves[0].reshape(n, nh, -1).index_select(0, src) * (alpha * M.double()).unsqueeze(-1)
    out = torch.zeros((n, ) + lifted.shape[1:], dtype=torch.float64, device=H.device).index_add(0, trg, lifted).reshape(n, -1)
    grads = torch.autograd.grad((out * dOut.double()).sum(), leaves)
    return out.detach(), alpha.detach(), grads


@pytest.mark.parametrize("shift", ["global", "segment"])
@pytest.mark.parametrize("nh,F", HEADS)
def test_gat_aggregate_drop_matches_fp64(cuda, nh, F, shift):
    from dance_b200 import ops
    n, p, key = 3000, 0.5, 77
    T, Tt, perm, src, trg = _graph(n)
    _, H, a_src, a_trg = _params(n, nh, F, seed=nh * 1000 + F + 2)
    dOut = torch.randn(n, nh * F, device=cuda, generator=torch.Generator(device=cuda).manual_seed(F + 3))
    s_src, s_trg = ops.gat_scores(H, a_src, a_trg, nh)
    drop = dict(dropout=p, seed=SEED, key=key)
    out, alpha, gmax = ops.gat_aggregate_fwd(T, H, s_src, s_trg, nh, "leakyrelu", 0.2, shift, **drop)
    dH, da_src, da_trg = ops.gat_aggregate_bwd(T, Tt, perm, H, a_src, a_trg, s_src, s_trg, alpha, dOut, nh, "leakyrelu", 0.2,
                                               gmax=gmax if shift == "global" else None, **drop)
    M = ops.dropout(torch.ones(T.nnz, nh, device=cuda), p, SEED, key)               # the attention mask, scaled
    ref_out, ref_alpha, (g_H, g_as, g_at) = _masked_reference(H, a_src, a_trg, src, trg, nh, shift, M, dOut)
    tag = f"{nh}x{F}.{shift}"
    assert _log(f"fwd.{tag}", rel_err(out, ref_out.cpu())) < FWD_REL and _log(f"fwd_row.{tag}", row_err(out, ref_out)) < FWD_ROW
    assert rel_err(alpha, ref_alpha.cpu()) < FWD_REL and row_err(alpha, ref_alpha) < FWD_ROW     # α is stored undropped
    assert _log(f"dH.{tag}", rel_err(dH, g_H.cpu())) < GRAD_REL and _log(f"dH_row.{tag}", row_err(dH, g_H, GRAD_FLOOR)) < GRAD_ROW
    assert _log(f"da.{tag}", max(rel_err(da_src, g_as.cpu()), rel_err(da_trg, g_at.cpu()))) < GRAD_REL
    # targets all of whose in-edges are dropped for a head get exactly zero in that head
    kept = torch.zeros(n, nh, device=cuda).index_add_(0, trg, (M != 0).float())
    dead = (kept == 0) & (_indeg(T) > 0).unsqueeze(1)
    assert dead.any()
    assert (out.reshape(n, nh, F)[dead] == 0).all()


@pytest.mark.parametrize("shift", ["global", "segment"])
@pytest.mark.parametrize("nh,F", [(2, 64), (2, 16), (3, 100)])
def test_gat_aggregate_drop_at_zero_is_bit_identical(cuda, nh, F, shift):
    """p = 0 through the _drop entry points: out, α (and gmax of the global shift) bit for bit; dH bit for bit under the per-target
    shift (under the global one its argmax rows take the atomically summed shift gradient); da within 1e-6 (atomic sums)."""
    from dance_b200 import ops
    n = 3000
    T, Tt, perm, _, _ = _graph(n)
    _, H, a_src, a_trg = _params(n, nh, F, seed=5 * F + nh)
    dOut = torch.randn(n, nh * F, device=cuda, generator=torch.Generator(device=cuda).manual_seed(1))
    s_src, s_trg = ops.gat_scores(H, a_src, a_trg, nh)
    res = []
    for kw in ({}, dict(dropout=0.0, seed=SEED, key=3)):
        out, alpha, gmax = ops.gat_aggregate_fwd(T, H, s_src, s_trg, nh, "leakyrelu", 0.2, shift, **kw)
        gm = gmax if shift == "global" else None
        res.append((out, alpha, gmax) + ops.gat_aggregate_bwd(T, Tt, perm, H, a_src, a_trg, s_src, s_trg, alpha, dOut, nh, gmax=gm, **kw))
    (out0, al0, gm0, dH0, das0, dat0), (out1, al1, gm1, dH1, das1, dat1) = res
    assert torch.equal(out0, out1) and torch.equal(al0, al1)
    if shift == "segment":                      # gmax is not written under the per-target shift
        assert torch.equal(dH0, dH1)
    else:
        assert torch.equal(gm0, gm1) and rel_err(dH1, dH0.cpu()) < 1e-6
    assert rel_err(das1, das0.cpu()) < 1e-6 and rel_err(dat1, dat0.cpu()) < 1e-6


@pytest.mark.parametrize("concat,act", [(True, "elu"), (False, None)])
def test_gat_combine_identity_matches_broadcast_skip(cuda, concat, act):
    from dance_b200 import ops
    n, nh, F = 2000, 3, 40
    gen = torch.Generator(device=cuda).manual_seed(8)
    agg = torch.randn(n, nh * F, device=cuda, generator=gen)
    x = torch.randn(n, F + 4, device=cuda, generator=gen)[:, :F]
    bias = torch.randn(nh * F if concat else F, device=cuda, generator=gen)
    out = ops.gat_combine_fwd(agg, x, bias, nh, concat, act, identity=True)
    assert torch.equal(out, ops.gat_combine_fwd(agg, x.repeat(1, nh), bias, nh, concat, act))
    dout = torch.randn_like(out)
    dpre, dact, dx = ops.gat_combine_bwd(dout, out, nh, F, concat, act, identity=True)
    dpre0, dact0 = ops.gat_combine_bwd(dout, out, nh, F, concat, act)
    assert torch.equal(dpre, dpre0) and torch.equal(dact, dact0)
    want = torch.zeros(n, F, device=cuda)
    for h in range(nh):
        want = want + dpre0[:, h * F:(h + 1) * F]
    assert torch.equal(dx, want)


# ---------------------------------------------------------------------------------------------------------- engine
def _gat_graph(golden, cuda):
    """As tests/test_gpu_engine.py, plus the position in edge_index order (i → its k neighbours) of every target-CSR entry."""
    import scipy.sparse as sp
    from dance_b200 import ops
    g = golden("knn_graph")
    n, k = g["knn_idx"].shape
    src_csr = ops.CSR(torch.arange(0, n * k + 1, k, dtype=torch.int32, device=cuda),
                      torch.from_numpy(g["knn_idx"].reshape(-1).astype(np.int32)).to(cuda), None, (n, n))
    T, pos = ops.csr_transpose(src_csr)
    Tt, t_perm = ops.csr_transpose(T)
    adj = sp.csr_matrix((np.ones(len(g["adj_indices"])), g["adj_indices"], g["adj_indptr"]), shape=(n, n))
    L = (adj + sp.eye(n)).tocsr()
    L.sort_indices()
    edge_index = torch.from_numpy(np.stack([np.repeat(np.arange(n), k), g["knn_idx"].reshape(-1)]).astype(np.int64))
    return g, T, Tt, t_perm, ops.CSR.from_scipy(L, cuda, with_values=False), edge_index, pos.long().cpu(), torch.from_numpy(L.toarray())


def _engine_masks(eng, n, nnz, pos, step):
    """The engine's masks of training step ``step`` as tests/gat_dropout_ref.py takes them (attention in edge_index order)."""
    from dance_b200 import ops
    masks = []
    for l, L in enumerate(eng.layers):
        W = eng.nh * L["F"]
        mk = lambda rows, cols, site: ops.dropout(torch.ones(rows, cols, device=eng.device), eng.dropout, eng.drop_seed,
                                                  eng.drop_key(l, site, step)).double().cpu()
        attn_csr = mk(nnz, eng.nh, "attn")
        attn = torch.empty_like(attn_csr)
        attn[pos] = attn_csr
        masks.append({"input": mk(n, L["fin"], "input"), "proj": mk(n, W, "proj"), "attn": attn})
    return masks


CONFIGS = {"proj": (16, 64, 16), "ident": (16, 16, 32)}      # (dim, gat_hid_embed, embedding): ident has FIN == FOUT in both layers


@pytest.mark.parametrize("precision", ["fp32", "tf32x3"])
@pytest.mark.parametrize("tag", ["proj", "ident"])
def test_gat_engine_dropout_step_matches_restatement(cuda, golden, tag, precision):
    """One train_step with dropout 0.3 against tests/gat_dropout_ref.py in fp64 with the engine's own masks: embedding, loss,
    every gradient and the weights after Adam (1e-4 / 2e-4 rel, as test_gat_engine_matches_reference)."""
    from dance_b200.engine import GATEngine
    from gat_dropout_ref import graph_ae_gat_forward
    g, T, Tt, t_perm, Lc, edge_index, pos, labels = _gat_graph(golden, cuda)
    gg = golden("graph_ae_gat_dropout")
    x = torch.from_numpy(g["X"]).to(cuda)
    dim, hid, emb = CONFIGS[tag]
    eng = GATEngine(dim, hid, emb, 2, device=cuda, lr=1e-2, precision=precision, seed=SEED, dropout=0.3)
    assert [L["identity"] for L in eng.layers] == [tag == "ident"] * 2
    eng.load_state_dict({k[len(tag) + 6:]: gg[k] for k in gg.files if k.startswith(f"{tag}.init.")})
    sd0 = eng.state_dict()
    masks = _engine_masks(eng, x.shape[0], T.nnz, pos, step=0)
    z = eng.train_step(x, T, Tt, t_perm, Lc)
    assert eng.step == 1

    sd = {k: v.double().cpu().requires_grad_() for k, v in sd0.items()}
    z_ref = graph_ae_gat_forward(x.double().cpu(), edge_index, sd, masks)
    loss = torch.nn.functional.binary_cross_entropy_with_logits(z_ref @ z_ref.t(), labels.double())
    opt = torch.optim.Adam(sd.values(), lr=1e-2)
    opt.zero_grad()
    loss.backward()
    assert rel_err(z.cpu().numpy(), z_ref.detach().numpy()) < 1e-4
    assert abs(eng.loss.item() - loss.item()) < 1e-4 * loss.item()
    for k, gt in eng.grads().items():
        want = sd[k].grad
        if want is None:                                         # identity skip: skip_proj is never read
            assert tag == "ident" and "skip_proj" in k and (gt == 0).all(), k
            continue
        assert rel_err(gt.cpu().numpy().reshape(want.shape), want.numpy()) < 2e-4, k
    opt.step()
    for k, v in eng.state_dict().items():
        assert rel_err(v.cpu().numpy().reshape(sd[k].shape), sd[k].detach().numpy()) < 1e-4, k
    if tag == "ident":
        for _ in range(3):
            eng.train_step(x, T, Tt, t_perm, Lc)
        after = eng.state_dict()
        for l in range(2):
            k = f"gat.gat_net.{l}.skip_proj.weight"
            assert torch.equal(after[k], sd0[k]), k
            assert not torch.equal(after[f"gat.gat_net.{l}.linear_proj.weight"], sd0[f"gat.gat_net.{l}.linear_proj.weight"])


def test_gat_engine_steps_draw_new_masks(cuda, golden):
    g, T, Tt, t_perm, Lc, edge_index, pos, labels = _gat_graph(golden, cuda)
    from dance_b200.engine import GATEngine
    eng = GATEngine(16, 64, 16, 2, device=cuda, seed=SEED, dropout=0.3)
    keys = {(s, l, site) for s in range(2) for l in range(2) for site in GATEngine.SITES}
    assert len({eng.drop_key(l, site, s) for s, l, site in keys}) == len(keys)
    m0 = _engine_masks(eng, 300, T.nnz, pos, 0)
    m1 = _engine_masks(eng, 300, T.nnz, pos, 1)
    for l in range(2):
        for site in GATEngine.SITES:
            assert not torch.equal(m0[l][site], m1[l][site]), (l, site)
    # the embedding of a step is a dropped-out forward: with lr = 0 two steps still differ
    eng.lr = 0.0
    x = torch.from_numpy(g["X"]).to(cuda)
    z0 = eng.train_step(x, T, Tt, t_perm, Lc).clone()
    z1 = eng.train_step(x, T, Tt, t_perm, Lc).clone()
    assert not torch.equal(z0, z1) and torch.isfinite(z1).all()
    with pytest.raises(ValueError):
        GATEngine(16, 64, 16, 2, device=cuda, dropout=1.5)


# ---------------------------------------------------------------------------------------------------------- handler / module
def _args(**over):
    d = dict(total_epoch=0, feature_AE_epoch=[2, 1], feature_AE_batch_size=128, feature_AE_learning_rate=1e-3, feature_AE_regu_strength=0.9,
             feature_AE_dropout_prob=0, feature_AE_concat_prev_embed=None, graph_AE_epoch=3, graph_AE_use_GAT=True, graph_AE_GAT_dropout=0.5,
             graph_AE_learning_rate=1e-2, graph_AE_embedding_size=16, graph_AE_concat_prev_embed=False, graph_AE_normalize_embed=None,
             graph_AE_neighborhood_factor=10, graph_AE_retain_weights=False, gat_multi_heads=2, gat_hid_embed=64)
    d.update(over)
    return argparse.Namespace(**d)


def test_graph_ae_handler_gat_dropout(cuda):
    from dance_b200.modules.scgnn2 import graph_AE_handler
    from oracle import port
    X = port.synthetic_embedding(400, d=128, n_clusters=4, seed=8)
    run = lambda **over: graph_AE_handler(X, None, _args(**over), {"device": cuda, "epoch_num": 0, "seed": 3})[0]
    a, b = run(), run()
    assert np.isfinite(a).all() and rel_err(b, a) < 1e-4           # same seed → same masks (the float atomics of da are unordered)
    assert rel_err(run(graph_AE_GAT_dropout=0), a) > 1e-3
    # a hidden width equal to the input width: the identity skip in layer 0
    c = run(gat_hid_embed=128)
    assert c.shape == (400, 16) and np.isfinite(c).all()
    for bad in (-0.1, 1.5):
        with pytest.raises(ValueError):
            run(graph_AE_GAT_dropout=bad)


def test_scgnn2_fit_gat_dropout_em(cuda):
    from dance_b200.modules.scgnn2 import ScGNN2
    from oracle import port
    X = port.synthetic_expression(256, 48, density=0.3, seed=1)
    em = ScGNN2(_args(total_epoch=1, clustering_louvain_only=False, clustering_embed="graph", clustering_method="KMeans", seed=0,
                      cluster_AE_batch_size=12800, cluster_AE_epoch=2, cluster_AE_learning_rate=1e-3, cluster_AE_regu_strength=0.9,
                      cluster_AE_dropout_prob=0, graph_AE_GAT_dropout=0.3), device="cuda", seed=0)
    em.fit(X)
    assert em.predict().shape == X.shape and np.isfinite(em.predict()).all() and len(em.cluster_labels) == 256
