"""graph-sc's device code against float64 where the fit tests cannot see it.

GraphSC.fit (tests/test_gpu_graphsc.py) observes the engine only after Adam, whose step is close to lr · sign(g) and blind to the
scale of each gradient.  Here GraphSCEngine.train_batch runs one batch with Adam replaced by a no-op, and its loss, its recorded
embedding, every parameter gradient and the BatchNorm running statistics are compared with float64 autograd through
tests/graphsc_ref.py (pinned to the reference's own fit by tests/test_graphsc_step_ref_cpu.py) across the layer configurations.
Then each kernel graph-sc runs is compared with a float64 restatement at its width, layout and degree edges: the block
degrees and aggregate (hub rows, empty rows, padding, both feature slots and slices, strided operands), the fused batch decoder
(many CTAs, padded leading dimensions, saturated logits), act / act_bwd for every code, and scatter_rows."""
import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

import graphsc_ref as R
from conftest import rel_err

pytestmark = pytest.mark.gpu

SEED = 3
SENTINEL = -7.25          # fills the columns around strided operands; a kernel that writes past its width overwrites it


def _strided(rows, cols, dev, left=3, right=5, fill=SENTINEL):
    """An [rows, cols] view into a [rows, left + cols + right] buffer filled with ``fill``: (buffer, view)."""
    buf = torch.full((rows, left + cols + right), fill, dtype=torch.float32, device=dev)
    return buf, buf[:, left:left + cols]


def _margins_intact(buf, cols, left=3):
    b = buf.cpu()
    return bool((b[:, :left] == SENTINEL).all()) and bool((b[:, left + cols:] == SENTINEL).all())


def _graphlite(gd):
    from dance_b200.graph import GraphLite
    g = GraphLite(torch.from_numpy(gd["src"]).long(), torch.from_numpy(gd["dst"]).long(), gd["n_nodes"])
    g.edata["weight"] = torch.from_numpy(gd["weight"]).float()
    g.ndata["features"] = torch.from_numpy(gd["features"]).float()
    n_cells = gd["n_nodes"] - gd["n_genes"]
    g.ndata["feat_id"] = torch.cat([-torch.ones(gd["n_genes"], dtype=torch.int32), torch.arange(n_cells, dtype=torch.int32)])
    return g


# ================================================================================================================================
# 1. GraphSCEngine: one batch's loss, embedding, gradients and running statistics against float64 autograd
# ================================================================================================================================
HIDDEN = {                                     # the hidden Linear stack behind the graph convolutions
    "none": dict(n_hidden=0),
    "linear": dict(n_hidden=1, hidden_1=48),
    "relu": dict(n_hidden=1, hidden_1=64, hidden_relu=True),
    "bn_relu2": dict(n_hidden=2, hidden_1=96, hidden_2=40, hidden_bn=True, hidden_relu=True),
    "bn": dict(n_hidden=1, hidden_1=36, hidden_bn=True),
}

# Every pair of values of any two columns appears in some row.  in_feats and hidden_dim cross the aggregate's 32-feature slots
# and 128-feature slices; B = 1 and 2 run without BatchNorm (a one-row batch raises, and over two rows BatchNorm's output is
# ±γ + β whatever its input, so every gradient in front of it is rounding noise); the ragged batches end mid-tile in the
# decoder (8 rows per CTA) and mid-warp in the aggregate.
#        agg     activation    layers hidden     dropout precision in_feats hidden_dim  B
CASES = [
    ("sum", "relu", 1, "none", 0.3, None, 129, 32, 1),
    ("sum", "relu", 1, "linear", 0.0, None, 1, 32, 37),
    ("sum", "relu", 1, "relu", 0.3, None, 33, 128, 2),
    ("sum", "relu", 2, "bn_relu2", 0.0, "fp32", 1, 200, 129),
    ("sum", "relu", 2, "bn", 0.0, "fp32", 129, 200, 37),
    ("sum", "leaky_relu", 1, "bn_relu2", 0.0, None, 33, 257, 129),
    ("sum", "leaky_relu", 2, "bn", 0.3, "fp32", 1, 128, 37),
    ("sum", "leaky_relu", 2, "relu", 0.3, "fp32", 129, 257, 129),
    ("sum", "gelu", 1, "linear", 0.3, "fp32", 300, 257, 2),
    ("sum", "gelu", 2, "relu", 0.0, None, 1, 257, 1),
    ("sum", "gelu", 2, "none", 0.3, "fp32", 1, 128, 2),
    ("mean", "relu", 1, "bn", 0.0, "fp32", 300, 32, 129),
    ("mean", "relu", 2, "linear", 0.0, "fp32", 33, 200, 1),
    ("mean", "relu", 2, "none", 0.3, None, 300, 257, 1),
    ("mean", "leaky_relu", 1, "bn_relu2", 0.0, None, 300, 128, 37),
    ("mean", "leaky_relu", 2, "relu", 0.3, "fp32", 300, 200, 2),
    ("mean", "leaky_relu", 2, "linear", 0.0, None, 129, 128, 1),
    ("mean", "leaky_relu", 2, "none", 0.0, "fp32", 33, 32, 2),
    ("mean", "gelu", 1, "bn", 0.0, None, 33, 257, 129),
    ("mean", "gelu", 1, "bn_relu2", 0.3, "fp32", 129, 32, 37),
    ("mean", "gelu", 1, "none", 0.0, None, 1, 200, 37),
    ("mean", "gelu", 2, "relu", 0.0, None, 129, 32, 2),
]
N_CELLS, N_GENES = 200, 80


def _case_id(c):
    agg, act, nl, hid, p, prec, fin, hd, B = c
    return f"{agg}-{act}-L{nl}-{hid}-p{p}-{prec or 'tf32x3'}-in{fin}-h{hd}-B{B}"


def engine_errors(cuda, case):
    """One GraphSCEngine.train_batch (Adam a no-op) against R.forward / R.batch_loss in float64 at step 0.  Returns
    {name: (error, bound)}: the loss, the embedding, every gradient tensor and the running statistics relative; a bias in front
    of a BatchNorm, whose exact gradient is 0, absolutely over its layer's weight gradient norm; for B = 1 the largest |value|
    of the loss and of every gradient, which must be exactly 0."""
    from dance_b200.engine import GraphSCEngine, prepare_graph
    agg, act, n_layers, hidden, p, precision, in_feats, hidden_dim, B = case
    cfg = dict(agg=agg, activation=act, in_feats=in_feats, hidden_dim=hidden_dim, dropout=p, n_layers=n_layers, hidden_1=0,
               hidden_2=0, hidden_relu=False, hidden_bn=False)
    cfg.update(HIDDEN[hidden])
    seed = sum(map(ord, _case_id(case))) % 997
    gd = R.synthetic_graph(N_CELLS, N_GENES, in_feats, seed=seed)
    gd["weight"] = gd["weight"].astype(np.float32).astype(np.float64)          # the values the device sees
    gd["features"] = gd["features"].astype(np.float32).astype(np.float64)
    graph, host = prepare_graph(_graphlite(gd), cuda), R.csr_by_destination(gd)
    ids = np.random.default_rng(seed).choice(N_CELLS, B, replace=False) + N_GENES
    init = R.init_state(cfg, seed)

    eng = GraphSCEngine(**cfg, device=cuda, drop_seed=SEED, precision=precision)
    eng.load_state_dict(init)
    eng.params.adam_step = lambda lr: None         # the gradients stay as the backward left them
    eng.z = torch.full((N_CELLS, eng.emb_dim), SENTINEL, device=cuda)
    loss = torch.empty(1, device=cuda)
    ids_t = torch.from_numpy(ids)
    eng.train_batch(eng.block(graph, ids_t, ids_t.to(torch.int32).to(cuda)), 1e-3, loss)
    sd = eng.state_dict()

    params = {k: v.clone().requires_grad_(True) for k, v in init.items() if not R._is_buffer(k)}
    bn_state = {k: v.clone() for k, v in init.items() if R._is_buffer(k)}
    c64, masks = dict(cfg, stride=eng.stride), R.device_masks(SEED, p)
    _, emb = R.forward(params, c64, host, ids, masks, 0, 0, bn_state)
    logits, _ = R.forward(params, c64, host, ids, masks, 0, 1, bn_state)
    ref = R.batch_loss(logits)
    ref.backward()

    z = eng.z.cpu()
    rows = torch.from_numpy(ids - N_GENES)
    others = torch.ones(N_CELLS, dtype=torch.bool)
    others[rows] = False
    assert bool((z[others] == SENTINEL).all()), "scatter_rows wrote a cell outside the batch"
    err = {"z": (rel_err(z[rows], emb.detach()), TOL)}
    if B == 1:                                     # pos_weight is 0: the loss and every gradient vanish exactly
        err["loss"] = (abs(loss.item()), 0.0)
        err.update({f"grad {k}": (float(eng.params.g[k].abs().max()), 0.0) for k in eng.params.names})
        return err
    err["loss"] = (abs(loss.item() - ref.item()) / abs(ref.item()), TOL)
    pre_bn = {li + ".bias": li + ".weight" for li, bn in eng.lin if bn}
    for k in eng.params.names:
        g = eng.params.g[k]
        if k in pre_bn:
            wnorm = float(params[pre_bn[k]].grad.norm())
            assert float(params[k].grad.abs().max()) <= 1e-12 * wnorm
            err[f"grad {k}"] = (float(g.norm()) / wnorm, TOL_PRE_BN)
        else:
            err[f"grad {k}"] = (rel_err(g, params[k].grad), PINNED.get((_case_id(case), f"grad {k}"), TOL))
    for k, v in bn_state.items():
        if k.endswith("num_batches_tracked"):
            assert int(sd[k]) == int(v) == 2, k
        else:
            err[k] = (rel_err(sd[k], v), TOL)
    return err


# Measured on an H100 SXM (80 GB, 700 W): without BatchNorm every tensor is within 7e-7, with it within 6e-6, bar one pin.
# In front of a BatchNorm the gradient is projected off the batch mean and the normalised input, so whatever sums it over rows
# cancels: float32 rounding of the terms, relative ~1e-7, grows by ‖Σ|terms|‖ / ‖Σ terms‖.  That ratio is 113 for the pinned
# layer bias (measured 1.6e-5) and 28 for the 6e-6 of the two-layer BatchNorm stack (float64, per-row bias gradients).  A bias
# right in front of a BatchNorm has an exact gradient of 0; its float32 sum of B rows keeps rounding noise, measured up to
# 3.5e-6 of its layer's weight gradient norm at B = 129.
TOL, TOL_PRE_BN = 1e-5, 1e-5
PINNED = {("mean-gelu-L1-bn-p0.0-tf32x3-in33-h257-B129", "grad layer1.bias"): 3e-5}


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_engine_batch_gradients_vs_float64(cuda, case):
    bad = {k: e for k, (e, bound) in engine_errors(cuda, case).items() if not e <= bound}
    assert not bad, bad


# ================================================================================================================================
# 2. The kernels at their edges
# ================================================================================================================================
@pytest.fixture(scope="module")
def edge_graph(cuda):
    """A destination-indexed CSR of 2400 nodes with rows of 1..8 in-edges, 40 rows without any, and one hub row of 2100
    in-edges (a warp's lanes stride it 66 times); weights in [0.25, 2).  ``dst``: 190 distinct destinations including the hub and
    six empty rows, with −1 padding at the start, in the middle and at the end."""
    from dance_b200.ops import CSR
    rng = np.random.default_rng(11)
    n, hub = 2400, 7
    deg = rng.integers(1, 9, n)
    empty = rng.choice(np.arange(hub + 1, n), 40, replace=False)
    deg[empty], deg[hub] = 0, 2100
    indices = np.concatenate([rng.choice(n, d, replace=False) for d in deg]).astype(np.int64)
    indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    weights = rng.uniform(0.25, 2.0, indices.size).astype(np.float32).astype(np.float64)
    plain = np.setdiff1d(np.arange(n), np.concatenate([empty, [hub]]))
    valid = rng.permutation(np.concatenate([rng.choice(plain, 183, replace=False), [hub], empty[:6]]))
    dst = np.concatenate([[-1], valid[:95], [-1, -1], valid[95:], [-1]])
    dev = lambda a, t: torch.from_numpy(a).to(t).to(cuda)
    A_w = CSR(dev(indptr, torch.int32), dev(indices, torch.int32), dev(weights, torch.float32), (n, n))
    A_1 = CSR(A_w.rowptr, A_w.colidx, None, (n, n))
    return dict(indptr=indptr, indices=indices, weights=weights, n=n, hub=hub, empty=empty, dst=dst, valid=dst[dst >= 0],
                dst_dev=dev(dst, torch.int32), A={True: A_w, False: A_1})


def test_block_degrees_edges(cuda, edge_graph):
    from dance_b200 import ops
    g = edge_graph
    A, n = g["A"][True], g["n"]
    u, _, _ = R.block_edges(g["indptr"], g["indices"], None, g["valid"])
    uniq = np.unique(u)
    ref = R.block_outdeg(g["indptr"], g["indices"], g["valid"], n)
    assert np.array_equal(ops.graphsc_block_degrees(A, g["dst_dev"]).cpu().numpy(), ref)
    # src_cap exactly the number of sources: every slot filled, a permutation of the sources, src_pos its inverse
    deg, src, pos = ops.graphsc_block_degrees(A, g["dst_dev"], src_cap=uniq.size)
    src, pos = src.cpu().numpy(), pos.cpu().numpy()
    assert np.array_equal(deg.cpu().numpy(), ref)
    assert np.array_equal(np.sort(src), uniq)
    assert np.array_equal(pos[src], np.arange(uniq.size))
    # a larger cap (Σ row lengths, the engine's): the tail is −1
    cap = int((g["indptr"][g["valid"] + 1] - g["indptr"][g["valid"]]).sum())
    _, src, pos = ops.graphsc_block_degrees(A, g["dst_dev"], src_cap=cap)
    src, pos = src.cpu().numpy(), pos.cpu().numpy()
    assert np.array_equal(np.sort(src[:uniq.size]), uniq) and (src[uniq.size:] == -1).all()
    assert np.array_equal(pos[src[:uniq.size]], np.arange(uniq.size))
    # the hub alone: 2100 distinct sources, each counted once
    hub = torch.tensor([g["hub"]], dtype=torch.int32, device=cuda)
    deg = ops.graphsc_block_degrees(A, hub).cpu().numpy()
    assert deg.sum() == 2100 and np.array_equal(np.nonzero(deg)[0], np.unique(g["indices"][g["indptr"][g["hub"]]:g["indptr"][g["hub"] + 1]]))
    # no destinations, or padding only: all-zero degrees and an all −1 source list
    for dst in (torch.empty(0, dtype=torch.int32, device=cuda), torch.full((5, ), -1, dtype=torch.int32, device=cuda)):
        deg = torch.full((n, ), 9, dtype=torch.int32, device=cuda)
        _, src, _ = ops.graphsc_block_degrees(A, dst, outdeg=deg, src_cap=7)
        assert torch.count_nonzero(deg).item() == 0 and (src.cpu() == -1).all()


def _agg64(g, weighted, dst, x, agg, mask):
    """R.block_aggregate and the same sum over |terms| (every coefficient is positive): (value, scale)."""
    w = g["weights"] if weighted else None
    val = R.block_aggregate(g["indptr"], g["indices"], w, dst, x, g["n"], agg, mask)
    return val, R.block_aggregate(g["indptr"], g["indices"], w, dst, x.abs(), g["n"], agg, mask)


def _agg64_T(g, weighted, dst, dout, agg, mask):
    """The adjoint of _agg64 by autograd, into [n, F] global rows: (value, scale)."""
    out = []
    for d in (dout, dout.abs()):
        x = torch.zeros(g["n"], d.shape[1], dtype=torch.float64, requires_grad=True)
        w = g["weights"] if weighted else None
        (R.block_aggregate(g["indptr"], g["indices"], w, dst, x, g["n"], agg, mask) * d).sum().backward()
        out.append(x.grad)
    return out


def _rows_within(dev_rows, ref, scale, tol):
    """Every row within tol · ‖its sum of |terms|‖ (norm-wise); rows whose terms are all 0 exactly 0."""
    d = np.asarray(dev_rows, np.float64) - np.asarray(ref, np.float64)
    lim = tol * np.linalg.norm(np.asarray(scale, np.float64), axis=1)
    bad = np.linalg.norm(d, axis=1) > lim
    return not bad.any(), (np.linalg.norm(d, axis=1) / np.maximum(lim / tol, 1e-30)).max()


@pytest.mark.parametrize("F", [1, 31, 32, 33, 127, 128, 129, 300, 513])
@pytest.mark.parametrize("agg", ["sum", "mean"])
@pytest.mark.parametrize("p", [0.0, 0.5])
@pytest.mark.parametrize("weighted", [True, False], ids=["weighted", "unweighted"])
def test_block_aggregate_edges(cuda, edge_graph, F, agg, p, weighted):
    """Forward and transposed, global rows and x_pos rows, on strided operands, against float64; the dropout mask is keyed by
    (global node id, global feature index), so a slice other than the first, or a lane slot other than 0, that keyed its
    features locally would differ."""
    from dance_b200 import ops
    g = edge_graph
    A, n, valid, dst_dev = g["A"][weighted], g["n"], g["valid"], g["dst_dev"]
    key = 21 + F
    mask = R.keep_mask(SEED, key, torch.arange(n), F, p).double() / (1 - p) if p else None
    outdeg = ops.graphsc_block_degrees(A, dst_dev)
    rows = torch.from_numpy(np.nonzero(g["dst"] >= 0)[0])
    rng = np.random.default_rng(F)
    tol = 1e-6

    # forward over global rows: x [n, F] and out [n_dst, F] as column slices of wider buffers
    x64 = torch.from_numpy(rng.standard_normal((n, F))).float().double()
    xbuf, x = _strided(n, F, cuda)
    x.copy_(x64)
    obuf, out = _strided(g["dst"].size, F, cuda, left=2, right=7)
    ops.graphsc_block_aggregate(A, dst_dev, outdeg, x, agg, p, SEED, key, out=out)
    ref, scale = _agg64(g, weighted, valid, x64, agg, mask)
    o = out.cpu().double()
    ok, e = _rows_within(o[rows], ref, scale, tol)
    assert ok, ("forward", e)
    assert torch.count_nonzero(o[torch.from_numpy(g["dst"] < 0)]).item() == 0, "a padding slot's row is not zero"
    assert torch.count_nonzero(o[torch.from_numpy(np.isin(g["dst"], g["empty"]))]).item() == 0, "an empty row's output is not 0"
    assert _margins_intact(obuf, F, left=2) and _margins_intact(xbuf, F)

    # transposed over global rows, into a strided dx
    dout64 = torch.from_numpy(rng.standard_normal((g["dst"].size, F))).float().double()
    dbuf, dout = _strided(g["dst"].size, F, cuda)
    dout.copy_(dout64)
    dxbuf, dx = _strided(n, F, cuda, left=1, right=4)
    ops.graphsc_block_aggregate(A, dst_dev, outdeg, dout, agg, p, SEED, key, transposed=True, out=dx)
    refT, scaleT = _agg64_T(g, weighted, valid, dout64[rows], agg, mask)
    ok, e = _rows_within(dx.cpu().double(), refT, scaleT, tol)
    assert ok, ("transposed", e)
    # the transposed form zeroes [out_rows, F] only: it used to clear the whole span from out's first to its last element,
    # the columns a row-padded out leaves to its caller included
    assert _margins_intact(dxbuf, F, left=1), "the transposed aggregate wrote outside its [out_rows, F] block"
    # adjoint identity: <A x, dout> = <x, Aᵀ dout>, both sides from the device
    lhs, rhs = float((o[rows] * dout64[rows]).sum()), float((x64 * dx.cpu().double()).sum())
    assert abs(lhs - rhs) <= tol * float((x64.abs() * scaleT).sum()), (lhs, rhs)

    # through x_pos (layer 2 of a two-layer block): x rows are source slots, out_rows exceeds the source count
    cap = int((g["indptr"][valid + 1] - g["indptr"][valid]).sum())
    _, src, pos = ops.graphsc_block_degrees(A, dst_dev, src_cap=cap)
    src_h, pos_h = src.cpu().long(), pos.cpu().long()
    n_src = int((src_h >= 0).sum())
    out_rows = cap + 5
    xr64 = torch.from_numpy(rng.standard_normal((out_rows, F))).float().double()
    xrbuf, xr = _strided(out_rows, F, cuda)
    xr.copy_(xr64)
    out2 = ops.graphsc_block_aggregate(A, dst_dev, outdeg, xr, agg, p, SEED, key, x_pos=pos)
    xg = torch.zeros(n, F, dtype=torch.float64)
    xg[src_h[:n_src]] = xr64[pos_h[src_h[:n_src]]]
    ref, scale = _agg64(g, weighted, valid, xg, agg, mask)
    ok, e = _rows_within(out2.cpu().double()[rows], ref, scale, tol)
    assert ok, ("forward x_pos", e)
    dxrbuf, dxr = _strided(out_rows, F, cuda, left=2, right=2)
    ops.graphsc_block_aggregate(A, dst_dev, outdeg, dout, agg, p, SEED, key, x_pos=pos, transposed=True, out=dxr)
    refr, scaler = torch.zeros(out_rows, F, dtype=torch.float64), torch.zeros(out_rows, F, dtype=torch.float64)
    slots = pos_h[src_h[:n_src]]
    refr[slots], scaler[slots] = refT[src_h[:n_src]], scaleT[src_h[:n_src]]
    ok, e = _rows_within(dxr.cpu().double(), refr, scaler, tol)
    assert ok, ("transposed x_pos", e)
    assert torch.count_nonzero(dxr.cpu()[n_src:]).item() == 0, "a row past the sources is not zero"
    assert _margins_intact(dxrbuf, F, left=2)


def _decoder_check(cuda, z, p, key):
    """ops.graphsc_batch_decoder on z (float32 values, on the host) through strided z / dz against R.batch_loss in float64."""
    from dance_b200 import ops
    B, d = z.shape
    zbuf, zv = _strided(B, d, cuda, left=2, right=3)
    zv.copy_(z)
    dbuf, dz = _strided(B, d, cuda, left=1, right=6)
    loss, _ = ops.graphsc_batch_decoder(zv, p, SEED, key, dz=dz)
    zd = z.double().requires_grad_(True)
    zt = zd * (R.keep_mask(SEED, key, torch.arange(B), d, p).double() / (1 - p)) if p else zd
    ref = R.batch_loss(zt @ zt.t())
    ref.backward()
    assert _margins_intact(dbuf, d, left=1), "the decoder wrote outside dz's [B, d] block"
    assert _margins_intact(zbuf, d, left=2)
    dz = dz.cpu()
    assert bool(torch.isfinite(loss).all()) and bool(torch.isfinite(dz).all())
    return abs(loss.item() - ref.item()) / abs(ref.item()), rel_err(dz, zd.grad)


@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("B", [8, 9, 4097])
@pytest.mark.parametrize("d", [31, 32, 33, 64, 1024])
def test_batch_decoder_edges(cuda, B, d, p):
    """One CTA per 8 rows (B = 4097: 513 CTAs add into one loss), 32-wide k-chunks and column tiles, padded ldz / lddz."""
    g = torch.Generator().manual_seed(B * 31 + d)
    z = torch.randn(B, d, generator=g) * (2.0 / d**0.5)
    e_loss, e_dz = _decoder_check(cuda, z, p, 5 + d)
    assert e_loss <= 1e-5 and e_dz <= 1e-5, (e_loss, e_dz)


@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("B,d", [(9, 33), (129, 64)])
def test_batch_decoder_saturated_logits(cuda, B, d, p):
    """Off-diagonal logits of |S| ~ 100 and diagonal ones in the hundreds, where softplus and σ saturate."""
    g = torch.Generator().manual_seed(B + d)
    z = torch.randn(B, d, generator=g) * (100.0 / d**0.5)**0.5
    e_loss, e_dz = _decoder_check(cuda, z, p, 7)
    assert e_loss <= 1e-5 and e_dz <= 1e-5, (e_loss, e_dz)


# ---- act / act_bwd --------------------------------------------------------------------------------------------------------------
ACT64 = {"none": lambda x: x, "relu": Fn.relu, "elu": Fn.elu, "tanh": torch.tanh, "leaky_relu": Fn.leaky_relu, "gelu": Fn.gelu}
SPECIAL = [0.0, 1e-30, -1e-30, 30.0, -30.0, 1e4, -1e4, 1.0, -1.0, -0.75, -8.0, -10.0, -13.0, 5.0, -5.0]


@pytest.mark.parametrize("act", list(ACT64))
def test_act_and_backward_vs_float64(cuda, act):
    """Every activation code over more elements than the grid-stride loop's grid (sm_count · 16 blocks of 256), on strided
    operands, against float64 torch with its subgradient at 0.  The backward takes the output y (relu, elu, tanh, leaky_relu)
    or the pre-activation x (gelu)."""
    from dance_b200 import ops
    sm = torch.cuda.get_device_properties(cuda).multi_processor_count
    cols = 301
    rows = sm * 16 * 256 // cols + 9
    g = torch.Generator().manual_seed(17)
    x = torch.randn(rows, cols, generator=g) * 3
    x[rows // 2:rows // 2 + 40] = torch.rand(40, cols, generator=g) * -8 - 6          # gelu's cancelling tail, −14 … −6
    flat = x.view(-1)
    s = torch.tensor(SPECIAL)
    flat[:s.numel()], flat[-s.numel():] = s, s
    x64 = x.double()

    xbuf, xv = _strided(rows, cols, cuda)
    xv.copy_(x)
    ybuf, y = _strided(rows, cols, cuda, left=1, right=2)
    ops.act(xv, act, out=y)
    yref = ACT64[act](x64)
    err = (y.cpu().double() - yref).abs()
    # 1 + erf(x/√2) cancels for x < 0: gelu's float32 error is a few ulp of |x|/2 there, not of gelu(x)
    lim = 1e-6 * yref.abs() + (2.0**-22 * x64.abs() if act == "gelu" else 0.0)
    assert bool((err <= lim).all()), (act, float((err - lim).max()))
    assert _margins_intact(ybuf, cols, left=1) and _margins_intact(xbuf, cols)

    dy = torch.randn(rows, cols, generator=g)
    dybuf, dyv = _strided(rows, cols, cuda, left=2, right=1)
    dyv.copy_(dy)
    dxbuf, dx = _strided(rows, cols, cuda, left=4, right=3)
    if act == "gelu":
        ops.act_bwd(dyv, act, x=xv, out=dx)
    else:
        ops.act_bwd(dyv, act, y=None if act == "none" else y, out=dx)
    xg = x64.clone().requires_grad_(True)
    ACT64[act](xg).backward(dy.double())
    err = (dx.cpu().double() - xg.grad).abs()
    # from y, the derivative inherits y's rounding (1 − y² for tanh near ±1, y + 1 for elu far below 0): ≤ 1e-6 · |dy|; gelu's
    # derivative Φ(x) + xφ(x) crosses 0 near x = −0.75 and is below 1e-13 for x ≲ −8, where the bound is the absolute one
    lim = 1e-6 * xg.grad.abs() + 1e-6 * dy.double().abs()
    assert bool((err <= lim).all()), (act, float((err - lim).max()))
    assert _margins_intact(dxbuf, cols, left=4) and _margins_intact(dybuf, cols, left=2)

    if act in ("relu", "leaky_relu"):
        # where y <= 0, relu's gradient is torch's threshold_backward: exactly +0 for any dy, ±inf and NaN included;
        # leaky_relu's is 0.01 · dy in float32
        ys = torch.tensor([0.0, -0.0, -2.0], device=cuda).repeat_interleave(6).view(3, 6)
        dys = torch.tensor([float("inf"), -float("inf"), float("nan"), -1.5, -1e-30, 2.0], device=cuda).repeat(3, 1)
        dx = ops.act_bwd(dys, act, y=ys).cpu()
        if act == "relu":
            assert bool((dx.view(torch.int32) == 0).all()), dx
        else:
            ref = dys.cpu() * 0.01
            assert torch.equal(dx.isnan(), ref.isnan()) and torch.equal(dx[~dx.isnan()], ref[~ref.isnan()]), (dx, ref)


def test_scatter_rows_offset_permuted_strided(cuda):
    """out[idx[i] − offset] = x[i] from a strided x into a strided out; rows idx does not name keep their contents."""
    from dance_b200 import ops
    rows, cols, out_rows, offset = 300, 129, 517, 41
    rng = np.random.default_rng(8)
    idx = rng.permutation(out_rows)[:rows] + offset
    xbuf, x = _strided(rows, cols, cuda)
    x.copy_(torch.from_numpy(rng.standard_normal((rows, cols))))
    obuf, out = _strided(out_rows, cols, cuda, left=5, right=2)
    out.copy_(torch.from_numpy(rng.standard_normal((out_rows, cols))))
    expect = obuf.cpu().clone()
    expect[torch.from_numpy(idx - offset), 5:5 + cols] = x.cpu()
    ops.graphsc_scatter_rows(x, torch.from_numpy(idx).to(torch.int32).to(cuda), out, offset=offset)
    assert torch.equal(obuf.cpu(), expect)
