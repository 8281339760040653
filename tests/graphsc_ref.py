"""graph-sc (GraphSC) test infrastructure: the dgl surface ``GraphSC.fit`` touches beyond ``oracle/dgl_lite.py``, the device's
dropout masks on the host, and a float64 restatement of one mini-batch and of ``fit``.

* ``Block`` / ``MultiLayerFullNeighborSampler`` / ``DataLoader`` extend dgl_lite's full-neighbour blocks with what graphsc.py
  :179-216 and WeightedGraphConv.forward (:428-484) call: ``in_degrees`` / ``out_degrees`` of the BLOCK, ``adjacency_matrix()``
  (rows = sources, columns = destinations, unit values) and ``dstnodes()``.  Batches are drawn as dgl_lite.DataLoader draws them
  (``torch.randperm`` on the default generator; ``drop_last=False`` keeps the short last batch) and recorded in ``history``.
* ``keep_mask``: ``keep(seed, key, row, col)`` of common.cuh (dance_b200.synth restates the hash), the key layout of
  ``GraphSCEngine.drop_key``.
* ``fit``: float64 restatement with the masks as inputs (``masks(step, pass, site, rows, width)`` returns a scaled mask or None).

Plain torch on the CPU; nothing here imports the reference.
"""
from __future__ import annotations

import contextlib
import sys
from pathlib import Path
from typing import Callable, Dict, List, Optional

import numpy as np
import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from dance_b200.synth import _uniform  # noqa: E402
from oracle import dgl_lite  # noqa: E402

SITES = ("layer1", "layer2", "decoder")
DEC_P = 0.1


def drop_key(step: int, pas: int, site: int) -> int:
    """GraphSCEngine.drop_key: (step · 2 + pass) · 3 + site."""
    return (step * 2 + pas) * len(SITES) + site


def keep_mask(seed: int, key: int, rows, width: int, p: float) -> torch.Tensor:
    """Boolean keep bits [len(rows), width] of the device's counter-based dropout."""
    rows = torch.as_tensor(rows).long()
    u = _uniform(int(seed), int(key), rows, torch.arange(width, dtype=torch.long))
    return u >= torch.tensor(p, dtype=torch.float32)


def device_masks(seed: int, p: float):
    """masks(step, pass, site, rows, width) → keep / (1 − p) in float64 (None when that site draws nothing)."""

    def masks(step, pas, site, rows, width):
        q = DEC_P if site == 2 else p
        if q == 0:
            return None
        return keep_mask(seed, drop_key(step, pas, site), rows, width, q).double() / (1.0 - q)

    return masks


# ---------------------------------------------------------------------------------------------------------------------------------
# dgl surface of GraphSC.fit
# ---------------------------------------------------------------------------------------------------------------------------------
class Block(dgl_lite.Block):

    def in_degrees(self):
        return torch.bincount(self.dst, minlength=self.n_dst)

    def out_degrees(self):
        return torch.bincount(self.src, minlength=self.src_nodes.numel())

    def dstnodes(self):
        return torch.arange(self.n_dst)

    def adjacency_matrix(self):
        idx = torch.stack([self.src, self.dst])
        return torch.sparse_coo_tensor(idx, torch.ones(self.src.numel()), (self.src_nodes.numel(), self.n_dst)).coalesce()


class MultiLayerFullNeighborSampler(dgl_lite.NeighborSampler):

    def __init__(self, num_layers, **kwargs):
        super().__init__([-1] * num_layers)


class DataLoader(dgl_lite.DataLoader):
    history: List[torch.Tensor] = []
    on_batch: Optional[Callable] = None

    def __iter__(self):
        order = self.idx[torch.randperm(self.idx.numel())] if self.shuffle else self.idx
        for i in range(0, order.numel(), self.bs):
            seeds = order[i:i + self.bs]
            DataLoader.history.append(seeds.clone())
            blocks, cur = [], seeds
            for _ in range(self.sampler.n_layers):
                b = Block(self.g, cur)
                blocks.insert(0, b)
                cur = b.src_nodes
            if DataLoader.on_batch is not None:
                DataLoader.on_batch(blocks)
            yield cur, seeds, blocks


@contextlib.contextmanager
def reference_fit_env(ref, seed: int, p: float, losses: list):
    """Run the reference's GraphSC.fit on these blocks with the device's masks injected: the model's nn.Dropout and the
    decoder's F.dropout multiply by keep_mask; every batch's loss is appended to ``losses``."""
    dl = sys.modules["dgl.dataloading"]
    had_attr = hasattr(sys.modules["dgl"], "dataloading")
    sys.modules["dgl"].dataloading = dl
    saved = dl.DataLoader, getattr(dl, "MultiLayerFullNeighborSampler", None), ref.F, ref.BCELoss
    state = {"step": -1, "blocks": None, "feat": 0, "dec": 0}

    def on_batch(blocks):
        state.update(step=state["step"] + 1, blocks=blocks, feat=0, dec=0)

    class _F:
        def __getattr__(self, name):
            return getattr(F, name)

        @staticmethod
        def dropout(z, q=0.5, training=True, inplace=False):
            m = keep_mask(seed, drop_key(state["step"], state["dec"], 2), torch.arange(z.shape[0]), z.shape[1], q)
            state["dec"] += 1
            return z * (m.to(z.dtype) / (1.0 - q))

    class _Dropout(torch.nn.Module):
        def forward(self, x):
            nl = len(state["blocks"])
            pas, layer = divmod(state["feat"], nl)
            state["feat"] += 1
            rows = state["blocks"][layer].src_nodes
            return x * (keep_mask(seed, drop_key(state["step"], pas, layer), rows, x.shape[1], p).to(x.dtype) / (1.0 - p))

    def bce(logits, target, pos_weight=None):
        B = logits.shape[0]
        assert torch.equal(target, torch.eye(B, dtype=target.dtype)), "the labels of a batch are its self-loops"
        out = saved[3](logits, target, pos_weight=pos_weight)
        factor = float((B * B - B) * 2) or 1.0
        losses.append(B * B / factor * out.item())
        return out

    dl.DataLoader, dl.MultiLayerFullNeighborSampler = DataLoader, MultiLayerFullNeighborSampler
    DataLoader.history, DataLoader.on_batch = [], on_batch
    ref.F, ref.BCELoss = _F(), bce
    try:
        yield _Dropout
    finally:
        dl.DataLoader, ref.F, ref.BCELoss = saved[0], saved[2], saved[3]
        if saved[1] is not None:
            dl.MultiLayerFullNeighborSampler = saved[1]
        DataLoader.on_batch = None
        if not had_attr:
            del sys.modules["dgl"].dataloading


# ---------------------------------------------------------------------------------------------------------------------------------
# float64 restatement
# ---------------------------------------------------------------------------------------------------------------------------------
def block_edges(indptr: np.ndarray, indices: np.ndarray, weights: Optional[np.ndarray], dst: np.ndarray):
    """Edges (u, position of v in dst, w) of the full-neighbour block with destinations dst, in CSR order."""
    lens = indptr[dst + 1] - indptr[dst]
    pos = np.repeat(np.arange(dst.size), lens)
    eid = np.concatenate([np.arange(indptr[v], indptr[v + 1]) for v in dst]) if dst.size else np.zeros(0, np.int64)
    w = weights[eid] if weights is not None else np.ones(eid.size)
    return indices[eid].astype(np.int64), pos.astype(np.int64), w.astype(np.float64)


def block_outdeg(indptr, indices, dst, n_nodes: int) -> np.ndarray:
    u, _, _ = block_edges(indptr, indices, None, dst)
    return np.bincount(u, minlength=n_nodes)


def block_aggregate(indptr, indices, weights, dst, x_rows: torch.Tensor, n_nodes: int, agg: str = "sum",
                    mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """s_v · Σ_{u→v} w · c_u · (mask ⊙ x)[u]; ``x_rows`` / ``mask`` are indexed by global node id ([n_nodes, F])."""
    u, pos, w = block_edges(indptr, indices, weights, dst)
    outdeg = np.bincount(u, minlength=n_nodes)
    indeg = np.maximum(indptr[dst + 1] - indptr[dst], 1).astype(np.float64)
    x = x_rows if mask is None else x_rows * mask
    # WeightedGraphConv takes both degree norms in float32 (``degrees().float().clamp(min=1) ** -0.5``, graphsc.py:446, :471)
    c = torch.from_numpy(np.maximum(outdeg, 1).astype(np.float32)).pow(-0.5).double()
    msg = x[torch.from_numpy(u)] * (torch.from_numpy(w) * c[torch.from_numpy(u)])[:, None]
    out = torch.zeros(dst.size, x.shape[1], dtype=torch.float64).index_add_(0, torch.from_numpy(pos), msg)
    if agg == "mean":
        out = out / torch.from_numpy(indeg)[:, None]
    return out * torch.from_numpy(indeg.astype(np.float32)).pow(-0.5).double()[:, None]


ACTS = {"relu": F.relu, "leaky_relu": F.leaky_relu, "gelu": F.gelu}


def forward(sd: Dict[str, torch.Tensor], cfg: dict, graph: dict, batch: np.ndarray, masks, step: int, pas: int,
            bn_state: Dict[str, torch.Tensor]):
    """One GCNAE.forward on the batch's blocks (graphsc.py:369-380), float64, train mode.  Returns (logits, emb)."""
    indptr, indices, weights, n = graph["indptr"], graph["indices"], graph["weights"], graph["n_nodes"]
    act = ACTS[cfg["activation"]]
    dsts = [batch]
    for _ in range(cfg["n_layers"] - 1):
        u, _, _ = block_edges(indptr, indices, None, dsts[0])
        dsts.insert(0, np.unique(np.concatenate([dsts[0], u])))
    x = graph["features"]                              # [n_nodes, F] by global id
    for l, dst in enumerate(dsts):
        m = masks(step, pas, l, torch.arange(n), x.shape[1])
        a = block_aggregate(indptr, indices, weights, dst, x, n, cfg["agg"], m)
        h = act(a @ sd[f"layer{l + 1}.weight"] + sd[f"layer{l + 1}.bias"])
        if l + 1 < len(dsts):
            x = torch.zeros(n, h.shape[1], dtype=torch.float64).index_copy(0, torch.from_numpy(dst), h)
        else:
            x = h
    for i in range(cfg["n_hidden"]):
        li = f"encoder.{i * cfg['stride']}"
        x = x @ sd[li + ".weight"].t() + sd[li + ".bias"]
        if cfg["hidden_bn"]:
            bi = f"encoder.{i * cfg['stride'] + 1}"
            x = F.batch_norm(x, bn_state[bi + ".running_mean"], bn_state[bi + ".running_var"], sd[bi + ".weight"], sd[bi + ".bias"],
                             training=True, momentum=0.1, eps=1e-5)
            bn_state[bi + ".num_batches_tracked"] += 1
        if cfg["hidden_relu"]:
            x = F.relu(x)
    m = masks(step, pas, 2, torch.arange(x.shape[0]), x.shape[1])
    zt = x if m is None else x * m
    return zt @ zt.t(), x


def batch_loss(logits: torch.Tensor) -> torch.Tensor:
    """norm · BCEWithLogits(logits, I, pos_weight) with graphsc.py:208-216's constants for y = I."""
    B = logits.shape[0]
    pw = float(B * B - B) / B
    factor = float((B * B - B) * 2) or 1.0
    y = torch.eye(B, dtype=torch.float64)
    return B * B / factor * F.binary_cross_entropy_with_logits(logits, y, pos_weight=torch.tensor([pw], dtype=torch.float64))


def fit(sd: Dict[str, torch.Tensor], cfg: dict, graph: dict, batches: List[np.ndarray], epochs_batches: int, lr: float, masks):
    """GraphSC.fit's loop (graphsc.py:185-231) over the given batches (global node ids, in order), float64: two forwards per
    batch, the first one's embedding recorded, the second one's loss stepped by Adam.  Returns (losses, z [n_cells, d], sd)."""
    params = {k: v.clone().double().requires_grad_(True) for k, v in sd.items() if not _is_buffer(k)}
    bn_state = {k: v.clone().double() if "num_batches" not in k else v.clone() for k, v in sd.items() if _is_buffer(k)}
    opt = torch.optim.Adam(params.values(), lr=lr)
    G = graph["n_genes"]
    z = None
    losses = []
    for step, batch in enumerate(batches):
        _, emb = forward(params, cfg, graph, batch, masks, step, 0, bn_state)
        if z is None:
            z = torch.zeros(graph["n_nodes"] - G, emb.shape[1], dtype=torch.float64)
        z[torch.from_numpy(batch - G)] = emb.detach()
        logits, _ = forward(params, cfg, graph, batch, masks, step, 1, bn_state)
        loss = batch_loss(logits)
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    out = {k: v.detach() for k, v in params.items()}
    out.update(bn_state)
    return np.array(losses), z, out


def _is_buffer(k: str) -> bool:
    return k.endswith(("running_mean", "running_var", "num_batches_tracked"))


# ---------------------------------------------------------------------------------------------------------------------------------
# the reference's GraphSC.fit on a cell–gene graph (``ref`` = oracle.ref_loader.graphsc())
# ---------------------------------------------------------------------------------------------------------------------------------
def synthetic_graph(n_cells: int, n_genes: int, in_feats: int, seed: int, normalize_edges: bool = True, density: float = 0.1):
    """A cell–gene graph as CellFeatureGraph builds it (cell_feature_graph.py:34-79), float64: genes 0..G−1, cells G..G+N−1,
    cell→gene and gene→cell edges weighted by the expression (renormalised per destination when normalize_edges), then a
    self-loop of weight 1 on every node.  Returns a dict with src / dst / weight / features / n_genes / n_nodes."""
    rng = np.random.default_rng(seed)
    X = rng.poisson(2.0, (n_cells, n_genes)) * (rng.random((n_cells, n_genes)) < density)
    X[np.arange(n_cells), rng.integers(0, n_genes, n_cells)] += 1          # every cell expresses something
    X = np.log1p(X.astype(np.float64))
    c, g = np.nonzero(X)
    w = X[c, g]
    src = np.concatenate([c + n_genes, g])
    dst = np.concatenate([g, c + n_genes])
    w = np.concatenate([w, w])
    n = n_genes + n_cells
    if normalize_edges:
        indeg = np.bincount(dst, minlength=n).astype(np.float64)
        wsum = np.bincount(dst, weights=w, minlength=n)
        w = indeg[dst] * w / wsum[dst]
    src = np.concatenate([src, np.arange(n)])
    dst = np.concatenate([dst, np.arange(n)])
    w = np.concatenate([w, np.ones(n)])
    feats = rng.standard_normal((n, in_feats))
    feats = (feats - feats.mean(0)) / feats.std(0)
    return dict(src=src, dst=dst, weight=w, features=feats, n_genes=n_genes, n_nodes=n)


def csr_by_destination(gd: dict):
    order = np.argsort(gd["dst"], kind="stable")
    indptr = np.zeros(gd["n_nodes"] + 1, np.int64)
    indptr[1:] = np.cumsum(np.bincount(gd["dst"], minlength=gd["n_nodes"]))
    return dict(indptr=indptr, indices=gd["src"][order].astype(np.int64), weights=gd["weight"][order], n_nodes=gd["n_nodes"],
                n_genes=gd["n_genes"], features=torch.from_numpy(gd["features"]).double())


def model_kwargs(cfg: dict) -> dict:
    keys = ("agg", "activation", "in_feats", "n_hidden", "hidden_dim", "hidden_1", "hidden_2", "dropout", "n_layers", "hidden_relu",
            "hidden_bn")
    return {k: cfg[k] for k in keys}


def fixture_graph() -> dict:
    """The graph of tests/golden/graphsc_fit.npz: 600 cells × 200 genes, 50 node features, weights and features rounded to
    float32 (the values the device sees).  Regenerated rather than stored; the fixture keeps a checksum (graph_checksum)."""
    gd = synthetic_graph(600, 200, 50, seed=0)
    gd["weight"] = gd["weight"].astype(np.float32).astype(np.float64)
    gd["features"] = gd["features"].astype(np.float32).astype(np.float64)
    return gd


def graph_checksum(gd: dict) -> np.ndarray:
    return np.array([gd["src"].size, gd["n_nodes"], (gd["src"] * 3 + gd["dst"]).sum(), gd["weight"].sum(), (gd["weight"]**2).sum(),
                     gd["features"].sum(), (gd["features"]**2).sum()], np.float64)


def init_state(cfg: dict, seed: int) -> Dict[str, torch.Tensor]:
    """A GCNAE state_dict (the reference's keys and shapes) drawn from ``seed``: weights uniform in ±sqrt(6 / (fan_in + fan_out)),
    biases uniform in ±0.1 (non-zero, unlike the reference's GraphConv init), BatchNorm affine 1 ± 0.1 / ±0.1, running statistics
    0 / 1.  Float32 values (float64 tensors), so the device and the reference start from the same numbers."""
    rng = np.random.default_rng(seed)
    f32 = lambda a: torch.from_numpy(np.asarray(a, np.float32).astype(np.float64))
    uni = lambda shape, a: f32(rng.uniform(-a, a, shape))
    sd = {}
    for l in range(cfg["n_layers"]):
        fin = cfg["in_feats"] if l == 0 else cfg["hidden_dim"]
        sd[f"layer{l + 1}.weight"] = uni((fin, cfg["hidden_dim"]), (6.0 / (fin + cfg["hidden_dim"]))**0.5)
        sd[f"layer{l + 1}.bias"] = uni((cfg["hidden_dim"], ), 0.1)
    stride = 1 + bool(cfg["hidden_bn"]) + bool(cfg["hidden_relu"])
    prev = cfg["hidden_dim"]
    for i, w in enumerate([cfg["hidden_1"], cfg["hidden_2"]][:cfg["n_hidden"]]):
        sd[f"encoder.{i * stride}.weight"] = uni((w, prev), (6.0 / (w + prev))**0.5)
        sd[f"encoder.{i * stride}.bias"] = uni((w, ), 0.1)
        if cfg["hidden_bn"]:
            bn = f"encoder.{i * stride + 1}"
            sd[bn + ".weight"] = 1.0 + uni((w, ), 0.1)
            sd[bn + ".bias"] = uni((w, ), 0.1)
            sd[bn + ".running_mean"] = torch.zeros(w, dtype=torch.float64)
            sd[bn + ".running_var"] = torch.ones(w, dtype=torch.float64)
            sd[bn + ".num_batches_tracked"] = torch.tensor(0, dtype=torch.long)
        prev = w
    return sd


def run_reference_fit(ref, cfg: dict, gd: dict, init: Dict[str, torch.Tensor], fit_seed: int, epochs: int, lr: float,
                      batch_size: int, drop_seed: int):
    """GraphSC(**cfg).fit in float64 from the state ``init`` with the device's masks; returns dict(init, final, z, losses,
    batches)."""
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        model = ref.GraphSC(**model_kwargs(cfg), n_clusters=4, device="cpu")
        model.model.load_state_dict(init)
        g = dgl_lite.Graph(torch.from_numpy(gd["src"]), torch.from_numpy(gd["dst"]), gd["n_nodes"])
        g.edata["weight"] = torch.from_numpy(gd["weight"]).double()[:, None]          # [E, 1], as cell_feature_graph.py stores it
        g.ndata["features"] = torch.from_numpy(gd["features"]).double()
        g.ndata["feat_id"] = torch.cat([-torch.ones(gd["n_genes"], dtype=torch.long), torch.arange(gd["n_nodes"] - gd["n_genes"])])
        losses = []
        with reference_fit_env(ref, drop_seed, cfg["dropout"], losses) as Dropout:
            if model.model.dropout is not None:
                model.model.dropout = Dropout()
            torch.manual_seed(fit_seed)
            model.fit(g, epochs=epochs, lr=lr, batch_size=batch_size)
            batches = [b.numpy() for b in DataLoader.history]
        final = {k: v.detach().clone() for k, v in model.model.state_dict().items()}
        return dict(init=init, final=final, z=np.asarray(model.z, np.float64), losses=np.array(losses), batches=batches)
    finally:
        torch.set_default_dtype(prev)
