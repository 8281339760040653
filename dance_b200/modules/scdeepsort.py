"""scDeepSort on the H100-native kernels — host-side mirror of
``dance/modules/single_modality/cell_type_annotation/scdeepsort.py`` (GNN :26-88, ScDeepSort :91-349) and of
``dance/models/nn/gnn.py`` (AdaptiveSAGE :8-96).

Parity note (SURVEY App. B): ``AdaptiveSAGE.forward`` computes the weighted neighbour mean into ``"neigh"`` and
then ignores it — the layer output depends only on the destination node's own features.  With the default
``use_neigh=False`` this module reproduces exactly that (Linear → ReLU → Linear on the cell features, ``alpha``
never receives a gradient); ``neighbour_mean`` exposes the aggregate the reference computes and discards
(edge scalars w_e·alpha[idx(e)] + mean-reduce SpMM), which is the message-passing kernel of this path.
"""
from __future__ import annotations

from copy import deepcopy
from typing import Dict, Optional

import numpy as np
import torch

from .. import ops
from ..engine import FlatParams
from ..graph import GraphLite


class ScDeepSort:

    def __init__(self, dim_in: int, dim_hid: int, num_layers: int, species: str = "", tissue: str = "", *, dropout: int = 0,
                 batch_size: int = 500, device: str = "cuda", precision: Optional[str] = None, seed: Optional[int] = None):
        if num_layers < 1:
            raise ValueError("num_layers must be >= 1")
        if not 0.0 <= float(dropout) < 1.0:
            raise ValueError("dropout must be in [0, 1)")
        self.dense_dim, self.hidden_dim, self.n_layers = dim_in, dim_hid, num_layers
        self.species, self.tissue, self.batch_size = species, tissue, batch_size
        self.device = torch.device(device if device != "auto" else "cuda")
        if self.device.type != "cuda":
            raise RuntimeError("dance_b200 runs on CUDA devices only")
        self.precision, self.seed = precision, seed
        self.dropout = float(dropout)
        self._drop_gen = None                  # device generator for the dropout masks (created on first use)
        self.params: Optional[FlatParams] = None

    # ---- model ------------------------------------------------------------------------------
    def _build(self, num_genes: int, num_labels: int):
        gen = torch.Generator().manual_seed(self.seed) if self.seed is not None else None
        self.num_genes, self.num_labels = int(num_genes), int(num_labels)
        # n_layers AdaptiveSAGE layers (dense_dim → hidden, then hidden → hidden; scdeepsort.py:77-80) and the output Linear.  Every layer's
        # output depends on the destination node's own features only (module docstring), so the stack is an MLP on the cell features.
        spec = [("alpha", (self.num_genes + 2, 1))]
        for i in range(self.n_layers):
            spec += [(f"layers.{i}.layers.1.weight", (self.hidden_dim, self.dense_dim if i == 0 else self.hidden_dim)),
                     (f"layers.{i}.layers.1.bias", (self.hidden_dim, ))]
        spec += [("linear.weight", (self.num_labels, self.hidden_dim)), ("linear.bias", (self.num_labels, ))]
        self.params = FlatParams(spec, self.device)
        P = self.params.p
        P["alpha"].fill_(1.0)                                                           # scdeepsort.py:72
        gain = 2.0**0.5                                                                 # calculate_gain("relu")
        for w, b in [(P[f"layers.{i}.layers.1.weight"], P[f"layers.{i}.layers.1.bias"]) for i in range(self.n_layers)] + \
                [(P["linear.weight"], P["linear.bias"])]:
            fan_out, fan_in = w.shape
            w.copy_((torch.rand(w.shape, generator=gen) * 2 - 1) * gain * (6.0 / (fan_in + fan_out))**0.5)   # xavier_uniform_(gain)
            b.copy_((torch.rand(b.shape, generator=gen) * 2 - 1) / fan_in**0.5)                              # nn.Linear default
        self._alpha_frozen = True   # alpha has no gradient in the reference (unused aggregate) → Adam skips it

    def state_dict(self) -> Dict[str, torch.Tensor]:
        sd = {k: v.detach().clone() for k, v in self.params.p.items()}
        for i in range(self.n_layers):
            sd[f"layers.{i}.alpha"] = sd["alpha"].clone()     # the same Parameter is registered in every layer of the reference (gnn.py:50)
        return sd

    def load_state_dict(self, sd):
        for k, dst in self.params.p.items():
            dst.copy_(torch.as_tensor(sd[k], dtype=torch.float32).reshape(dst.shape))

    def _forward(self, x: torch.Tensor, keep=None):
        """Returns (layer inputs [x_0 … x_{L-1}] after dropout, last hidden h, logits).  ``keep``: per-layer dropout scale tensors
        (training) or None (evaluation)."""
        P = self.params.p
        inputs, h = [], x
        for i in range(self.n_layers):
            if keep is not None:
                h = h * keep[i]
            inputs.append(h)
            h = ops.gemm(h, P[f"layers.{i}.layers.1.weight"], transB=True, bias=P[f"layers.{i}.layers.1.bias"], act="relu",
                         precision=self.precision)
        logits = ops.gemm(h, P["linear.weight"], transB=True, bias=P["linear.bias"], precision=self.precision)
        return inputs, h, logits

    def _train_batch(self, x: torch.Tensor, y: torch.Tensor, lr: float, weight_decay: float, loss_acc: torch.Tensor):
        P, G = self.params.p, self.params.g
        keep = None
        if self.dropout > 0.0:
            # nn.Dropout in front of every AdaptiveSAGE linear (gnn.py:56,92-94): the layer sees only the destination features, so
            # the mask acts on the layer's input; the backward below uses the same masks.  Masks come from a device generator.
            if self._drop_gen is None:
                self._drop_gen = torch.Generator(device=self.device)
                self._drop_gen.manual_seed(int(self.seed) if self.seed is not None else torch.seed() % (2**31))
            widths = [self.dense_dim] + [self.hidden_dim] * (self.n_layers - 1)
            keep = [(torch.rand((x.shape[0], w), device=self.device, generator=self._drop_gen) >= self.dropout).to(torch.float32) /
                    (1.0 - self.dropout) for w in widths]
        inputs, h, logits = self._forward(x, keep)
        _, dlogits = ops.softmax_ce_sum(logits, y, loss_out=loss_acc)                                       # CrossEntropyLoss(sum)
        ops.gemm(dlogits, h, transA=True, out=G["linear.weight"], precision=self.precision)
        ops.colsum(dlogits, out=G["linear.bias"])
        dh = ops.gemm(dlogits, P["linear.weight"], mask=h, precision=self.precision)                        # ⊙ relu'(h)
        for i in reversed(range(self.n_layers)):
            ops.gemm(dh, inputs[i], transA=True, out=G[f"layers.{i}.layers.1.weight"], precision=self.precision)
            ops.colsum(dh, out=G[f"layers.{i}.layers.1.bias"])
            if i > 0:
                # gradient w.r.t. this layer's (dropped-out) input = the previous layer's ReLU output times its dropout scale
                prev = inputs[i] if keep is None else None
                if keep is None:
                    dh = ops.gemm(dh, P[f"layers.{i}.layers.1.weight"], mask=prev, precision=self.precision)
                else:
                    # mask by the ReLU of the previous layer (its output is > 0 exactly where inputs[i] / keep is), then the dropout scale
                    dh = ops.gemm(dh, P[f"layers.{i}.layers.1.weight"], mask=inputs[i], precision=self.precision) * keep[i]
        G["alpha"].zero_()
        a = self.params.p["alpha"].clone() if weight_decay else None
        self.params.adam_step(lr, weight_decay=weight_decay)
        if a is not None:
            self.params.p["alpha"].copy_(a)    # Adam skips parameters whose grad is None: alpha never moves, not even by weight decay

    # ---- reference API ------------------------------------------------------------------------
    def fit(self, graph: GraphLite, labels: torch.Tensor, epochs: int = 300, lr: float = 1e-3, weight_decay: float = 0,
            val_ratio: float = 0.2, batches=None):
        """Same contract as ScDeepSort.fit (scdeepsort.py:142-211).  ``batches`` (optional) = explicit list of
        per-epoch index lists, used by the parity tests in place of the DataLoader's own shuffling."""
        cell_id = graph.ndata["cell_id"]
        num_genes = int((cell_id != -1).sum())
        num_cells = int((cell_id == -1).sum())
        self._build(num_genes, int(labels.max().item()) + 1)
        gen = torch.Generator().manual_seed(self.seed) if self.seed is not None else None
        perm = torch.randperm(num_cells, generator=gen) + num_genes
        num_val = int(num_cells * val_ratio)
        val_idx, train_idx = perm[:num_val], perm[num_val:]
        full_labels = -torch.ones(num_genes + num_cells, dtype=torch.long)
        full_labels[-num_cells:] = labels
        self._feat = graph.ndata["features"].to(self.device, torch.float32)
        self._lab = full_labels.to(self.device)
        max_val_acc, best = 0.0, None
        self.history = []
        for epoch in range(epochs):
            order = batches[epoch] if batches is not None else [train_idx[torch.randperm(len(train_idx), generator=gen)][i:i + self.batch_size]
                                                                 for i in range(0, len(train_idx), self.batch_size)]
            loss = self.cal_loss(order, lr, weight_decay)
            train_acc = self.evaluate(train_idx)[-1]
            val_correct, val_unsure, val_acc = self.evaluate(val_idx) if num_val else (0, 0, 0.0)
            if max_val_acc <= val_acc:
                max_val_acc = val_acc
                best = deepcopy(self.state_dict())
            self.history.append((loss / max(len(train_idx), 1), train_acc, val_acc))
        if best is not None:
            self.load_state_dict(best)

    def cal_loss(self, batch_index_lists, lr: float, weight_decay: float) -> float:
        """One epoch of mini-batches (scdeepsort.py:213-250): returns Σ_b loss_b·size_b / Σ size_b."""
        total_loss = total_size = 0.0
        acc = torch.zeros(1, dtype=torch.float32, device=self.device)
        for idx in batch_index_lists:
            idx = torch.as_tensor(idx, dtype=torch.int64, device=self.device)
            acc.zero_()
            self._train_batch(self._feat.index_select(0, idx), self._lab.index_select(0, idx), lr, weight_decay, acc)
            size = idx.numel()
            total_size += size
            total_loss += acc.item() * size
        return total_loss / max(total_size, 1)

    @torch.no_grad()
    def evaluate(self, idx, unsure_rate: float = 2.0):
        """(correct, unsure, accuracy) with the reference's rule on RAW logits (scdeepsort.py:278-283, App. B)."""
        if len(idx) == 0:
            return 0, 0, 0.0
        idx = torch.as_tensor(idx, dtype=torch.int64, device=self.device)
        _, _, logits = self._forward(self._feat.index_select(0, idx))
        mx, arg = logits.max(1)
        unsure = mx < unsure_rate / self.num_labels
        correct = (~unsure) & (arg == self._lab.index_select(0, idx))
        return int(correct.sum()), int(unsure.sum()), float(correct.sum()) / len(idx)

    @torch.no_grad()
    def predict_proba(self, graph: GraphLite) -> np.ndarray:
        cell_mask = graph.ndata["cell_id"] == -1
        feat = graph.ndata["features"].to(self.device, torch.float32)[cell_mask.to(self.device)]
        out = []
        for i in range(0, feat.shape[0], self.batch_size):
            out.append(self._forward(feat[i:i + self.batch_size])[2])
        return torch.softmax(torch.cat(out), dim=-1).cpu().numpy()

    def predict(self, graph: GraphLite, unsure_rate: float = 2.0, return_unsure: bool = False):
        pred_prob = self.predict_proba(graph)
        pred = pred_prob.argmax(1)
        unsure = pred_prob.max(1) < unsure_rate / self.num_labels
        return (pred, unsure) if return_unsure else pred

    @staticmethod
    def preprocessing_pipeline(n_components: int = 400, log_level="INFO"):
        """scdeepsort.py:134-140."""
        from ..transforms import Compose, PCACellFeatureGraph, SetConfig
        return Compose(PCACellFeatureGraph(n_components=n_components, split_name="train"), SetConfig({"label_channel": "cell_type"}),
                       log_level=log_level)

    def score(self, graph: GraphLite, y, **kw):
        """Default metric 'acc' of BaseClassificationMethod (modules/base.py:156-168): one-hot y, argmax match.  Returned as a
        numpy scalar (the example calls ``score.item()``, examples/.../scdeepsort.py:72)."""
        pred = self.predict(graph)
        y = y.cpu().numpy() if isinstance(y, torch.Tensor) else np.asarray(y)
        true = y.argmax(1) if y.ndim == 2 else y
        return np.float64((pred == true).mean())

    # ---- the aggregate the reference computes and discards ----------------------------------------
    def neighbour_mean(self, graph: GraphLite, h: Optional[torch.Tensor] = None) -> torch.Tensor:
        """block.update_all(message_func, fn.mean("m","neigh")) over the FULL graph (gnn.py:62-90)."""
        g = graph.to(self.device)
        T, _ = g.csr_by_destination("weight")
        vals = ops.sage_edge_values(T, T.vals, self.params.p["alpha"].reshape(-1), self.num_genes)
        h = g.ndata["features"].to(torch.float32) if h is None else h
        F_ = h.shape[1]
        if F_ % 4:
            raise NotImplementedError("feature width must be a multiple of 4")
        return ops.spmm(ops.CSR(T.rowptr, T.colidx, vals, T.shape), h.contiguous(), reduce="mean")
