"""Explicit forward/backward/optimiser engines of the scGNN hot path.

No autograd: every step is a fixed sequence of C-ABI kernel launches on torch's current
stream (capturable in a CUDA graph).  Parameters, gradients and Adam moments live in ONE
flat fp32 buffer each, so the optimiser is a single launch and — under cell-sharded data
parallelism — the gradient all-reduce is a single NCCL call on one bucket.

Reference being replaced:
  * Feature_AE + train_handler + loss_function_graph   scgnn2.py:338-370, 1217-1328
  * Graph_AE (GCN branch) + graph_AE_handler loop + gae_loss_function
                                                       scgnn2.py:373-412, 479-502, 555-615
  * Graph_AE (GAT branch, with GATLayer's dropout and identity skips)
                                                       scgnn2.py:376-378, 883-1215, 575-593
"""
from __future__ import annotations

import os
from typing import Callable, Dict, List, Optional, Tuple

import numpy as np
import torch

from . import ops
from .ops import CSR


class FlatParams:
    """Named fp32 parameters carved out of one flat buffer (+ grads and Adam state)."""

    def __init__(self, shapes: List[Tuple[str, Tuple[int, ...]]], device):
        self.names = [n for n, _ in shapes]
        self.shapes = dict(shapes)
        # every tensor starts on a 16-byte boundary so that TMA / float4 paths apply
        offs, total = {}, 0
        for n, shp in shapes:
            numel = 1
            for s in shp:
                numel *= s
            offs[n] = (total, numel)
            total += (numel + 3) // 4 * 4
        self.total = total
        self.flat = torch.zeros(total, dtype=torch.float32, device=device)
        self.grad = torch.zeros(total, dtype=torch.float32, device=device)
        self.exp_avg = torch.zeros(total, dtype=torch.float32, device=device)
        self.exp_avg_sq = torch.zeros(total, dtype=torch.float32, device=device)
        self.step = 0
        self.p: Dict[str, torch.Tensor] = {}
        self.g: Dict[str, torch.Tensor] = {}
        for n, shp in shapes:
            o, numel = offs[n]
            self.p[n] = self.flat[o:o + numel].view(*shp)
            self.g[n] = self.grad[o:o + numel].view(*shp)

    def adam_step(self, lr: float, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0.0):
        self.step += 1
        ops.adam_step(self.flat, self.grad, self.exp_avg, self.exp_avg_sq, self.step, lr, betas[0], betas[1], eps,
                      weight_decay)


def _linear_init_(w: torch.Tensor, b: torch.Tensor, gen: Optional[torch.Generator] = None):
    """nn.Linear.reset_parameters: kaiming_uniform(a=sqrt(5)) ⇒ U(-1/sqrt(fan_in), 1/sqrt(fan_in)) for both."""
    fan_in = w.shape[1]
    bound = 1.0 / fan_in**0.5
    w.copy_((torch.rand(w.shape, generator=gen) * 2 - 1) * bound)
    b.copy_((torch.rand(b.shape, generator=gen) * 2 - 1) * bound)


class FeatureAEEngine:
    """Feature_AE (dim→512→128→512→dim, ReLU everywhere) with explicit backward and Adam.

    ``state_dict`` keys match the reference module (fc1.weight … fc4.bias, scgnn2.py:352-355)
    so reference checkpoints load unchanged.
    """

    HID, EMB = 512, 128

    def __init__(self, dim: int, device="cuda", lr: float = 1e-3, precision: Optional[str] = None, seed: Optional[int] = None):
        self.dim, self.device, self.lr, self.precision = dim, torch.device(device), lr, precision
        H, E = self.HID, self.EMB
        self.params = FlatParams([("fc1.weight", (H, dim)), ("fc1.bias", (H, )), ("fc2.weight", (E, H)), ("fc2.bias", (E, )),
                                  ("fc3.weight", (H, E)), ("fc3.bias", (H, )), ("fc4.weight", (dim, H)), ("fc4.bias", (dim, ))],
                                 self.device)
        self.seed = seed
        gen = torch.Generator().manual_seed(seed) if seed is not None else None
        for i in (1, 2, 3, 4):
            _linear_init_(self.params.p[f"fc{i}.weight"], self.params.p[f"fc{i}.bias"], gen)
        self._bufs = {}
        self.loss_acc = torch.zeros(1, dtype=torch.float32, device=self.device)
        # hook called between backward and the optimiser step (gradient all-reduce under data parallelism)
        self.grad_hook: Optional[Callable[[torch.Tensor], None]] = None

    # -- checkpoint interface -------------------------------------------------
    def state_dict(self) -> Dict[str, torch.Tensor]:
        return {k: v.detach().clone() for k, v in self.params.p.items()}

    def load_state_dict(self, sd):
        for k, v in sd.items():
            self.params.p[k].copy_(torch.as_tensor(v, dtype=torch.float32))

    # -- buffers ----------------------------------------------------------------
    def _buffers(self, B: int, slot: int = 0):
        """Activation / gradient buffers of a batch of B rows.  ``slot`` selects one of several independent sets, so that a
        caller can still be reading batch b's outputs (device→host copy on a side stream) while batch b+1 trains."""
        bufs = self._bufs.get((B, slot))
        if bufs is None:
            H, E, D = self.HID, self.EMB, self.dim
            mk = lambda *s: torch.empty(*s, dtype=torch.float32, device=self.device)
            bufs = dict(h1=mk(B, H), z=mk(B, E), h3=mk(B, H), r=mk(B, D), dr=mk(B, D), dh3=mk(B, H), dz=mk(B, E), dh1=mk(B, H))
            self._bufs[(B, slot)] = bufs
        return bufs

    # -- forward ----------------------------------------------------------------
    def input_dropout(self, x: torch.Tensor, p: float) -> torch.Tensor:
        """``F.dropout(x, p)`` with this engine's device generator (inverted dropout: kept entries scaled by 1 / (1 - p))."""
        if not 0.0 <= p < 1.0:
            raise ValueError("dropout probability must be in [0, 1)")
        if getattr(self, "_drop_gen", None) is None:
            self._drop_gen = torch.Generator(device=self.device)
            self._drop_gen.manual_seed(int(self.seed) + 7919 if getattr(self, "seed", None) is not None else torch.seed() % (2**31))
        keep = torch.rand(x.shape, device=self.device, generator=self._drop_gen) >= p
        return x * keep.to(torch.float32).mul_(1.0 / (1.0 - p))

    def forward(self, x: torch.Tensor, bufs=None):
        """Returns (z, recon) like Feature_AE.forward (scgnn2.py:368-370)."""
        P, pr = self.params.p, self.precision
        b = bufs or self._buffers(x.shape[0])
        ops.gemm(x, P["fc1.weight"], transB=True, bias=P["fc1.bias"], act="relu", out=b["h1"], precision=pr)
        ops.gemm(b["h1"], P["fc2.weight"], transB=True, bias=P["fc2.bias"], act="relu", out=b["z"], precision=pr)
        ops.gemm(b["z"], P["fc3.weight"], transB=True, bias=P["fc3.bias"], act="relu", out=b["h3"], precision=pr)
        ops.gemm(b["h3"], P["fc4.weight"], transB=True, bias=P["fc4.bias"], act="relu", out=b["r"], precision=pr)
        return b["z"], b["r"]

    # -- one optimiser step -------------------------------------------------------
    def train_step(self, x: torch.Tensor, ltmg: Optional[torch.Tensor] = None, regu_strength: float = 0.9,
                   regularizer_type: str = "noregu", slot: int = 0, row_weight: Optional[torch.Tensor] = None,
                   x_dropout: Optional[torch.Tensor] = None, x_input: Optional[torch.Tensor] = None):
        """One mini-batch of train_handler (scgnn2.py:1256-1281): forward, loss_function_graph
        ('noregu' | 'LTMG'), backward, Adam.  The batch loss is accumulated into ``self.loss_acc``.
        ``x_input``: what the network sees when it differs from the loss target ``x`` — ``F.dropout(data, p=masked_prob)`` of
        train_handler (scgnn2.py:1256); the first layer's weight gradient is taken against it.
        Returns (z, recon) views into the engine's buffers (valid until the next call with the same batch size)."""
        P, G, pr = self.params.p, self.params.g, self.precision
        B = x.shape[0]
        b = self._buffers(B, slot)
        x_in = x if x_input is None else x_input
        z, r = self.forward(x_in, b)
        if regularizer_type == "noregu":
            ops.mse_sum_loss_grad(r, x, None, 0.0, relu_mask=True, grad=b["dr"], loss_out=self.loss_acc)
        elif regularizer_type == "LTMG":
            # ltmg=None ⇔ the all-zero TRS matrix of the reference driver (scgnn2.py:40)
            ops.mse_sum_loss_grad(r, x, ltmg, regu_strength, relu_mask=True, grad=b["dr"], loss_out=self.loss_acc)
        elif regularizer_type == "Celltype":
            # Cluster-AE inside the EM loop (scgnn2.py:1316-1326): 0.3·BCE + ‖(x_dropout − r)[x_dropout≠0]‖ + 0.3·(adj_cc @ mse).sum()
            # + 0.1·(celltype_cc @ mse).sum(); the two dense products are per-row weights here (row_weight, see ops.graph_regu_weights)
            ops.celltype_loss_grad(r, x, x_dropout, row_weight, relu_mask=True, grad=b["dr"], loss_out=self.loss_acc)
        else:
            raise ValueError(f"unsupported regularizer_type {regularizer_type!r}")
        # layer 4:  r = relu(h3 W4ᵀ + b4)
        ops.gemm(b["dr"], b["h3"], transA=True, out=G["fc4.weight"], precision=pr)
        ops.colsum(b["dr"], out=G["fc4.bias"])
        ops.gemm(b["dr"], P["fc4.weight"], mask=b["h3"], out=b["dh3"], precision=pr)
        # layer 3
        ops.gemm(b["dh3"], b["z"], transA=True, out=G["fc3.weight"], precision=pr)
        ops.colsum(b["dh3"], out=G["fc3.bias"])
        ops.gemm(b["dh3"], P["fc3.weight"], mask=b["z"], out=b["dz"], precision=pr)
        # layer 2
        ops.gemm(b["dz"], b["h1"], transA=True, out=G["fc2.weight"], precision=pr)
        ops.colsum(b["dz"], out=G["fc2.bias"])
        ops.gemm(b["dz"], P["fc2.weight"], mask=b["h1"], out=b["dh1"], precision=pr)
        # layer 1
        ops.gemm(b["dh1"], x_in, transA=True, out=G["fc1.weight"], precision=pr)
        ops.colsum(b["dh1"], out=G["fc1.bias"])
        if regularizer_type == "Celltype":
            # `loss = loss + 1 * l1 + 0 * l2` over all parameters (train_handler, scgnn2.py:1268-1274)
            ops.l1_grad_add(self.params.flat, self.params.grad, 1.0, self.loss_acc)
        if self.grad_hook is not None:
            self.grad_hook(self.params.grad)
        self.params.adam_step(self.lr)
        return z, r

    def idle_step(self):
        """Optimiser step of a rank whose shard has no rows left in this epoch (uneven shards under data parallelism): it
        contributes a zero gradient to the all-reduce and applies the same reduced gradient, so the replicas stay identical and
        every rank issues the same number of collectives."""
        self.params.grad.zero_()
        if self.grad_hook is not None:
            self.grad_hook(self.params.grad)
        self.params.adam_step(self.lr)

    def train_epoch(self, X: torch.Tensor, batch_size: int, regularizer_type: str = "noregu", regu_strength: float = 0.9,
                    ltmg: Optional[torch.Tensor] = None, z_out: Optional[torch.Tensor] = None,
                    recon_out: Optional[torch.Tensor] = None, n_steps: Optional[int] = None) -> torch.Tensor:
        """One epoch over device-resident X in order (DataLoader without shuffle, scgnn2.py:299).
        Optionally gathers the per-batch embeddings / reconstructions (the reference's ``torch.cat``
        of all batches, scgnn2.py:1284-1291).  Returns the device scalar of summed batch losses.
        ``n_steps`` (data parallelism): optimiser steps of the epoch = ``parallel.epoch_steps(bounds, batch_size)``."""
        from .parallel import batch_schedule
        self.loss_acc.zero_()
        for rng in batch_schedule(X.shape[0], batch_size, n_steps):
            if rng is None:
                self.idle_step()
                continue
            b0, b1 = rng
            z, r = self.train_step(X[b0:b1], None if ltmg is None else ltmg[b0:b1], regu_strength, regularizer_type)
            if z_out is not None:
                z_out[b0:b1].copy_(z)
            if recon_out is not None:
                recon_out[b0:b1].copy_(r)
        return self.loss_acc


def _xavier_uniform_(w: torch.Tensor, gen: Optional[torch.Generator] = None):
    fan_in, fan_out = w.shape[0], w.shape[1]  # GraphConvolution.weight is [in, out]; xavier is symmetric in the two
    bound = (6.0 / (fan_in + fan_out))**0.5
    w.copy_((torch.rand(w.shape, generator=gen) * 2 - 1) * bound)


class GraphAEEngine:
    """Graph_AE, GCN branch: gc1 (dim→32, ReLU), gc2/gc3 (32→emb, identity) sharing hidden1,
    reparameterise, inner-product decoder, pos-weighted BCE + KLD — all matrix-free.

    gc2 and gc3 are evaluated as ONE projection + ONE SpMM over the packed weight
    ``[W2 | W3]`` (F = 2·emb): both read the same hidden1 and the same Â (scgnn2.py:389-391).
    """

    HID = 32

    def __init__(self, dim: int, embedding_size: int = 16, device="cuda", lr: float = 1e-2, precision: Optional[str] = None,
                 seed: Optional[int] = None):
        self.dim, self.emb, self.device, self.lr, self.precision = dim, embedding_size, torch.device(device), lr, precision
        self.params = FlatParams([("gc1.weight", (dim, self.HID)), ("gc23.weight", (self.HID, 2 * embedding_size))], self.device)
        gen = torch.Generator().manual_seed(seed) if seed is not None else None
        w1 = torch.empty(dim, self.HID)
        w2 = torch.empty(self.HID, embedding_size)
        w3 = torch.empty(self.HID, embedding_size)
        for w in (w1, w2, w3):
            _xavier_uniform_(w, gen)
        self.load_state_dict({"gc1.weight": w1, "gc2.weight": w2, "gc3.weight": w3})
        self._bufs = {}
        self.loss = torch.zeros(1, dtype=torch.float32, device=self.device)
        self.grad_hook: Optional[Callable[[torch.Tensor], None]] = None

    def state_dict(self):
        e = self.emb
        w23 = self.params.p["gc23.weight"]
        return {"gc1.weight": self.params.p["gc1.weight"].detach().clone(), "gc2.weight": w23[:, :e].detach().clone(),
                "gc3.weight": w23[:, e:].detach().clone()}

    def load_state_dict(self, sd):
        e = self.emb
        self.params.p["gc1.weight"].copy_(torch.as_tensor(sd["gc1.weight"], dtype=torch.float32))
        self.params.p["gc23.weight"][:, :e].copy_(torch.as_tensor(sd["gc2.weight"], dtype=torch.float32))
        self.params.p["gc23.weight"][:, e:].copy_(torch.as_tensor(sd["gc3.weight"], dtype=torch.float32))

    def grads(self):
        e = self.emb
        g23 = self.params.g["gc23.weight"]
        return {"gc1.weight": self.params.g["gc1.weight"], "gc2.weight": g23[:, :e], "gc3.weight": g23[:, e:]}

    def _buffers(self, n: int):
        b = self._bufs.get(n)
        if b is None:
            H, e = self.HID, self.emb
            mk = lambda *s: torch.empty(*s, dtype=torch.float32, device=self.device)
            b = dict(s1=mk(n, H), h1=mk(n, H), s2=mk(n, 2 * e), ml=mk(n, 2 * e), z=mk(n, e), dz=mk(n, e), dml=mk(n, 2 * e),
                     ds2=mk(n, 2 * e), dh1=mk(n, H), ds1=mk(n, H))
            self._bufs[n] = b
        return b

    # -- cell-sharded execution ---------------------------------------------------
    def set_sharding(self, comm, bounds):
        """Row-shard the graph across ranks: this rank owns rows bounds[comm.rank] of Â (``adj`` passed
        to forward/train_step is then the local row block, column ids global)."""
        self.comm, self.bounds = comm, bounds

    def _gather(self, local: torch.Tensor, key: str) -> torch.Tensor:
        comm = getattr(self, "comm", None)
        if comm is None or not comm.enabled:
            return local
        full = self._bufs.setdefault(("full", key, local.shape[1]),
                                     torch.empty(self.bounds[-1][1], local.shape[1], dtype=torch.float32, device=self.device))
        return comm.all_gather_rows(local, self.bounds, out=full)

    def forward(self, x: torch.Tensor, adj: CSR, eps: Optional[torch.Tensor] = None):
        """Graph_AE.forward(use_GAT=False) (scgnn2.py:402-412): returns (z, mu, logvar); z = mu when eps is None.
        Under sharding x / eps / outputs are the local rows."""
        P, pr, e = self.params.p, self.precision, self.emb
        b = self._buffers(x.shape[0])
        ops.gemm(x, P["gc1.weight"], out=b["s1"], precision=pr)          # support = input @ W      (scgnn2.py:499)
        ops.spmm(adj, self._gather(b["s1"], "s1"), act="relu", out=b["h1"])   # act(spmm(adj, support)) (scgnn2.py:500-501)
        ops.gemm(b["h1"], P["gc23.weight"], out=b["s2"], precision=pr)
        ops.spmm(adj, self._gather(b["s2"], "s2"), out=b["ml"])
        mu, logvar = b["ml"][:, :e], b["ml"][:, e:]
        if eps is None:
            return mu, mu, logvar
        ops.reparam_fwd(mu, logvar, eps, out=b["z"])
        return b["z"], mu, logvar

    def train_step(self, x: torch.Tensor, adj: CSR, labels: CSR, norm: float, pos_weight: float, eps: torch.Tensor,
                   adj_t: Optional[CSR] = None, labels_t: Optional[CSR] = None):
        """One epoch of the graph_AE_handler loop (scgnn2.py:575-593): forward, gae_loss_function,
        backward, Adam.  ``adj_t`` = Âᵀ for the backward SpMMs; defaults to Â itself (the
        preprocess_graph output is symmetric, scgnn2.py:1196).  Real-valued labels (``labels.vals`` set, graph_AE_retain_weights)
        come with ``labels_t``, the same rows of Lᵀ (see ops.gae_loss_grad).  Loss is left in ``self.loss``
        (under sharding: all-reduced, so every rank holds the global value)."""
        P, G, pr, e = self.params.p, self.params.g, self.precision, self.emb
        adj_t = adj_t or adj
        comm = getattr(self, "comm", None)
        sharded = comm is not None and comm.enabled
        n_loc = x.shape[0]
        row_begin = self.bounds[comm.rank][0] if sharded else 0
        b = self._buffers(n_loc)
        z, mu, logvar = self.forward(x, adj, eps)
        dmu, dlv = b["dml"][:, :e], b["dml"][:, e:]
        z_all = self._gather(z, "z")
        n_all = z_all.shape[0]
        path = ops.get_path("gae")
        if sharded and e <= 16 and (path == "tc" or (path == "auto" and n_all * n_all >= (1 << 24))):
            # the tensor-core decoder is partitioned by super-block (row blocks s and nb−1−s, equal work each): this rank takes its
            # share, writes partial gradients into a full-size buffer and the ranks sum them (one 64 MB all-reduce at 1 M)
            from .parallel import shard_bounds
            sb0, sb1 = shard_bounds(ops.gae_sym_super_blocks(n_all), comm.world)[comm.rank]
            dzf = self._bufs.setdefault(("dz_full", n_all), torch.empty(n_all, e, dtype=torch.float32, device=self.device))
            ops.gae_loss_grad_sym(z_all, labels, norm, pos_weight, sb0, sb1, mu, logvar, True, dz_full=dzf, dmu=dmu, dlogvar=dlv,
                                  loss=self.loss, row_begin=row_begin, n_rows=n_loc, labels_t=labels_t)
            comm.allreduce_sum_(dzf)
            b["dz"].copy_(dzf[row_begin:row_begin + n_loc])
        else:
            ops.gae_loss_grad(z_all, labels, norm, pos_weight, mu, logvar, True, dz=b["dz"], dmu=dmu, dlogvar=dlv, loss=self.loss,
                              row_begin=row_begin, n_rows=n_loc, labels_t=labels_t)
        ops.reparam_bwd(b["dz"], logvar, eps, dmu, dlv)                  # chain through z = mu + eps·exp(logvar)
        ops.spmm(adj_t, self._gather(b["dml"], "dml"), out=b["ds2"])     # d support2 = Âᵀ · d[mu|logvar]
        ops.gemm(b["h1"], b["ds2"], transA=True, out=G["gc23.weight"], precision=pr)
        ops.gemm(b["ds2"], P["gc23.weight"], transB=True, mask=b["h1"], out=b["dh1"], precision=pr)  # ⊙ relu'(hidden1)
        ops.spmm(adj_t, self._gather(b["dh1"], "dh1"), out=b["ds1"])
        ops.gemm(x, b["ds1"], transA=True, out=G["gc1.weight"], precision=pr)
        if sharded:
            comm.allreduce_sum_(self.params.grad)
            comm.allreduce_sum_(self.loss)
        if self.grad_hook is not None:
            self.grad_hook(self.params.grad)
        self.params.adam_step(self.lr)
        return z, mu, logvar


class GATEngine:
    """The 2-layer GAT of Graph_AE (scgnn2.py:376-378, 883-917): layer 1 concat + ELU, layer 2 head-mean,
    skip projections and biases, global-max edge softmax — explicit forward / backward / Adam.

    Per layer the attention projection and the skip projection read the same input, so they are stored
    packed ``[linear_proj ; skip_proj]`` and evaluated by ONE GEMM; ``state_dict`` splits them back into the
    reference's keys (``gat.gat_net.{l}.linear_proj.weight`` …).  A layer whose input width equals its per-head output
    width adds its raw input to every head instead (scgnn2.py:1167-1171): it runs the projection half of the GEMM only, and
    ``skip_proj`` — kept for the state_dict, as in the reference — gets an exactly zero gradient, so Adam never moves it.

    ``dropout`` is GATLayer's ``nn.Dropout(p)`` in training steps, at its three sites (scgnn2.py:1005, 1010, 1029): the layer
    input, the projection ``H`` and the attention coefficients.  The masks are counter-based draws under ``seed`` with one key
    per (training step, layer, site) — :meth:`drop_key` — and the backward regenerates them (see :func:`ops.dropout`).
    """

    SITES = ("input", "proj", "attn")

    def __init__(self, dim: int, hid: int = 64, embedding_size: int = 16, heads: int = 2, device="cuda", lr: float = 1e-2,
                 precision: Optional[str] = None, seed: Optional[int] = None, *, dropout: float = 0.0):
        self.device, self.lr, self.precision, self.nh = torch.device(device), lr, precision, heads
        self.dropout = ops._drop_prob(dropout)
        # seed of the dropout draws; without a seed (and with dropout), one from torch's default generator
        self.drop_seed = int(seed) & 0xFFFFFFFF if seed is not None else (int(torch.randint(0, 2**31, (1, )).item()) if self.dropout else 0)
        self.step = 0        # training steps taken: part of every dropout key
        self.layers = [dict(fin=dim, F=hid, concat=True, act="elu"), dict(fin=hid * heads, F=embedding_size, concat=False, act=None)]
        for L in self.layers:
            L["identity"] = L["fin"] == L["F"]
        shapes = []
        for l, L in enumerate(self.layers):
            W = heads * L["F"]
            shapes += [(f"l{l}.projskip", (2 * W, L["fin"])), (f"l{l}.a_trg", (W, )), (f"l{l}.a_src", (W, )),
                       (f"l{l}.bias", (W if L["concat"] else L["F"], ))]
        self.params = FlatParams(shapes, self.device)
        gen = torch.Generator().manual_seed(seed) if seed is not None else None
        for l, L in enumerate(self.layers):
            W, fin, F = heads * L["F"], L["fin"], L["F"]
            proj = torch.empty(W, fin)
            proj.copy_((torch.rand(W, fin, generator=gen) * 2 - 1) * (6.0 / (W + fin))**0.5)   # xavier_uniform_
            skip = (torch.rand(W, fin, generator=gen) * 2 - 1) / fin**0.5          # nn.Linear default init
            # xavier_uniform_ on a (1, NH, F) tensor: fan_in = NH·F, fan_out = F   (torch's fan computation for 3-D tensors)
            ab = (6.0 / (heads * F + F))**0.5
            self.params.p[f"l{l}.projskip"][:W].copy_(proj)
            self.params.p[f"l{l}.projskip"][W:].copy_(skip)
            self.params.p[f"l{l}.a_trg"].copy_((torch.rand(W, generator=gen) * 2 - 1) * ab)
            self.params.p[f"l{l}.a_src"].copy_((torch.rand(W, generator=gen) * 2 - 1) * ab)
            self.params.p[f"l{l}.bias"].zero_()
        self.loss = torch.zeros(1, dtype=torch.float32, device=self.device)
        self._cache = {}

    # reference key layout: gat.gat_net.{l}.{linear_proj.weight, skip_proj.weight, scoring_fn_target, scoring_fn_source, bias}
    def state_dict(self):
        sd = {}
        for l, L in enumerate(self.layers):
            W, F = self.nh * L["F"], L["F"]
            pre = f"gat.gat_net.{l}."
            sd[pre + "linear_proj.weight"] = self.params.p[f"l{l}.projskip"][:W].detach().clone()
            sd[pre + "skip_proj.weight"] = self.params.p[f"l{l}.projskip"][W:].detach().clone()
            sd[pre + "scoring_fn_target"] = self.params.p[f"l{l}.a_trg"].detach().clone().view(1, self.nh, F)
            sd[pre + "scoring_fn_source"] = self.params.p[f"l{l}.a_src"].detach().clone().view(1, self.nh, F)
            sd[pre + "bias"] = self.params.p[f"l{l}.bias"].detach().clone()
        return sd

    def _split(self, store, l):
        W, F = self.nh * self.layers[l]["F"], self.layers[l]["F"]
        pre = f"gat.gat_net.{l}."
        return {pre + "linear_proj.weight": store[f"l{l}.projskip"][:W], pre + "skip_proj.weight": store[f"l{l}.projskip"][W:],
                pre + "scoring_fn_target": store[f"l{l}.a_trg"].view(1, self.nh, F),
                pre + "scoring_fn_source": store[f"l{l}.a_src"].view(1, self.nh, F), pre + "bias": store[f"l{l}.bias"]}

    def load_state_dict(self, sd):
        for l in range(len(self.layers)):
            for k, dst in self._split(self.params.p, l).items():
                dst.copy_(torch.as_tensor(sd[k], dtype=torch.float32).reshape(dst.shape))

    def grads(self):
        out = {}
        for l in range(len(self.layers)):
            out.update(self._split(self.params.g, l))
        return out

    def drop_key(self, layer: int, site: str, step: Optional[int] = None) -> int:
        """Key of the dropout draw at ``site`` ("input" | "proj" | "attn") of ``layer`` in training step ``step`` (default: the
        step :meth:`train_step` runs next).  ``ops.dropout(ones, p, eng.drop_seed, key)`` reproduces the mask; for "attn" over
        [nnz, heads], row p is the edge at position p of the target CSR."""
        s = self.step if step is None else step
        return (s * len(self.layers) + layer) * len(self.SITES) + self.SITES.index(site)

    def _drop_kw(self, l: int, site: str) -> dict:
        return dict(dropout=self.dropout, seed=self.drop_seed, key=self.drop_key(l, site))

    def forward(self, x: torch.Tensor, T: CSR, keep: bool = False, training: bool = False):
        """GAT.forward on the target-indexed CSR ``T`` (row v = sources of v's in-edges); returns the node embedding.
        ``training``: apply the layers' dropout (train() mode) with the keys of the current step."""
        P, pr, nh = self.params.p, self.precision, self.nh
        drop = training and self.dropout > 0
        h = x
        for l, L in enumerate(self.layers):
            W = nh * L["F"]
            if drop:
                h = ops.dropout(h, self.dropout, self.drop_seed, self.drop_key(l, "input"))   # out of place: ELU backward reads `out`
            if L["identity"]:
                hs = ops.gemm(h, P[f"l{l}.projskip"][:W], transB=True, precision=pr)   # [n, W]: projection; the skip is h itself
                H, skip = hs, h
            else:
                hs = ops.gemm(h, P[f"l{l}.projskip"], transB=True, precision=pr)       # [n, 2W]: projection | skip projection
                H, skip = hs[:, :W], hs[:, W:]
            if drop:
                ops.dropout(H, self.dropout, self.drop_seed, self.drop_key(l, "proj"), out=H)
            s_src, s_trg = ops.gat_scores(H, P[f"l{l}.a_src"], P[f"l{l}.a_trg"], nh)
            agg, alpha, gmax = ops.gat_aggregate_fwd(T, H, s_src, s_trg, nh, "leakyrelu", 0.2, "global", keep_alpha=keep,
                                                     **(self._drop_kw(l, "attn") if drop else {}))
            out = ops.gat_combine_fwd(agg, skip, P[f"l{l}.bias"], nh, L["concat"], L["act"], identity=L["identity"])
            if keep:
                self._cache[l] = dict(x=h, hs=hs, s_src=s_src, s_trg=s_trg, alpha=alpha, gmax=gmax, out=out, drop=drop)
            h = out
        return h

    def train_step(self, x: torch.Tensor, T: CSR, Tt: CSR, t_perm: torch.Tensor, labels: CSR, labels_t: Optional[CSR] = None):
        """One epoch of graph_AE_handler with use_GAT=True (scgnn2.py:575-593): forward (train mode), loss_function
        (plain mean BCE on z zᵀ, scgnn2.py:618-619), backward, Adam.  Soft labels (``labels.vals`` set, graph_AE_retain_weights)
        come with ``labels_t``, Lᵀ.  Returns the embedding of this (dropped-out) forward."""
        P, G, pr, nh = self.params.p, self.params.g, self.precision, self.nh
        z = self.forward(x, T, keep=True, training=True)
        _, dz, _, _ = ops.gae_loss_grad(z, labels, 1.0, 1.0, use_pos_weight=False, loss=self.loss, labels_t=labels_t)
        dout = dz
        for l in reversed(range(len(self.layers))):
            L, c = self.layers[l], self._cache[l]
            W, F = nh * L["F"], L["F"]
            drop, ident = c["drop"], L["identity"]
            if ident:
                dskip, dact, dx = ops.gat_combine_bwd(dout, c["out"], nh, F, L["concat"], L["act"], identity=True)
            else:
                dhs = torch.empty_like(c["hs"])                                       # [n, 2W]: d projection | d skip
                dH, dskip = dhs[:, :W], dhs[:, W:]
                _, dact = ops.gat_combine_bwd(dout, c["out"], nh, F, L["concat"], L["act"], dpre=dskip)
            ops.colsum(dact, out=G[f"l{l}.bias"])
            H = c["hs"][:, :W]
            dHm, da_src, da_trg = ops.gat_aggregate_bwd(T, Tt, t_perm, H, P[f"l{l}.a_src"], P[f"l{l}.a_trg"], c["s_src"], c["s_trg"],
                                                        c["alpha"], dskip, nh, gmax=c["gmax"],
                                                        **(self._drop_kw(l, "attn") if drop else {}))
            if ident:
                dH = dHm
            else:
                dH.copy_(dHm)
            if drop:
                ops.dropout(dH, self.dropout, self.drop_seed, self.drop_key(l, "proj"), out=dH)
            G[f"l{l}.a_src"].copy_(da_src)
            G[f"l{l}.a_trg"].copy_(da_trg)
            if ident:
                # skip_proj's half of the gradient stays zero (FlatParams starts it at zero and nothing writes it)
                ops.gemm(dH, c["x"], transA=True, out=G[f"l{l}.projskip"][:W], precision=pr)
                if l > 0:
                    dout = ops.gemm(dH, P[f"l{l}.projskip"][:W], out=dx, accumulate=True, precision=pr)
            else:
                ops.gemm(dhs, c["x"], transA=True, out=G[f"l{l}.projskip"], precision=pr)
                if l > 0:
                    dout = ops.gemm(dhs, P[f"l{l}.projskip"], precision=pr)
            if l > 0 and drop:
                ops.dropout(dout, self.dropout, self.drop_seed, self.drop_key(l, "input"), out=dout)
        self.params.adam_step(self.lr)
        self.step += 1
        return z


class GraphSCEngine:
    """graph-sc's GCNAE (graphsc.py:290-411) trained by GraphSC.fit's loop (:185-231) on the device.

    Per mini-batch of cell nodes: the block out-degrees (one histogram per layer, ``ops.graphsc_block_degrees``), two train-mode
    forwards with independent dropout draws (the first one's embedding is recorded in cell order, the second one's logits give
    the loss), the fused decoder loss / gradient, the backward and one Adam step over the flat parameter bucket.  WeightedGraphConv
    aggregates before its product with W (linear, so equal to the reference's W-first order up to rounding).  Nothing inside
    :meth:`train_epoch` synchronises with the host: batch composition is known on the host (the permutation is drawn there), the
    per-batch losses stay in :attr:`losses` and the embeddings in :attr:`z`.

    Dropout keys (``ops.dropout(ones, p, drop_seed, key)`` reproduces a mask): :meth:`drop_key`; feature-dropout rows are
    global node ids, decoder rows are positions in the batch.
    """

    SITES = ("layer1", "layer2", "decoder")
    DEC_P = 0.1           # InnerProductDecoder's F.dropout(z, 0.1), always in training mode (graphsc.py:408-411)

    def __init__(self, *, agg: str = "sum", activation: str = "relu", in_feats: int = 50, n_hidden: int = 1, hidden_dim: int = 200,
                 hidden_1: int = 300, hidden_2: int = 0, dropout: float = 0.1, n_layers: int = 1, hidden_relu: bool = False,
                 hidden_bn: bool = False, device="cuda", drop_seed: int = 0, precision: Optional[str] = None):
        if agg not in ("sum", "mean"):
            raise ValueError(f"agg must be 'sum' or 'mean', got {agg!r}")
        if n_layers not in (1, 2):
            raise ValueError(f"n_layers must be 1 or 2, got {n_layers}")
        if n_hidden not in (0, 1, 2):
            raise ValueError(f"n_hidden must be 0, 1 or 2, got {n_hidden}")
        if not 0.0 <= float(dropout) < 1.0:
            raise ValueError(f"dropout must be in [0, 1), got {dropout}")
        hidden = [hidden_1, hidden_2][:n_hidden]
        for name, w in (("in_feats", in_feats), ("hidden_dim", hidden_dim), ("hidden_1", hidden_1 if n_hidden >= 1 else 1),
                        ("hidden_2", hidden_2 if n_hidden == 2 else 1)):
            if int(w) <= 0:
                raise ValueError(f"{name} must be a positive layer width, got {w}")
        self.agg, self.activation, self.n_layers, self.hidden = agg, activation, n_layers, hidden
        self.dropout, self.hidden_relu, self.hidden_bn = float(dropout), bool(hidden_relu), bool(hidden_bn)
        self.device, self.drop_seed, self.precision = torch.device(device), int(drop_seed), precision
        self.stride = 1 + self.hidden_bn + self.hidden_relu
        self.emb_dim = hidden[-1] if hidden else hidden_dim
        shapes = [(f"layer{l + 1}.weight", (in_feats if l == 0 else hidden_dim, hidden_dim)) for l in range(n_layers)]
        shapes = [s for l in range(n_layers) for s in (shapes[l], (f"layer{l + 1}.bias", (hidden_dim, )))]
        self.lin, prev = [], hidden_dim
        for i, w in enumerate(hidden):
            li = f"encoder.{i * self.stride}"
            shapes += [(li + ".weight", (w, prev)), (li + ".bias", (w, ))]
            bn = f"encoder.{i * self.stride + 1}" if self.hidden_bn else None
            if bn:
                shapes += [(bn + ".weight", (w, )), (bn + ".bias", (w, ))]
            self.lin.append((li, bn))
            prev = w
        self.params = FlatParams(shapes, self.device)
        self.running = {bn + k: torch.zeros(self.params.shapes[bn + ".weight"], dtype=torch.float32, device=self.device)
                        for _, bn in self.lin if bn for k in (".running_mean", ".running_var")}
        self.num_batches_tracked = 0
        self.reset_parameters()
        self.step = 0
        self.z: Optional[torch.Tensor] = None
        self.losses: Optional[torch.Tensor] = None
        self._ones_buf: Optional[torch.Tensor] = None

    def reset_parameters(self, gen: Optional[torch.Generator] = None):
        """GraphConv: xavier_uniform weight, zero bias; nn.Linear: kaiming-uniform; BatchNorm1d: 1 / 0, running 0 / 1."""
        P = self.params.p
        for l in range(self.n_layers):
            w = torch.empty(P[f"layer{l + 1}.weight"].shape)
            _xavier_uniform_(w, gen)
            P[f"layer{l + 1}.weight"].copy_(w)
            P[f"layer{l + 1}.bias"].zero_()
        for li, bn in self.lin:
            w, b = torch.empty(P[li + ".weight"].shape), torch.empty(P[li + ".bias"].shape)
            _linear_init_(w, b, gen)
            P[li + ".weight"].copy_(w)
            P[li + ".bias"].copy_(b)
            if bn:
                P[bn + ".weight"].fill_(1.0)
                P[bn + ".bias"].zero_()
                self.running[bn + ".running_mean"].zero_()
                self.running[bn + ".running_var"].fill_(1.0)
        self.num_batches_tracked = 0

    # ---- state --------------------------------------------------------------------------------------------------------------
    def state_dict(self) -> Dict[str, torch.Tensor]:
        """The reference GCNAE's state_dict keys and shapes (layer weights [in, out], Linear weights [out, in])."""
        sd = {}
        for n in self.params.names:
            sd[n] = self.params.p[n].detach().clone()
            if n.endswith(".bias") and n[:-5] + ".running_mean" in self.running:
                for k in (".running_mean", ".running_var"):
                    sd[n[:-5] + k] = self.running[n[:-5] + k].clone()
                sd[n[:-5] + ".num_batches_tracked"] = torch.tensor(self.num_batches_tracked, dtype=torch.long)
        return sd

    def load_state_dict(self, sd):
        missing = [k for k in self.state_dict() if k not in sd]
        if missing:
            raise KeyError(f"state_dict lacks {missing}")
        for n in self.params.names:
            self.params.p[n].copy_(torch.as_tensor(sd[n], dtype=torch.float32))
        for k, v in self.running.items():
            v.copy_(torch.as_tensor(sd[k], dtype=torch.float32))
        for _, bn in self.lin:
            if bn:
                self.num_batches_tracked = int(sd[bn + ".num_batches_tracked"])

    def drop_key(self, step: int, pas: int, site: str) -> int:
        """Key of the dropout draw at ``site`` of forward ``pas`` (0: embedding, 1: loss) in mini-batch ``step``."""
        return (step * 2 + pas) * len(self.SITES) + self.SITES.index(site)

    # ---- one mini-batch -----------------------------------------------------------------------------------------------------
    def _ones(self, n: int) -> torch.Tensor:
        """[1, n] of ones (bias gradients are 1×n by n×out products): a view of one grow-only buffer."""
        if self._ones_buf is None or self._ones_buf.shape[1] < n:
            self._ones_buf = torch.ones(1, max(n, 256), dtype=torch.float32, device=self.device)
        return self._ones_buf[:, :n]

    def _conv(self, l: int, A, dst, deg, x, x_pos, pas: int, keep: dict):
        P, act = self.params.p, self.activation
        a = ops.graphsc_block_aggregate(A, dst, deg, x, self.agg, self.dropout, self.drop_seed,
                                        self.drop_key(self.step, pas, f"layer{l + 1}"), x_pos=x_pos)
        if act in ops.ACT:              # relu: in the GEMM epilogue; leaky_relu / gelu: their own pass over the pre-activation
            h = ops.gemm(a, P[f"layer{l + 1}.weight"], bias=P[f"layer{l + 1}.bias"], act=act, precision=self.precision)
        else:
            keep[f"pre{l}"] = ops.gemm(a, P[f"layer{l + 1}.weight"], bias=P[f"layer{l + 1}.bias"], precision=self.precision)
            h = ops.act(keep[f"pre{l}"], act)
        keep[f"agg{l}"], keep[f"h{l}"] = a, h
        return h

    def _forward(self, blk: dict, pas: int, keep: dict) -> torch.Tensor:
        A, X = blk["A"], blk["X"]
        if self.n_layers == 1:
            x = self._conv(0, A, blk["dst"], blk["deg"][0], X, None, pas, keep)
        else:
            h1 = self._conv(0, A, blk["src"], blk["deg"][0], X, None, pas, keep)
            x = self._conv(1, A, blk["dst"], blk["deg"][1], h1, blk["pos"], pas, keep)
        P = self.params.p
        for i, (li, bn) in enumerate(self.lin):
            keep[f"in{i}"] = x
            relu = "relu" if self.hidden_relu else None
            y = ops.gemm(x, P[li + ".weight"], transB=True, bias=P[li + ".bias"], act=None if bn else relu, precision=self.precision)
            if bn:
                keep[f"lin{i}"] = y
                y, sm, si = ops.batchnorm_fwd(y, P[bn + ".weight"], P[bn + ".bias"], self.running[bn + ".running_mean"],
                                              self.running[bn + ".running_var"], True, 0.1, 1e-5, act=relu)
                keep[f"bn{i}"] = (sm, si)
            keep[f"out{i}"] = y
            x = y
        return x

    def _backward(self, blk: dict, dz: torch.Tensor, keep: dict):
        P, G, pr = self.params.p, self.params.g, self.precision
        ones = self._ones(dz.shape[0])
        dx = dz
        for i in reversed(range(len(self.lin))):
            li, bn = self.lin[i]
            if bn:
                sm, si = keep[f"bn{i}"]
                dx, _, _ = ops.batchnorm_bwd(dx, keep[f"out{i}"], keep[f"lin{i}"], P[bn + ".weight"], sm, si,
                                             act="relu" if self.hidden_relu else None, dgamma=G[bn + ".weight"], dbeta=G[bn + ".bias"])
            elif self.hidden_relu:
                dx = ops.act_bwd(dx, "relu", y=keep[f"out{i}"])
            ops.gemm(dx, keep[f"in{i}"], transA=True, out=G[li + ".weight"], precision="fp32")
            ops.gemm(ones, dx, out=G[li + ".bias"].view(1, -1), precision="fp32")
            dx = ops.gemm(dx, P[li + ".weight"], precision=pr)
        for l in reversed(range(self.n_layers)):
            W = P[f"layer{l + 1}.weight"]
            a = keep[f"agg{l}"]
            dpre = ops.act_bwd(dx, self.activation, y=keep[f"h{l}"], x=keep.get(f"pre{l}"))
            ops.gemm(a, dpre, transA=True, out=G[f"layer{l + 1}.weight"], precision="fp32")
            ops.gemm(self._ones(a.shape[0]), dpre, out=G[f"layer{l + 1}.bias"].view(1, -1), precision="fp32")
            if l == 1:
                da = ops.gemm(dpre, W, transB=True, precision=pr)
                dx = ops.graphsc_block_aggregate(A=blk["A"], dst=blk["dst"], outdeg=blk["deg"][1], x=da, agg=self.agg, p=self.dropout,
                                                 seed=self.drop_seed, key=self.drop_key(self.step, 1, "layer2"), x_pos=blk["pos"],
                                                 transposed=True, out_rows=keep["agg0"].shape[0])

    def train_batch(self, blk: dict, lr: float, loss_out: torch.Tensor):
        """Both forwards, the loss into ``loss_out`` [1], the backward and one Adam step for the batch ``blk`` (see train_epoch)."""
        B = blk["dst"].numel()
        if self.hidden_bn and B == 1:
            raise ValueError(f"Expected more than 1 value per channel when training, got input size torch.Size([1, {self.hidden[0]}])")
        self._ones(max(B, blk["src"].numel() if blk["src"] is not None else 0))     # sized before the step: no allocation in it
        keep = {}
        z = self._forward(blk, 0, keep)
        ops.graphsc_scatter_rows(z, blk["dst"], self.z, offset=blk["cell_offset"])
        keep = {}
        z = self._forward(blk, 1, keep)
        _, dz = ops.graphsc_batch_decoder(z, self.DEC_P, self.drop_seed, self.drop_key(self.step, 1, "decoder"), loss=loss_out)
        self._backward(blk, dz, keep)
        self.params.adam_step(lr)
        if self.hidden_bn:
            self.num_batches_tracked += 2
        self.step += 1

    def train_epoch(self, graph: dict, train_ids, batch_size: int, lr: float) -> torch.Tensor:
        """One epoch of GraphSC.fit: the batch order is ``train_ids[torch.randperm(n_train)]`` on torch's default CPU generator
        (as dgl's DataLoader(shuffle=True) draws it), batches of ``batch_size`` with the short last one kept.  ``graph`` comes from
        :func:`prepare_graph`.  Returns the per-batch losses (device) and leaves the embeddings of this epoch in :attr:`z`
        [n_cells, d] (cell order)."""
        train_ids = torch.as_tensor(train_ids, dtype=torch.long)
        order = train_ids[torch.randperm(train_ids.numel())]
        self.last_order = order
        order_dev = order.to(torch.int32).pin_memory().to(self.device, non_blocking=True)
        n_cells = graph["n_cells"]
        if self.z is None or self.z.shape[0] != n_cells:
            self.z = torch.zeros(n_cells, self.emb_dim, dtype=torch.float32, device=self.device)
        nb = (order.numel() + batch_size - 1) // batch_size
        self.losses = torch.empty(nb, dtype=torch.float32, device=self.device)
        for b in range(nb):
            sl = slice(b * batch_size, (b + 1) * batch_size)
            self.train_batch(self.block(graph, order[sl], order_dev[sl]), lr, self.losses[b:b + 1])
        return self.losses

    def block(self, graph: dict, ids_host, ids_dev: torch.Tensor) -> dict:
        """The block of the mini-batch whose cells are the global node ids ``ids_host`` (host) / ``ids_dev`` (int32, device), as
        :meth:`train_batch` takes it: the destination list and its out-degrees, and for two layers the source list, each
        source's slot in it and layer 1's out-degrees.  ``graph`` comes from :func:`prepare_graph`; nothing here synchronises."""
        A = graph["A"]
        blk = dict(A=A, X=graph["X"], dst=ids_dev, cell_offset=graph["cell_offset"], src=None, pos=None)
        if self.n_layers == 1:
            blk["deg"] = [ops.graphsc_block_degrees(A, ids_dev)]
        else:
            indptr, ids = graph["indptr_host"], np.asarray(ids_host)
            cap = int(min(A.shape[0], (indptr[ids + 1] - indptr[ids]).sum()))       # Σ row lengths bounds the sources
            deg2, src, pos = ops.graphsc_block_degrees(A, ids_dev, src_cap=cap)
            blk.update(src=src, pos=pos, deg=[ops.graphsc_block_degrees(A, src), deg2])
        return blk


def prepare_graph(graph, device="cuda") -> dict:
    """The device view of a cell–gene graph (GraphLite with ndata 'features', 'feat_id' and edata 'weight'): the
    destination-indexed CSR with edge weights, the node features, the training (cell) node ids and the first cell's node id."""
    dev = torch.device(device)
    A, _ = graph.to(dev).csr_by_destination("weight")
    if A.vals is not None and A.vals.dtype != torch.float32:
        A = CSR(A.rowptr, A.colidx, A.vals.float().contiguous(), A.shape)
    feat_id = torch.as_tensor(graph.ndata["feat_id"]).cpu()
    train_ids = torch.nonzero(feat_id != -1).flatten()
    off = int(train_ids[0]) if train_ids.numel() else 0
    if not torch.equal(feat_id[train_ids].long(), torch.arange(train_ids.numel())) or not torch.equal(
            train_ids, torch.arange(off, off + train_ids.numel())):
        raise ValueError("expected the cell nodes to follow the gene nodes in cell order (CellFeatureGraph's layout)")
    X = torch.as_tensor(graph.ndata["features"]).to(dev, torch.float32).contiguous()
    return dict(A=A, X=X, indptr_host=A.rowptr.cpu().numpy().astype(np.int64), train_ids=train_ids, cell_offset=off,
                n_cells=train_ids.numel())
