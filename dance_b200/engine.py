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
