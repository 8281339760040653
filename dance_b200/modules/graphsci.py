"""GraphSCI on the H100-native kernels — host-side mirror of ``dance/modules/single_modality/imputation/graphsci.py``
(buildNetwork :37-45, activations :48-63, MultiplyLayer :66-87, AEModel :90-112, GNNModel :115-131, GraphSCI :134-560).

Model (one full-batch step = train forward → loss → eval forward for the validation loss → backward → Adam, :333-365):

* GNN over the gene graph (G nodes, node features = masked expression transposed, [G, N cells]) — four ``dgl.nn.GraphConv``
  (norm="both", the graph's edge weights are NOT passed, :126-129):  Ân = D_in^-1/2 A D_out^-1/2 from structural degrees;
  conv1 multiplies by W first (N > 256), the others aggregate first (in ≤ out).  Reference quirk kept: ``z_adj_log_std`` is
  produced by ``dec_mean`` as well (:129), ``dec_log_std`` never runs.  z_adj = mean + exp(log_std)·ε.
* AE over cells: h = ReLU(X·(z_adj·Wfᵀ) + b) (MultiplyLayer), two (Linear, BatchNorm, ReLU) encoder blocks, three
  (Linear, BatchNorm) heads with Sigmoid / clamp(softplus) / clamp(exp).
* loss = le·ZINB-NLL(masked) + la·norm·CE(z_adj, A; class weights) − ka·KL_adj + ke·KL_exp (get_loss :455-483; the reference
  moves every tensor to the CPU for this — here it is two fused kernels).

Randomness (dropout masks, ε) comes from a device ``torch.Generator`` seeded with ``seed``; tests inject ε explicitly and use
dropout = 0, which is how the fixtures were produced.

Two training schedules compute the same step.  The materialising one keeps every activation, keep-mask and loss gradient
(about 25 [cells, genes] fp32 matrices); the lean one keeps five (a scratch matrix, the multiply layer's output and the
three heads' pre-BatchNorm outputs, which the fused heads kernel overwrites with their gradients), draws its dropout masks
from a counter-based hash so the backward regenerates them instead of storing them, and evaluates in row chunks.
:func:`choose_schedule` picks one from the problem size and the device's memory (DESIGN §8); :data:`SCHEDULE` forces one.
"""
from __future__ import annotations

from pathlib import Path
from typing import Dict, Optional

import numpy as np
import scipy.sparse as sp
import torch

from .. import graphsci_ops, ops
from ..engine import FlatParams

H1 = H2 = 256
HEADS = ("dec_pi", "dec_disp", "dec_mean")
# dropout sites in the order the reference draws them: GNN (graphsci.py:118-121), then AE (:81, buildNetwork :40)
DROP_SITES = ("feat", "h1", "h2_mean", "h2_log_std", "X", "enc.1", "enc.5", "dec_pi", "dec_disp", "dec_mean")

# Training schedule: "auto" (choose_schedule), or "materialise" / "lean" to force one (tests and benchmarks; user code never
# needs it).
SCHEDULE = "auto"
# Rows per chunk of the lean schedule's evaluation forward (four [chunk, genes] fp32 buffers).
EVAL_CHUNK_ROWS = 32768

# Device memory of one train() step, in fp32 floats per cell (DESIGN §8): each schedule's own [cells, genes] matrices, those the
# caller holds (X, Xraw, the GNN features Xᵀ, and a byte mask as a quarter), and per cell the [cells, 256] conv1 weight, its
# gradient and two Adam moments plus about ten [cells, 256] encoder activations and gradients.
OWN_MATRICES = {"materialise": 25, "lean": 5}
CALLER_MATRICES = 3.25
ROW_FLOATS = 14 * H1
# share of the device's memory the materialising schedule may plan to use: the estimate leaves out allocator slack and the
# [genes, genes] matrices (at 200 000 × 3 000 it is 65.8 GiB, the measured peak 69.8 GiB; DESIGN §8)
HEADROOM = 0.85


def schedule_bytes(schedule: str, n_cells: int, n_genes: int) -> int:
    """Estimated device bytes of one train() step under ``schedule`` ("materialise" | "lean")."""
    return int(4 * n_cells * ((OWN_MATRICES[schedule] + CALLER_MATRICES) * n_genes + ROW_FLOATS))


def choose_schedule(n_cells: int, n_genes: int, device_bytes: int) -> str:
    """"materialise" while its estimate fits in HEADROOM of ``device_bytes``, else "lean"."""
    return "materialise" if schedule_bytes("materialise", n_cells, n_genes) <= HEADROOM * device_bytes else "lean"


def _t(x, device, dtype=torch.float32):
    if isinstance(x, torch.Tensor):
        return x.to(device=device, dtype=dtype).contiguous()
    return torch.as_tensor(np.ascontiguousarray(x)).to(device=device, dtype=dtype).contiguous()


class _BN:
    """Running statistics of one BatchNorm1d (affine parameters live in the flat bucket)."""

    def __init__(self, c, device):
        self.running_mean = torch.zeros(c, dtype=torch.float32, device=device)
        self.running_var = torch.ones(c, dtype=torch.float32, device=device)
        self.num_batches_tracked = 0


class GraphSCI:

    def __init__(self, num_cells, num_genes, dataset, dropout=0.1, gpu=0, seed=1, precision: Optional[str] = None,
                 save_path: Optional[str] = None):
        self.dataset, self.seed, self.dropout = dataset, seed, float(dropout)
        self.N, self.G = int(num_cells), int(num_genes)
        self.device = torch.device(f"cuda:{max(int(gpu), 0)}")            # the reference's gpu=-1 (CPU) has no counterpart here
        self.precision = precision
        self.save_path = Path(save_path) if save_path is not None else None
        N, G = self.N, self.G
        shapes = [("aemodel.mul_layer.bias", (G, )), ("aemodel.mul_layer.fc_layer.weight", (G, G)),
                  ("aemodel.enc.1.weight", (H1, G)), ("aemodel.enc.1.bias", (H1, )), ("aemodel.enc.2.weight", (H1, )), ("aemodel.enc.2.bias", (H1, )),
                  ("aemodel.enc.5.weight", (H2, H1)), ("aemodel.enc.5.bias", (H2, )), ("aemodel.enc.6.weight", (H2, )), ("aemodel.enc.6.bias", (H2, ))]
        for head in ("dec_pi", "dec_disp", "dec_mean"):
            shapes += [(f"aemodel.{head}.1.weight", (G, H2)), (f"aemodel.{head}.1.bias", (G, )), (f"aemodel.{head}.2.weight", (G, )),
                       (f"aemodel.{head}.2.bias", (G, ))]
        shapes += [("gnnmodel.conv1.weight", (N, H1)), ("gnnmodel.conv1.bias", (H1, )), ("gnnmodel.conv2.weight", (H1, H2)),
                   ("gnnmodel.conv2.bias", (H2, )), ("gnnmodel.dec_mean.weight", (H2, G)), ("gnnmodel.dec_mean.bias", (G, ))]
        self.params = FlatParams(shapes, self.device)
        self.bn = {k: _BN(c, self.device) for k, c in (("enc.2", H1), ("enc.6", H2), ("dec_pi.2", G), ("dec_disp.2", G), ("dec_mean.2", G))}
        self.unused: Dict[str, torch.Tensor] = {}
        self._init_params()
        self.gen = torch.Generator(device=self.device).manual_seed(int(seed))
        self.drop_seed = int(seed) & 0xFFFFFFFF         # the lean schedule's dropout draws: keep(drop_seed, drop_key(site), r, c)
        self.drop_step = 0                               # lean training steps taken: part of every dropout key
        self.best_state = None
        self.train_loss = self.valid_loss = self.loss_adj = self.loss_exp = self.kl = None

    # ---- parameters -------------------------------------------------------------------------
    def _init_params(self):
        g = torch.Generator().manual_seed(int(self.seed))
        P = self.params.p

        def linear_(w, b):      # nn.Linear.reset_parameters
            bound = 1.0 / w.shape[1]**0.5
            w.copy_((torch.rand(w.shape, generator=g) * 2 - 1) * bound)
            if b is not None:
                b.copy_((torch.rand(b.shape, generator=g) * 2 - 1) * bound)

        def glorot_(w, b):      # dgl GraphConv.reset_parameters: xavier_uniform_ weight, zero bias
            a = (6.0 / (w.shape[0] + w.shape[1]))**0.5
            w.copy_((torch.rand(w.shape, generator=g) * 2 - 1) * a)
            b.zero_()

        P["aemodel.mul_layer.bias"].zero_()
        linear_(P["aemodel.mul_layer.fc_layer.weight"], None)
        linear_(P["aemodel.enc.1.weight"], P["aemodel.enc.1.bias"])
        linear_(P["aemodel.enc.5.weight"], P["aemodel.enc.5.bias"])
        for k in ("enc.2", "enc.6"):
            P[f"aemodel.{k}.weight"].fill_(1.0)
            P[f"aemodel.{k}.bias"].zero_()
        for head in ("dec_pi", "dec_disp", "dec_mean"):
            linear_(P[f"aemodel.{head}.1.weight"], P[f"aemodel.{head}.1.bias"])
            P[f"aemodel.{head}.2.weight"].fill_(1.0)
            P[f"aemodel.{head}.2.bias"].zero_()
        glorot_(P["gnnmodel.conv1.weight"], P["gnnmodel.conv1.bias"])
        glorot_(P["gnnmodel.conv2.weight"], P["gnnmodel.conv2.bias"])
        glorot_(P["gnnmodel.dec_mean.weight"], P["gnnmodel.dec_mean.bias"])
        w = torch.empty(H2, self.G)
        glorot_(w, torch.empty(self.G))
        self.unused = {"dec_log_std.weight": w, "dec_log_std.bias": torch.zeros(self.G)}     # never used by forward (:129)

    def state_dict(self) -> Dict[str, Dict[str, torch.Tensor]]:
        ae = {k[len("aemodel."):]: v.detach().clone() for k, v in self.params.p.items() if k.startswith("aemodel.")}
        for k, b in self.bn.items():
            ae[f"{k}.running_mean"], ae[f"{k}.running_var"] = b.running_mean.clone(), b.running_var.clone()
            ae[f"{k}.num_batches_tracked"] = torch.tensor(b.num_batches_tracked)
        gnn = {k[len("gnnmodel."):]: v.detach().clone() for k, v in self.params.p.items() if k.startswith("gnnmodel.")}
        gnn.update({k: v.clone() for k, v in self.unused.items()})
        return {"aemodel": ae, "gnnmodel": gnn}

    def load_state_dict(self, state):
        for scope in ("aemodel", "gnnmodel"):
            for k, v in state[scope].items():
                full = f"{scope}.{k}"
                v = torch.as_tensor(np.asarray(v.cpu() if isinstance(v, torch.Tensor) else v))
                if full in self.params.p:
                    self.params.p[full].copy_(v.to(torch.float32))
                elif k.endswith("running_mean") or k.endswith("running_var"):
                    getattr(self.bn[k.rsplit(".", 1)[0]], k.rsplit(".", 1)[1]).copy_(v.to(torch.float32))
                elif k.endswith("num_batches_tracked"):
                    self.bn[k.rsplit(".", 1)[0]].num_batches_tracked = int(v)
                elif k in self.unused:
                    self.unused[k] = v.to(torch.float32).clone()

    # ---- graph ------------------------------------------------------------------------------
    def _bind_graph(self, graph):
        if getattr(self, "_graph_key", None) == id(graph):
            return
        u, v = graph.edges()
        u, v = np.asarray(u.cpu()).astype(np.int64), np.asarray(v.cpu()).astype(np.int64)
        G = graph.num_nodes()
        if G != self.G:
            raise ValueError(f"graph has {G} nodes, model was built for {self.G} genes")
        A = sp.csr_matrix((np.ones(len(u), np.float32), (u, v)), shape=(G, G))          # adj[u, v] = 1 (:256-259)
        outdeg = np.asarray(A.sum(1)).ravel().clip(min=1)
        indeg = np.asarray(A.sum(0)).ravel().clip(min=1)
        if (np.asarray(A.sum(0)).ravel() == 0).any():
            raise RuntimeError("There are 0-in-degree nodes in the graph (dgl GraphConv raises the same error)")
        # aggregation at dst over in-edges: rows = dst, cols = src, value = outdeg(src)^-1/2 · indeg(dst)^-1/2
        T = A.T.tocsr()
        T.sort_indices()
        rows = np.repeat(np.arange(G), np.diff(T.indptr))
        T.data = (outdeg[T.indices].astype(np.float32)**-0.5 * indeg[rows].astype(np.float32)**-0.5).astype(np.float32)
        self.An = ops.CSR.from_scipy(T, device=self.device)
        self.AnT, _ = ops.csr_transpose(self.An)
        dense = torch.from_numpy(A.toarray()).to(self.device)
        self.adj = dense                                                               # unit adjacency, the CE target
        rs = dense.sum(1)
        self.pos_weight = ((G * G - rs) / rs).contiguous()                             # class weights (:455)
        self.norm_adj = G * G / float((G * G - float(dense.sum().item())) * 2)         # (:456-457)
        self._graph_key = id(graph)
        self._graph = graph

    # ---- schedule ---------------------------------------------------------------------------
    def schedule(self) -> str:
        """The training schedule train() / evaluate() run: :data:`SCHEDULE` unless "auto", else :func:`choose_schedule`."""
        if SCHEDULE != "auto":
            if SCHEDULE not in OWN_MATRICES:
                raise ValueError(f"graphsci.SCHEDULE must be 'auto', 'materialise' or 'lean', got {SCHEDULE!r}")
            return SCHEDULE
        return choose_schedule(self.N, self.G, torch.cuda.get_device_properties(self.device).total_memory)

    def drop_key(self, site: str, step: Optional[int] = None) -> int:
        """Key of the lean schedule's dropout draw at ``site`` (one of :data:`DROP_SITES`) in training step ``step`` (default:
        the step train() runs next).  ``ops.dropout(ones, p, model.drop_seed, key)`` reproduces the mask."""
        s = self.drop_step if step is None else step
        return s * len(DROP_SITES) + DROP_SITES.index(site)

    # ---- forward pieces ---------------------------------------------------------------------
    def _drop(self, x, training):
        if not training or self.dropout == 0.0:
            return x, None
        keep = (torch.rand(x.shape, device=self.device, generator=self.gen) >= self.dropout).to(torch.float32) / (1.0 - self.dropout)
        return x * keep, keep

    def _gnn_forward(self, feat, training, eps=None):
        P = self.params.p
        pr = self.precision
        f_d, m0 = self._drop(feat, training)
        h1 = ops.spmm(self.An, ops.gemm(f_d, P["gnnmodel.conv1.weight"], precision=pr), act="tanh", bias=P["gnnmodel.conv1.bias"])
        h1_d, m1 = self._drop(h1, training)
        S1 = ops.spmm(self.An, h1_d)
        h2 = ops.gemm(S1, P["gnnmodel.conv2.weight"], bias=P["gnnmodel.conv2.bias"], act="relu", precision=pr)
        h2_a, m2a = self._drop(h2, training)
        S2a = ops.spmm(self.An, h2_a)
        mu = ops.gemm(S2a, P["gnnmodel.dec_mean.weight"], bias=P["gnnmodel.dec_mean.bias"], precision=pr)
        if training and self.dropout > 0.0:
            h2_b, m2b = self._drop(h2, training)
            S2b = ops.spmm(self.An, h2_b)
            ls = ops.gemm(S2b, P["gnnmodel.dec_mean.weight"], bias=P["gnnmodel.dec_mean.bias"], precision=pr)     # dec_mean again (:129)
        else:
            m2b, S2b, ls = m2a, S2a, mu
        if eps is None:
            eps = torch.randn(mu.shape, device=self.device, generator=self.gen)
        else:
            eps = _t(eps, self.device)
        z = ops.adj_sample(mu, ls, eps)
        return z, ls, mu, dict(f_d=f_d, m0=m0, h1=h1, m1=m1, S1=S1, h2=h2, m2a=m2a, m2b=m2b, S2a=S2a, S2b=S2b, eps=eps, shared=(ls is mu))

    def _ae_forward(self, X, z_adj, training):
        P = self.params.p
        pr = self.precision
        zf = ops.gemm(z_adj, P["aemodel.mul_layer.fc_layer.weight"], transB=True, precision=pr)
        X_d, mx = self._drop(X, training)
        h0 = ops.gemm(X_d, zf, bias=P["aemodel.mul_layer.bias"], act="relu", precision=pr)
        c = dict(zf=zf, X_d=X_d, mx=mx, h0=h0)
        h, pre_key = h0, "h0"
        for blk, lin, bn in (("e1", "enc.1", "enc.2"), ("e2", "enc.5", "enc.6")):
            h_d, m = self._drop(h, training)
            pre = ops.gemm(h_d, P[f"aemodel.{lin}.weight"], transB=True, bias=P[f"aemodel.{lin}.bias"], precision=pr)
            out, sm, si = self._bn_fwd(bn, pre, training, act="relu")
            c[blk] = dict(inp=h_d, m=m, pre=pre, out=out, sm=sm, si=si)
            h = out
        heads = {}
        for head in ("dec_pi", "dec_disp", "dec_mean"):
            h_d, m = self._drop(h, training)
            pre = ops.gemm(h_d, P[f"aemodel.{head}.1.weight"], transB=True, bias=P[f"aemodel.{head}.1.bias"], precision=pr)
            out, sm, si = self._bn_fwd(f"{head}.2", pre, training, act=None)
            heads[head] = dict(inp=h_d, m=m, pre=pre, out=out, sm=sm, si=si)
        c["heads"] = heads
        return heads["dec_pi"]["out"], heads["dec_disp"]["out"], heads["dec_mean"]["out"], c

    def _bn_fwd(self, key, pre, training, act):
        b = self.bn[key]
        out, sm, si = ops.batchnorm_fwd(pre, self.params.p[f"aemodel.{key}.weight"], self.params.p[f"aemodel.{key}.bias"], b.running_mean,
                                        b.running_var, training, 0.1, 1e-5, act=act)
        if training:
            b.num_batches_tracked += 1
        return out, sm, si

    def _losses(self, acc3, acc2, le, la, ke, ka):
        """Scalars from the two accumulator vectors (host floats; one small D2H each)."""
        nll, mse, cnt = (float(v) for v in acc3.cpu())
        ce, kls = (float(v) for v in acc2.cpu())
        G, N = self.G, self.N
        loss_adj = la * self.norm_adj * (ce / G)
        loss_exp = le * nll / cnt if cnt else float("nan")
        kl_adj = (0.5 / N) * (kls / G)
        kl_exp = 0.5 / G * (mse / cnt) if cnt else float("nan")
        kl = ka * kl_adj - ke * kl_exp
        log_lik = loss_exp + loss_adj
        return loss_adj, loss_exp, log_lik, kl, log_lik - kl

    def maskdata(self, X, mask):
        Xd = _t(X, self.device)
        return Xd * _t(mask, self.device, torch.bool).to(torch.float32)

    # ---- training ---------------------------------------------------------------------------
    def fit(self, train_data, train_data_raw, graph, mask=None, le=1, la=1, ke=1, ka=1, n_epochs=100, lr=1e-3, weight_decay=1e-5,
            train_idx=None, eps_sequence=None, verbose=False):
        """Mirror of ``GraphSCI.fit`` (:210-331).  ``eps_sequence``: optional iterable of [G, G] noise arrays consumed in the
        order train-forward, eval-forward, train-forward, … (test hook replacing ``torch.normal``'s generator)."""
        self._bind_graph(graph)
        X = _t(train_data, self.device)
        Xraw = _t(train_data_raw, self.device)
        n = X.shape[0]
        rng = np.random.default_rng(self.seed)
        if train_idx is None:
            train_idx = range(n)
        if mask is not None:
            mask = np.asarray(mask.cpu() if isinstance(mask, torch.Tensor) else mask).astype(bool)
            X_masked = self.maskdata(X, mask)
            X = None          # drop this reference to the unmasked copy; a tensor the caller passed stays alive through theirs
            train_mask = np.copy(mask)
            test_idx = np.setdiff1d(np.arange(n), np.asarray(list(train_idx)))
            train_mask[test_idx] = False
            valid_mask = ~mask
            valid_mask[test_idx] = False
        else:
            X_masked = X
            perm = rng.permutation(np.asarray(list(train_idx)))
            tr, va = perm[:int(len(perm) * 0.9)], perm[int(len(perm) * 0.9):]
            train_mask = np.zeros(tuple(X_masked.shape), dtype=bool)
            train_mask[tr] = True
            valid_mask = np.zeros(tuple(X_masked.shape), dtype=bool)
            valid_mask[va] = True
        self.train_data_masked = X_masked
        self._feat = X_masked.t().contiguous()                                         # graph.ndata["feat"] = masked.T (:270)
        if mask is not None and hasattr(graph, "ndata"):
            graph.ndata["feat"] = self._feat                                           # the reference mutates the caller's graph too
        n_counts = Xraw.sum(1)
        self.size_factors = (n_counts / torch.median(n_counts)).contiguous()
        self.weight_decay = weight_decay
        self.lr = lr
        tm = torch.from_numpy(train_mask).to(self.device).view(torch.uint8)
        vm = torch.from_numpy(valid_mask).to(self.device).view(torch.uint8)
        eps_it = iter(eps_sequence) if eps_sequence is not None else None
        nxt = (lambda: _t(next(eps_it), self.device)) if eps_it is not None else (lambda: None)
        self.params.step = 0
        self.params.exp_avg.zero_()
        self.params.exp_avg_sq.zero_()
        self.best_state = self.state_dict()
        min_valid = None
        for epoch in range(n_epochs):
            self.train(X_masked, Xraw, graph, tm, vm, le, la, ke, ka, eps_train=nxt(), eps_eval=nxt())
            if not epoch:
                min_valid = self.valid_loss
            elif min_valid >= self.valid_loss:
                min_valid = self.valid_loss
                self.save_model()
            if verbose:
                print(f"[Epoch{epoch}], train_loss {self.train_loss:.6f}, adj_loss {self.loss_adj:.6f}, express_loss {self.loss_exp:.6f}, "
                      f"kl_loss {abs(self.kl):.6f}, valid_loss {self.valid_loss:.6f}")
        return self

    def train(self, train_data, train_data_raw, graph, train_mask, valid_mask, le=1, la=1, ke=1, ka=1, eps_train=None, eps_eval=None):
        if self.schedule() == "lean":
            return self._train_lean(train_data, train_data_raw, graph, train_mask, valid_mask, le, la, ke, ka, eps_train, eps_eval)
        self._bind_graph(graph)
        X, Xraw = train_data, train_data_raw
        G, N = self.G, self.N
        P, Gd = self.params.p, self.params.g
        pr = self.precision
        z, ls, mu, gc = self._gnn_forward(self._graph_feat(graph), True, eps_train)
        a_pi, b_disp, c_mean, ac = self._ae_forward(X, z, True)
        acc3, (d_a, d_b, d_c), _ = ops.zinb_loss_grad(a_pi, b_disp, c_mean, Xraw, self.size_factors, train_mask, float(le), float(ke))
        acc2, dz_ce = ops.adj_loss_grad(z, mu, ls, self.adj, self.pos_weight, coef_ce=float(la) * self.norm_adj / G)
        self.loss_adj, self.loss_exp, self.log_lik, self.kl, self.train_loss = self._losses(acc3, acc2, le, la, ke, ka)
        vloss, _, _ = self.evaluate(X, Xraw, graph, valid_mask, le, la, ke, ka, eps=eps_eval)
        self.valid_loss = vloss

        # ---- backward: AE ----
        e2 = ac["e2"]
        de2 = None
        for head, dpre_act in (("dec_pi", d_a), ("dec_disp", d_b), ("dec_mean", d_c)):
            hd = ac["heads"][head]
            dpre, Gd[f"aemodel.{head}.2.weight"], Gd[f"aemodel.{head}.2.bias"] = self._bn_bwd(dpre_act, None, hd, f"{head}.2", None)
            ops.gemm(dpre, hd["inp"], transA=True, out=Gd[f"aemodel.{head}.1.weight"], precision=pr)
            ops.colsum(dpre, out=Gd[f"aemodel.{head}.1.bias"])
            dinp = ops.gemm(dpre, P[f"aemodel.{head}.1.weight"], precision=pr)
            if hd["m"] is not None:
                dinp = dinp * hd["m"]
            de2 = dinp if de2 is None else de2.add_(dinp)
        dh = de2
        for blk, lin, bn in (("e2", "enc.5", "enc.6"), ("e1", "enc.1", "enc.2")):
            bd = ac[blk]
            dpre, Gd[f"aemodel.{bn}.weight"], Gd[f"aemodel.{bn}.bias"] = self._bn_bwd(dh, bd["out"], bd, bn, "relu")
            ops.gemm(dpre, bd["inp"], transA=True, out=Gd[f"aemodel.{lin}.weight"], precision=pr)
            ops.colsum(dpre, out=Gd[f"aemodel.{lin}.bias"])
            dh = ops.gemm(dpre, P[f"aemodel.{lin}.weight"], precision=pr)          # gradient w.r.t. the block's (dropped-out) input
            if bd["m"] is not None:
                dh = dh * bd["m"]
        dpre0 = ops.act_bwd(dh, "relu", y=ac["h0"])                                    # ReLU of the multiply layer
        ops.colsum(dpre0, out=Gd["aemodel.mul_layer.bias"])
        dzf = ops.gemm(ac["X_d"], dpre0, transA=True, precision=pr)                       # [G, G]
        ops.gemm(dzf, z, transA=True, out=Gd["aemodel.mul_layer.fc_layer.weight"], precision=pr)
        dz = ops.gemm(dzf, P["aemodel.mul_layer.fc_layer.weight"], precision=pr)
        dz.add_(dz_ce)

        # ---- backward: GNN ----
        dmu, dls = ops.adj_reparam_bwd(dz, mu, ls, gc["eps"], coef_kl=-float(ka) * 0.5 / (N * G))
        Wm = P["gnnmodel.dec_mean.weight"]
        if gc["shared"]:
            dmu.add_(dls)
            ops.gemm(gc["S2a"], dmu, transA=True, out=Gd["gnnmodel.dec_mean.weight"], precision=pr)
            ops.colsum(dmu, out=Gd["gnnmodel.dec_mean.bias"])
            dh2 = ops.spmm(self.AnT, ops.gemm(dmu, Wm, transB=True, precision=pr))
            if gc["m2a"] is not None:
                dh2 = dh2 * gc["m2a"]
        else:
            ops.gemm(gc["S2a"], dmu, transA=True, out=Gd["gnnmodel.dec_mean.weight"], precision=pr)
            ops.gemm(gc["S2b"], dls, transA=True, out=Gd["gnnmodel.dec_mean.weight"], accumulate=True, precision=pr)
            ops.colsum(dmu, out=Gd["gnnmodel.dec_mean.bias"])
            ops.colsum(dls, out=Gd["gnnmodel.dec_mean.bias"], accumulate=True)
            dh2 = ops.spmm(self.AnT, ops.gemm(dmu, Wm, transB=True, precision=pr)) * gc["m2a"]
            dh2.add_(ops.spmm(self.AnT, ops.gemm(dls, Wm, transB=True, precision=pr)) * gc["m2b"])
        dpre2 = ops.act_bwd(dh2, "relu", y=gc["h2"])
        ops.gemm(gc["S1"], dpre2, transA=True, out=Gd["gnnmodel.conv2.weight"], precision=pr)
        ops.colsum(dpre2, out=Gd["gnnmodel.conv2.bias"])
        dh1 = ops.spmm(self.AnT, ops.gemm(dpre2, P["gnnmodel.conv2.weight"], transB=True, precision=pr))
        if gc["m1"] is not None:
            dh1 = dh1 * gc["m1"]
        dpre1 = ops.act_bwd(dh1, "tanh", y=gc["h1"])
        ops.colsum(dpre1, out=Gd["gnnmodel.conv1.bias"])
        dP = ops.spmm(self.AnT, dpre1)
        ops.gemm(gc["f_d"], dP, transA=True, out=Gd["gnnmodel.conv1.weight"], precision=pr)
        self.params.adam_step(self.lr, weight_decay=self.weight_decay)
        return self.train_loss

    def _bn_bwd(self, dY, Y, blk, key, act):
        dX, dg, db = ops.batchnorm_bwd(dY, Y, blk["pre"], self.params.p[f"aemodel.{key}.weight"], blk["sm"], blk["si"], act=act,
                                       training=True, dgamma=self.params.g[f"aemodel.{key}.weight"], dbeta=self.params.g[f"aemodel.{key}.bias"])
        return dX, dg, db

    def evaluate(self, features, features_raw, graph, mask=None, le=1, la=1, ke=1, ka=1, eps=None):
        """Eval-mode forward + loss (:367-409); returns (loss, z_adj, z_exp)."""
        self._bind_graph(graph)
        X, Xraw = _t(features, self.device), _t(features_raw, self.device)
        if mask is not None and not isinstance(mask, torch.Tensor):
            mask = torch.from_numpy(np.asarray(mask).astype(bool)).to(self.device).view(torch.uint8)
        feat = self._graph_feat(graph)
        if self.schedule() == "lean":
            return self._evaluate_lean(X, Xraw, feat, mask, le, la, ke, ka, eps)
        z, ls, mu, _ = self._gnn_forward(feat, False, eps)
        a_pi, b_disp, c_mean, _ = self._ae_forward(X, z, False)
        acc3, _, (mean, _, _) = ops.zinb_loss_grad(a_pi, b_disp, c_mean, Xraw, self.size_factors, mask, float(le), float(ke), want_grad=False,
                                                   want_outputs=True)
        acc2, _ = ops.adj_loss_grad(z, mu, ls, self.adj, self.pos_weight, want_grad=False)
        *_, loss = self._losses(acc3, acc2, le, la, ke, ka)
        z_exp = mean * self.size_factors.view(-1, 1)
        return loss, z, z_exp

    # ---- the lean schedule --------------------------------------------------------------------
    def _train_lean(self, X, Xraw, graph, train_mask, valid_mask, le, la, ke, ka, eps_train, eps_eval):
        """One train() step keeping five [cells, genes] matrices: ``scratch`` (f_d [G, N] in the GNN forward, then X_d [N, G]
        up to the dzf product, then f_d again, regenerated, for the conv1 weight gradient), ``h_d`` (the multiply layer's ReLU
        output with the enc.1 input dropout applied in place) and the heads' ``pre`` (overwritten by their gradients; the first
        then holds the multiply layer's gradient).  Dropout masks are hash draws (see :meth:`drop_key`), applied to the
        gradients by drawing them again."""
        self._bind_graph(graph)
        G, N = self.G, self.N
        P, Gd = self.params.p, self.params.g
        pr, p = self.precision, self.dropout
        drop = p > 0.0
        keys = {site: self.drop_key(site) for site in DROP_SITES}

        def dr(x, site, out=None):
            return ops.dropout(x, p, self.drop_seed, keys[site], out=out) if drop else x

        feat = self._graph_feat(graph)
        scratch = torch.empty(N * G, dtype=torch.float32, device=self.device) if drop else None

        # ---- GNN forward ----
        f_d = dr(feat, "feat", out=scratch.view(G, N) if drop else None)
        h1 = ops.spmm(self.An, ops.gemm(f_d, P["gnnmodel.conv1.weight"], precision=pr), act="tanh", bias=P["gnnmodel.conv1.bias"])
        del f_d
        S1 = ops.spmm(self.An, dr(h1, "h1"))
        h2 = ops.gemm(S1, P["gnnmodel.conv2.weight"], bias=P["gnnmodel.conv2.bias"], act="relu", precision=pr)
        Wm, bm = P["gnnmodel.dec_mean.weight"], P["gnnmodel.dec_mean.bias"]
        S2a = ops.spmm(self.An, dr(h2, "h2_mean"))
        mu = ops.gemm(S2a, Wm, bias=bm, precision=pr)
        if drop:
            S2b = ops.spmm(self.An, dr(h2, "h2_log_std"))
            ls = ops.gemm(S2b, Wm, bias=bm, precision=pr)                           # dec_mean again (:129)
        else:
            S2b, ls = S2a, mu
        eps = torch.randn(mu.shape, device=self.device, generator=self.gen) if eps_train is None else _t(eps_train, self.device)
        z = ops.adj_sample(mu, ls, eps)

        # ---- AE forward ----
        zf = ops.gemm(z, P["aemodel.mul_layer.fc_layer.weight"], transB=True, precision=pr)
        X_d = dr(X, "X", out=scratch.view(N, G) if drop else None)
        h_d = ops.gemm(X_d, zf, bias=P["aemodel.mul_layer.bias"], act="relu", precision=pr)
        if drop:
            dr(h_d, "enc.1", out=h_d)
        pre1 = ops.gemm(h_d, P["aemodel.enc.1.weight"], transB=True, bias=P["aemodel.enc.1.bias"], precision=pr)
        out1, sm1, si1 = self._bn_fwd("enc.2", pre1, True, act="relu")
        in2 = dr(out1, "enc.5")
        pre2 = ops.gemm(in2, P["aemodel.enc.5.weight"], transB=True, bias=P["aemodel.enc.5.bias"], precision=pr)
        out2, sm2, si2 = self._bn_fwd("enc.6", pre2, True, act="relu")
        pre = [ops.gemm(dr(out2, h), P[f"aemodel.{h}.1.weight"], transB=True, bias=P[f"aemodel.{h}.1.bias"], precision=pr) for h in HEADS]
        mean3 = torch.empty((3, G), dtype=torch.float32, device=self.device)
        invstd3 = torch.empty_like(mean3)
        for k, h in enumerate(HEADS):
            b = self.bn[f"{h}.2"]
            graphsci_ops.batchnorm_stats(pre[k], b.running_mean, b.running_var, True, 0.1, 1e-5, save_mean=mean3[k], save_invstd=invstd3[k])
            b.num_batches_tracked += 1
        gamma3, beta3 = self._head_affine()
        # loss, and each pre overwritten by its gradient through the BatchNorm
        acc3, dgamma3, dbeta3 = graphsci_ops.heads_train(pre, gamma3, beta3, mean3, invstd3, Xraw, self.size_factors, train_mask,
                                                         float(le), float(ke))
        for k, h in enumerate(HEADS):
            Gd[f"aemodel.{h}.2.weight"].copy_(dgamma3[k])
            Gd[f"aemodel.{h}.2.bias"].copy_(dbeta3[k])
        acc2, dz_ce = ops.adj_loss_grad(z, mu, ls, self.adj, self.pos_weight, coef_ce=float(la) * self.norm_adj / G)
        self.loss_adj, self.loss_exp, self.log_lik, self.kl, self.train_loss = self._losses(acc3, acc2, le, la, ke, ka)
        self.valid_loss = self._evaluate_lean(X, Xraw, feat, valid_mask, le, la, ke, ka, eps_eval, want_z_exp=False)[0]

        # ---- backward: AE ----
        de2 = None
        for k, h in enumerate(HEADS):
            dpre = pre[k]
            ops.gemm(dpre, dr(out2, h), transA=True, out=Gd[f"aemodel.{h}.1.weight"], precision=pr)
            ops.colsum(dpre, out=Gd[f"aemodel.{h}.1.bias"])
            dinp = ops.gemm(dpre, P[f"aemodel.{h}.1.weight"], precision=pr)
            dr(dinp, h, out=dinp)
            de2 = dinp if de2 is None else de2.add_(dinp)
        buf = pre[0]
        del pre, dpre
        dpre, Gd["aemodel.enc.6.weight"], Gd["aemodel.enc.6.bias"] = self._bn_bwd(de2, out2, dict(pre=pre2, sm=sm2, si=si2), "enc.6", "relu")
        ops.gemm(dpre, in2, transA=True, out=Gd["aemodel.enc.5.weight"], precision=pr)
        ops.colsum(dpre, out=Gd["aemodel.enc.5.bias"])
        dh = ops.gemm(dpre, P["aemodel.enc.5.weight"], precision=pr)
        dr(dh, "enc.5", out=dh)
        dpre, Gd["aemodel.enc.2.weight"], Gd["aemodel.enc.2.bias"] = self._bn_bwd(dh, out1, dict(pre=pre1, sm=sm1, si=si1), "enc.2", "relu")
        ops.gemm(dpre, h_d, transA=True, out=Gd["aemodel.enc.1.weight"], precision=pr)
        ops.colsum(dpre, out=Gd["aemodel.enc.1.bias"])
        dpre0 = ops.gemm(dpre, P["aemodel.enc.1.weight"], out=buf, precision=pr)       # [N, G] in a freed head buffer
        dr(dpre0, "enc.1", out=dpre0)
        ops.act_bwd(dpre0, "relu", y=h_d, out=dpre0)      # h_d > 0 exactly where h0 > 0 and the element was kept
        del h_d
        ops.colsum(dpre0, out=Gd["aemodel.mul_layer.bias"])
        dzf = ops.gemm(X_d, dpre0, transA=True, precision=pr)                            # [G, G]
        del X_d, dpre0, buf
        ops.gemm(dzf, z, transA=True, out=Gd["aemodel.mul_layer.fc_layer.weight"], precision=pr)
        dz = ops.gemm(dzf, P["aemodel.mul_layer.fc_layer.weight"], precision=pr)
        dz.add_(dz_ce)

        # ---- backward: GNN ----
        dmu, dls = ops.adj_reparam_bwd(dz, mu, ls, eps, coef_kl=-float(ka) * 0.5 / (N * G))
        if not drop:
            dmu.add_(dls)
            ops.gemm(S2a, dmu, transA=True, out=Gd["gnnmodel.dec_mean.weight"], precision=pr)
            ops.colsum(dmu, out=Gd["gnnmodel.dec_mean.bias"])
            dh2 = ops.spmm(self.AnT, ops.gemm(dmu, Wm, transB=True, precision=pr))
        else:
            ops.gemm(S2a, dmu, transA=True, out=Gd["gnnmodel.dec_mean.weight"], precision=pr)
            ops.gemm(S2b, dls, transA=True, out=Gd["gnnmodel.dec_mean.weight"], accumulate=True, precision=pr)
            ops.colsum(dmu, out=Gd["gnnmodel.dec_mean.bias"])
            ops.colsum(dls, out=Gd["gnnmodel.dec_mean.bias"], accumulate=True)
            dh2 = ops.spmm(self.AnT, ops.gemm(dmu, Wm, transB=True, precision=pr))
            dr(dh2, "h2_mean", out=dh2)
            dh2.add_(dr(ops.spmm(self.AnT, ops.gemm(dls, Wm, transB=True, precision=pr)), "h2_log_std"))
        dpre2 = ops.act_bwd(dh2, "relu", y=h2)
        ops.gemm(S1, dpre2, transA=True, out=Gd["gnnmodel.conv2.weight"], precision=pr)
        ops.colsum(dpre2, out=Gd["gnnmodel.conv2.bias"])
        dh1 = ops.spmm(self.AnT, ops.gemm(dpre2, P["gnnmodel.conv2.weight"], transB=True, precision=pr))
        dr(dh1, "h1", out=dh1)
        dpre1 = ops.act_bwd(dh1, "tanh", y=h1)
        ops.colsum(dpre1, out=Gd["gnnmodel.conv1.bias"])
        dP = ops.spmm(self.AnT, dpre1)
        f_d = dr(feat, "feat", out=scratch.view(G, N) if drop else None)                 # regenerated with the same key
        ops.gemm(f_d, dP, transA=True, out=Gd["gnnmodel.conv1.weight"], precision=pr)
        del f_d, scratch
        self.drop_step += 1
        self.params.adam_step(self.lr, weight_decay=self.weight_decay)
        return self.train_loss

    def _head_affine(self):
        """The heads' BatchNorm γ and β packed [3, G] (order of :data:`HEADS`), as the fused heads kernels take them."""
        P = self.params.p
        return (torch.stack([P[f"aemodel.{h}.2.weight"] for h in HEADS]), torch.stack([P[f"aemodel.{h}.2.bias"] for h in HEADS]))

    def _evaluate_lean(self, X, Xraw, feat, mask, le, la, ke, ka, eps, want_z_exp=True):
        """Eval-mode forward + loss in row chunks of :data:`EVAL_CHUNK_ROWS` (running-statistics BatchNorm, no dropout, so rows
        are independent).  Only z_exp (already times the size factors) is [cells, genes]; returns (loss, z_adj, z_exp | None)."""
        P, pr, G = self.params.p, self.precision, self.G
        z, ls, mu, _ = self._gnn_forward(feat, False, eps)
        zf = ops.gemm(z, P["aemodel.mul_layer.fc_layer.weight"], transB=True, precision=pr)
        mean3 = torch.empty((3, G), dtype=torch.float32, device=self.device)
        invstd3 = torch.empty_like(mean3)
        for k, h in enumerate(HEADS):
            b = self.bn[f"{h}.2"]
            graphsci_ops.batchnorm_stats(None, b.running_mean, b.running_var, False, 0.1, 1e-5, save_mean=mean3[k], save_invstd=invstd3[k])
        gamma3, beta3 = self._head_affine()
        n = X.shape[0]
        rows = max(1, min(int(EVAL_CHUNK_ROWS), n))
        z_exp = torch.empty((n, G), dtype=torch.float32, device=self.device) if want_z_exp else None
        h0 = torch.empty((rows, G), dtype=torch.float32, device=self.device)
        pre = [torch.empty_like(h0) for _ in HEADS]
        acc3 = None
        for r0 in range(0, n, rows):
            r1 = min(n, r0 + rows)
            m = r1 - r0
            h = ops.gemm(X[r0:r1], zf, bias=P["aemodel.mul_layer.bias"], act="relu", out=h0[:m], precision=pr)
            for lin, bn in (("enc.1", "enc.2"), ("enc.5", "enc.6")):
                hp = ops.gemm(h, P[f"aemodel.{lin}.weight"], transB=True, bias=P[f"aemodel.{lin}.bias"], precision=pr)
                h, _, _ = self._bn_fwd(bn, hp, False, act="relu")
            for k, hd in enumerate(HEADS):
                ops.gemm(h, P[f"aemodel.{hd}.1.weight"], transB=True, bias=P[f"aemodel.{hd}.1.bias"], out=pre[k][:m], precision=pr)
            acc3 = graphsci_ops.heads_eval([t[:m] for t in pre], gamma3, beta3, mean3, invstd3, Xraw[r0:r1], self.size_factors[r0:r1],
                                           None if mask is None else mask[r0:r1], acc=acc3,
                                           z_exp=None if z_exp is None else z_exp[r0:r1])
        acc2, _ = ops.adj_loss_grad(z, mu, ls, self.adj, self.pos_weight, want_grad=False)
        *_, loss = self._losses(acc3, acc2, le, la, ke, ka)
        return loss, z, z_exp

    def _graph_feat(self, graph):
        """Node features the GNN consumes: ``graph.ndata["feat"]`` ([genes, cells], as in the reference :126) when the graph
        object carries them, else the masked training matrix bound by ``fit``."""
        nd = getattr(graph, "ndata", None)
        if nd is not None and "feat" in nd:
            f = nd["feat"]
            if not (isinstance(f, torch.Tensor) and f.is_cuda and f.dtype == torch.float32 and f.is_contiguous()):
                f = _t(f, self.device)
                nd["feat"] = f
            return f
        return self._feat

    def save_model(self):
        self.best_state = self.state_dict()
        if self.save_path is not None:
            self.save_path.mkdir(parents=True, exist_ok=True)
            torch.save({k: {kk: vv.cpu() for kk, vv in v.items()} for k, v in self.best_state.items()}, self.save_path / f"{self.dataset}.pt")

    def load_model(self):
        if self.save_path is not None and (self.save_path / f"{self.dataset}.pt").exists():
            self.load_state_dict(torch.load(self.save_path / f"{self.dataset}.pt"))
        elif self.best_state is not None:
            self.load_state_dict(self.best_state)

    def predict(self, data, data_raw, graph, mask=None, eps=None):
        data = _t(data, self.device)
        if mask is not None:
            data = self.maskdata(data, mask)
        _, _, z_exp = self.evaluate(data, data_raw, graph, eps=eps)
        return z_exp

    def score(self, true_expr, imputed_expr, mask=None, metric="MSE", log1p=True, test_idx=None):
        allowed = {"RMSE", "PCC", "MRE"}
        if metric not in allowed:
            raise ValueError("scoring metric %r." % allowed)
        true_expr, imputed_expr = _t(true_expr, self.device), _t(imputed_expr, self.device)
        if test_idx is None:
            test_idx = range(len(true_expr))
        idx = torch.as_tensor(np.asarray(list(test_idx)), device=self.device)
        t, p = true_expr[idx], imputed_expr[idx]
        if log1p:
            p = torch.log1p(p)
        if mask is not None:
            mk = torch.as_tensor(np.asarray(mask)[np.asarray(list(test_idx))], device=self.device)
            p = torch.where(mk, t.to(p.dtype), p)
        else:
            mk = torch.zeros_like(t, dtype=torch.bool)       # the reference indexes `~mask[...]` and fails for mask=None; score everything
        if metric == "RMSE":
            return float(np.sqrt(torch.mean((t - p)**2).item()))
        tt, pp = t[~mk].cpu(), p[~mk].cpu()
        if metric == "PCC":
            return float(np.corrcoef(tt, pp)[0, 1])
        abs_actual = tt.abs().clamp(min=1e-10)
        return float(((pp - tt).abs() / abs_actual).mean().item())
