"""STAGATE on the H100-native kernels — host-side mirror of ``dance/modules/spatial/spatial_domain/stagate.py``
(GATConv :31-128, Stagate :131-284).

Forward (stagate.py:175-200), one attention head, no bias, no self-loop insertion::

    H1 = X·W1                     s_src = <H1, a_src>, s_dst = <H1, a_dst>
    α_e = softmax_{edges into v}( sigmoid(s_src[u] + s_dst[v]) )          (PyG softmax: shift by the per-target max, +1e-16)
    h1 = ELU(Σ_e α_e H1[u])       h2 = h1·W2   (attention=False → projection only)
    h3 = ELU(Σ_e α_e (h2·W2ᵀ)[u]) (tied attention: conv1's node scores ⇒ the SAME α)      h4 = h3·W1ᵀ
    loss = mean((X − h4)²)

Reference quirks reproduced on purpose:
* ``conv3.lin_src`` / ``conv4.lin_src`` are separate Parameters whose storage is re-pointed to ``conv2.lin_src.T`` /
  ``conv1.lin_src.T`` on every forward (:193-196).  Autograd therefore gives W1 and W2 TWO gradients each (one per use)
  with two independent Adam states, and both updates land in the same storage.  The engine keeps the second gradients in
  transposed form (``g3ᵀ = dH3ᵀ·h2`` has W2's shape) — Adam is elementwise, so stepping W2 with (g3ᵀ, its own moments) is
  the same arithmetic as stepping the transposed view.
* ``clip_grad_norm_`` (:221) runs over the six tensors that actually receive gradients; conv2/3/4's attention vectors
  never do (Adam skips them) but stay in ``state_dict``.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import numpy as np
import scipy.sparse as sp
import torch

from .. import ops
from ..engine import FlatParams


def _xavier_normal(shape, fan_in, fan_out, gain, gen):
    std = gain * (2.0 / (fan_in + fan_out))**0.5
    return torch.randn(shape, generator=gen) * std


class Stagate:

    def __init__(self, hidden_dims, device: str = "cuda", pretrain_path: Optional[str] = None, precision: Optional[str] = None,
                 seed: Optional[int] = None):
        self.pretrain_path = pretrain_path
        in_dim, num_hidden, out_dim = (int(v) for v in hidden_dims)
        if num_hidden > 512 or in_dim < 1 or out_dim < 1:
            raise ValueError("hidden width must be <= 512 (the reference default)")
        self.dims = (in_dim, num_hidden, out_dim)
        self.device = torch.device("cuda" if device in ("auto", "cpu") else device)
        if self.device.type != "cuda":
            raise RuntimeError("dance_b200 runs on CUDA devices only")
        self.precision = precision
        # trained tensors + the two "second use" gradient slots (own Adam moments, same storage as W2 / W1)
        self.params = FlatParams([("conv1.lin_src", (in_dim, num_hidden)), ("conv1.att_src", (num_hidden, )),
                                  ("conv1.att_dst", (num_hidden, )), ("conv2.lin_src", (num_hidden, out_dim)),
                                  ("conv3.lin_src.T", (num_hidden, out_dim)), ("conv4.lin_src.T", (in_dim, num_hidden))], self.device)
        gen = torch.Generator().manual_seed(seed) if seed is not None else None
        P = self.params.p
        g = 1.414
        P["conv1.lin_src"].copy_(_xavier_normal((in_dim, num_hidden), num_hidden, in_dim, g, gen))      # fan of a 2-D tensor: (size(1), size(0))
        P["conv1.att_src"].copy_(_xavier_normal((num_hidden, ), num_hidden, num_hidden, g, gen))         # (1, heads, C): fan_in = fan_out = C
        P["conv1.att_dst"].copy_(_xavier_normal((num_hidden, ), num_hidden, num_hidden, g, gen))
        P["conv2.lin_src"].copy_(_xavier_normal((num_hidden, out_dim), out_dim, num_hidden, g, gen))
        # attention vectors of conv2..4: initialised, never trained (kept for state_dict compatibility)
        self.unused = {f"conv{i}.att_{s}": _xavier_normal((1, 1, w), w, w, g, gen)
                       for i, w in ((2, out_dim), (3, num_hidden), (4, in_dim)) for s in ("src", "dst")}
        self._graph = None
        self.rep: Optional[np.ndarray] = None
        self.clust_res = None
        self._is_pretrained = False
        self.last_loss = None
        self.last_grad_norm = torch.zeros(1, dtype=torch.float32, device=self.device)

    # ---- parameters -------------------------------------------------------------------------
    def state_dict(self) -> Dict[str, torch.Tensor]:
        P = self.params.p
        sd = {"conv1.lin_src": P["conv1.lin_src"].clone(), "conv1.att_src": P["conv1.att_src"].view(1, 1, -1).clone(),
              "conv1.att_dst": P["conv1.att_dst"].view(1, 1, -1).clone(), "conv2.lin_src": P["conv2.lin_src"].clone(),
              "conv3.lin_src": P["conv2.lin_src"].t().clone(), "conv4.lin_src": P["conv1.lin_src"].t().clone()}
        sd.update({k: v.clone() for k, v in self.unused.items()})
        return sd

    def load_state_dict(self, sd):
        P = self.params.p
        as_t = lambda v: torch.as_tensor(np.asarray(v.cpu() if isinstance(v, torch.Tensor) else v), dtype=torch.float32)
        P["conv1.lin_src"].copy_(as_t(sd["conv1.lin_src"]))
        P["conv1.att_src"].copy_(as_t(sd["conv1.att_src"]).reshape(-1))
        P["conv1.att_dst"].copy_(as_t(sd["conv1.att_dst"]).reshape(-1))
        P["conv2.lin_src"].copy_(as_t(sd["conv2.lin_src"]))
        for k in self.unused:
            if k in sd:
                self.unused[k] = as_t(sd[k]).clone()

    # ---- graph ------------------------------------------------------------------------------
    def _bind_graph(self, edge_index_array, n: int):
        """edge_index[0] = source j, edge_index[1] = target i (PyG flow) → CSR indexed by target (+ its transpose)."""
        key = id(edge_index_array)
        if self._graph is not None and self._graph[0] == key and self._graph[1] == n:
            return
        ei = np.asarray(edge_index_array).astype(np.int64)
        T = sp.csr_matrix((np.ones(ei.shape[1], np.float32), (ei[1], ei[0])), shape=(n, n))
        T.sum_duplicates()
        T.sort_indices()
        if T.nnz != ei.shape[1]:
            raise ValueError("duplicate edges are not supported (the reference builds edge_index from np.nonzero(adj))")
        Tc = ops.CSR.from_scipy(T, device=self.device)
        Tt, perm = ops.csr_transpose(Tc)
        self._graph = (key, n, edge_index_array, Tc, Tt, perm)

    # ---- forward / backward -----------------------------------------------------------------
    def _forward(self, X: torch.Tensor, keep: bool):
        _, _, _, T, _, _ = self._graph
        P = self.params.p
        W1, W2 = P["conv1.lin_src"], P["conv2.lin_src"]
        H1 = ops.gemm(X, W1, precision=self.precision)
        s_src, s_dst = ops.gat_scores(H1, P["conv1.att_src"], P["conv1.att_dst"], 1)
        agg1, alpha, _ = ops.gat_aggregate_fwd(T, H1, s_src, s_dst, 1, score_act="sigmoid", shift="segment")
        h1 = ops.gat_combine_fwd(agg1, None, None, 1, True, act="elu")
        h2 = ops.gemm(h1, W2, precision=self.precision)
        H3 = ops.gemm(h2, W2, transB=True, precision=self.precision)
        Ta = ops.CSR(T.rowptr, T.colidx, alpha.view(-1), T.shape)
        h3 = ops.spmm(Ta, H3, act="elu")
        h4 = ops.gemm(h3, W1, transB=True, precision=self.precision)
        cache = (H1, s_src, s_dst, alpha, h1, h2, H3, h3) if keep else None
        return h2, h4, cache

    def forward(self, features, edge_index) -> Tuple[torch.Tensor, torch.Tensor]:
        X = self._to_dev(features)
        self._bind_graph(edge_index, X.shape[0])
        h2, h4, _ = self._forward(X, keep=False)
        return h2, h4

    __call__ = forward

    def _to_dev(self, x) -> torch.Tensor:
        if isinstance(x, torch.Tensor):
            return x.to(device=self.device, dtype=torch.float32).contiguous()
        return torch.as_tensor(np.ascontiguousarray(x, dtype=np.float32)).to(self.device)

    def _train_step(self, X: torch.Tensor, lr: float, weight_decay: float, gradient_clipping: float):
        _, n, _, T, Tt, perm = self._graph
        P, G = self.params.p, self.params.g
        W1, W2 = P["conv1.lin_src"], P["conv2.lin_src"]
        in_dim = self.dims[0]
        h2, h4, (H1, s_src, s_dst, alpha, h1, _, H3, h3) = self._forward(X, keep=True)
        loss_sum, dh4 = ops.mse_sum_loss_grad(h4, X)                                    # Σ(h4−X)², 2(h4−X); the mean's 1/(N·D) is applied at the clip
        ops.gemm(dh4, h3, transA=True, out=G["conv4.lin_src.T"], precision=self.precision)    # (h3ᵀ·dh4)ᵀ : conv4's own gradient, W1-shaped
        dh3 = ops.gemm(dh4, W1, precision=self.precision)
        dagg3 = ops.act_bwd(dh3, "elu", y=h3)
        # Layer 3's message path (dH3 = Σ α dagg3) feeds h2 → h1 → dagg1, so it runs first as a plain SpMM on the transposed
        # CSR; dα sums both layers' contributions and is formed in the tied backward once dagg1 exists.
        Tta = ops.CSR(Tt.rowptr, Tt.colidx, alpha.view(-1)[perm.long()], Tt.shape)
        dH3 = ops.spmm(Tta, dagg3)
        ops.gemm(dH3, h2, transA=True, out=G["conv3.lin_src.T"], precision=self.precision)    # (h2ᵀ·dH3)ᵀ : conv3's own gradient, W2-shaped
        dh2 = ops.gemm(dH3, W2, precision=self.precision)
        ops.gemm(h1, dh2, transA=True, out=G["conv2.lin_src"], precision=self.precision)
        dh1 = ops.gemm(dh2, W2, transB=True, precision=self.precision)
        dagg1 = ops.act_bwd(dh1, "elu", y=h1)
        dH1, da_src, da_dst, _ = ops.gat_aggregate_bwd(T, Tt, perm, H1, P["conv1.att_src"], P["conv1.att_dst"], s_src, s_dst, alpha,
                                                       dagg1, 1, score_act="sigmoid", H2=H3, dOut2=dagg3, want_dH2=False)
        G["conv1.att_src"].copy_(da_src)
        G["conv1.att_dst"].copy_(da_dst)
        ops.gemm(X, dH1, transA=True, out=G["conv1.lin_src"], precision=self.precision)
        numel = float(n * in_dim)
        ops.clip_grad_norm_(self.params.grad, gradient_clipping, pre_scale=1.0 / numel, norm_out=self.last_grad_norm)
        self._adam(lr, weight_decay)
        self.last_loss = loss_sum / numel

    def _adam(self, lr, weight_decay, betas=(0.9, 0.999), eps=1e-8):
        """Parameter order of the reference optimiser: conv1.*, conv2.lin_src, then conv3.lin_src, conv4.lin_src (aliases)."""
        fp = self.params
        fp.step += 1
        P, G = fp.p, fp.g

        def seg(name):
            o = P[name].data_ptr() - fp.flat.data_ptr()
            o //= 4
            return slice(o, o + P[name].numel())

        first = slice(seg("conv1.lin_src").start, seg("conv2.lin_src").stop)           # contiguous: W1, a_src, a_dst, W2
        ops.adam_step(fp.flat[first], fp.grad[first], fp.exp_avg[first], fp.exp_avg_sq[first], fp.step, lr, betas[0], betas[1], eps,
                      weight_decay)
        for alias, target in (("conv3.lin_src.T", "conv2.lin_src"), ("conv4.lin_src.T", "conv1.lin_src")):
            sa, st = seg(alias), seg(target)
            ops.adam_step(fp.flat[st], fp.grad[sa], fp.exp_avg[sa], fp.exp_avg_sq[sa], fp.step, lr, betas[0], betas[1], eps, weight_decay)

    # ---- reference API ----------------------------------------------------------------------
    @staticmethod
    def preprocessing_pipeline(hvg_flavor: str = "seurat_v3", n_top_hvgs: int = 3000, model_name: str = "radius", radius: float = 150,
                               n_neighbors: int = 5, log_level="INFO"):
        from ..transforms import AnnDataTransform, Compose, SetConfig
        from ..transforms.graph import StagateGraph
        return Compose(
            AnnDataTransform("scanpy.pp.highly_variable_genes", flavor=hvg_flavor, n_top_genes=n_top_hvgs, subset=True),
            AnnDataTransform("scanpy.pp.normalize_total", target_sum=1e4),
            AnnDataTransform("scanpy.pp.log1p"),
            StagateGraph(model_name, radius=radius, n_neighbors=n_neighbors),
            SetConfig({
                "feature_channel": "StagateGraph",
                "feature_channel_type": "obsp",
                "label_channel": "label",
                "label_channel_type": "obs"
            }),
            log_level=log_level,
        )

    def pretrain(self, x: np.ndarray, edge_index_array: np.ndarray, lr: float = 1e-3, weight_decay: float = 1e-4, epochs: int = 100,
                 gradient_clipping: float = 5):
        X = self._to_dev(np.asarray(x).astype(np.float32))
        self._bind_graph(edge_index_array, X.shape[0])
        for b in (self.params.exp_avg, self.params.exp_avg_sq):
            b.zero_()
        self.params.step = 0
        for _ in range(1, epochs + 1):
            self._train_step(X, lr, weight_decay, gradient_clipping)
        z, _, _ = self._forward(X, keep=False)
        self.rep = z.detach().cpu().numpy()

    def _pretrain(self, *args, force_pretrain: bool = False, **kwargs):
        import os
        if not force_pretrain:
            if self._is_pretrained:
                return
            if self.pretrain_path is not None and os.path.isfile(self.pretrain_path):
                self.load_pretrained(self.pretrain_path)
                self._is_pretrained = True
                return
        self.pretrain(*args, **kwargs)
        self._is_pretrained = True
        if self.pretrain_path is not None:
            self.save_pretrained(self.pretrain_path)

    def save_pretrained(self, path):
        np.save(path, self.rep)

    def load_pretrained(self, path):
        self.rep = np.load(path)

    def fit(self, inputs, epochs: int = 100, lr: float = 0.001, gradient_clipping: float = 5, weight_decay: float = 1e-4,
            num_cluster: int = 7, gmm_reg_covar: float = 1.5e-4, gmm_n_init: int = 10, gmm_max_iter: int = 300, gmm_tol: float = 2e-4,
            random_state: Optional[int] = None):
        x, edge_index_array = inputs
        self._pretrain(x, edge_index_array, lr, weight_decay, epochs, gradient_clipping)
        # cluster assignment on the 30-d representation: the same sklearn call as the reference (:270-273); not on the hot path
        from sklearn.mixture import GaussianMixture
        gmm = GaussianMixture(n_components=num_cluster, covariance_type="tied", n_init=gmm_n_init, tol=gmm_tol, max_iter=gmm_max_iter,
                              reg_covar=gmm_reg_covar, random_state=random_state)
        self.clust_res = gmm.fit_predict(self.rep)
        return self

    def predict(self, x=None):
        return self.clust_res

    def fit_predict(self, x, y=None, **fit_kwargs):
        self.fit(x, **fit_kwargs)
        return self.predict(x)

    def score(self, x, y, score_func=None) -> float:
        if score_func is None:
            from sklearn.metrics import adjusted_rand_score as score_func
        return float(score_func(np.asarray(y), self.predict(x)))

    def fit_score(self, x, y, score_func=None, **fit_kwargs) -> float:
        self.fit(x, **fit_kwargs)
        return self.score(x, y, score_func)
