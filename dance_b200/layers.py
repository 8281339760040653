"""Graph-convolution layers with explicit forward / backward on the C-ABI kernels.

``GraphConvLayer`` covers the two GraphConv flavours on the hot path (SURVEY §8 a13):

* ``dgl.nn.GraphConv(norm="both")`` as used by GraphSCI (graphsci.py:117-131): no edge weights; multiplies by W first
  when ``in_feats > out_feats`` and aggregates first otherwise;
* the in-tree ``WeightedGraphConv.forward`` of graph-sc (modules/single_modality/clustering/graphsc.py:428-484): messages
  are ``h_src · w_e`` (edge weights), W always first, ``agg`` "sum" or "mean", ``norm`` "both" | "right" | "none".

Both are ``out = act(N_dst · A · (N_src · X [· W]) [· W] + b)`` with diagonal degree scalings, so the layer folds the
scalings into the CSR values once (``bind``) and each call is one SpMM + one GEMM (bias / activation fused).
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import scipy.sparse as sp
import torch

from . import ops


class GraphConvLayer:

    def __init__(self, in_feats: int, out_feats: int, *, norm: str = "both", edge_weighted: bool = False, weight_first: Optional[bool] = None,
                 agg: str = "sum", bias: bool = True, activation: Optional[str] = None, device="cuda", precision: Optional[str] = None,
                 seed: Optional[int] = None):
        if norm not in ("both", "right", "none") or agg not in ("sum", "mean"):
            raise ValueError("norm must be both|right|none and agg sum|mean")
        self.in_feats, self.out_feats, self.norm, self.agg = in_feats, out_feats, norm, agg
        self.edge_weighted, self.activation, self.precision = edge_weighted, activation, precision
        self.weight_first = (in_feats > out_feats) if weight_first is None else weight_first
        self.device = torch.device(device)
        gen = torch.Generator().manual_seed(seed) if seed is not None else None
        a = (6.0 / (in_feats + out_feats))**0.5                      # xavier_uniform_ (dgl GraphConv.reset_parameters)
        self.weight = ((torch.rand((in_feats, out_feats), generator=gen) * 2 - 1) * a).to(self.device)
        self.bias = torch.zeros(out_feats, device=self.device) if bias else None
        self.grad_weight = torch.zeros_like(self.weight)
        self.grad_bias = torch.zeros_like(self.bias) if bias else None
        self._A = self._AT = None

    # ---- graph ------------------------------------------------------------------------------
    def bind(self, src, dst, num_nodes: int, edge_weight=None, allow_zero_in_degree: bool = False):
        """Edges u→v (messages flow src→dst).  Degrees are structural (edge counts), as in dgl."""
        src, dst = np.asarray(src).astype(np.int64), np.asarray(dst).astype(np.int64)
        n = int(num_nodes)
        indeg = np.bincount(dst, minlength=n)
        outdeg = np.bincount(src, minlength=n)
        if not allow_zero_in_degree and (indeg == 0).any():
            raise RuntimeError("There are 0-in-degree nodes in the graph")
        w = np.ones(len(src), np.float32) if (edge_weight is None or not self.edge_weighted) else np.asarray(edge_weight, np.float32).reshape(-1)
        vals = w.astype(np.float32)
        if self.norm == "both":
            vals = vals * (outdeg.clip(min=1).astype(np.float32)**-0.5)[src]
        if self.norm == "both":
            vals = vals * (indeg.clip(min=1).astype(np.float32)**-0.5)[dst]
        elif self.norm == "right":
            vals = vals / indeg.clip(min=1).astype(np.float32)[dst]
        if self.agg == "mean":
            vals = vals / indeg.clip(min=1).astype(np.float32)[dst]
        A = sp.csr_matrix((vals, (dst, src)), shape=(n, n))           # row = destination; duplicate edges add up, like update_all(sum)
        A.sort_indices()
        self._A = ops.CSR.from_scipy(A, device=self.device)
        self._AT, _ = ops.csr_transpose(self._A)
        return self

    # ---- forward / backward -----------------------------------------------------------------
    def forward(self, feat: torch.Tensor) -> torch.Tensor:
        if self._A is None:
            raise RuntimeError("bind() the graph first")
        self._x = feat
        if self.weight_first:
            self._h = ops.gemm(feat, self.weight, precision=self.precision)
            self._out = ops.spmm(self._A, self._h, act=self.activation, bias=self.bias)
        else:
            self._h = ops.spmm(self._A, feat)
            self._out = ops.gemm(self._h, self.weight, bias=self.bias, act=self.activation, precision=self.precision)
        return self._out

    __call__ = forward

    def backward(self, dout: torch.Tensor, need_input_grad: bool = True) -> Optional[torch.Tensor]:
        """Accumulates nothing: ``grad_weight`` / ``grad_bias`` are overwritten; returns d(feat) or None."""
        act = self.activation
        if act in ("relu", ):
            dpre = ops.relu_bwd(dout, self._out)
        elif act in ("tanh", "elu"):
            dpre, _ = ops.gat_combine_bwd(dout, self._out, 1, self.out_feats, True, act=act)
        elif act is None:
            dpre = dout
        else:
            raise NotImplementedError(act)
        if self.bias is not None:
            ops.colsum(dpre, out=self.grad_bias)
        if self.weight_first:
            dh = ops.spmm(self._AT, dpre)                                                   # d(X·W)
            ops.gemm(self._x, dh, transA=True, out=self.grad_weight, precision=self.precision)
            return ops.gemm(dh, self.weight, transB=True, precision=self.precision) if need_input_grad else None
        ops.gemm(self._h, dpre, transA=True, out=self.grad_weight, precision=self.precision)
        if not need_input_grad:
            return None
        return ops.spmm(self._AT, ops.gemm(dpre, self.weight, transB=True, precision=self.precision))


class AdjLinearLayer:
    """``out = act(Â · (X · W) + b)`` with explicit backward — the plain GCN layer several reference modules define in-tree:

    * scDSC ``GNNLayer``                       modules/single_modality/clustering/scdsc.py:475-501  (xavier_uniform W, no bias, ReLU switch)
    * DSTG ``GraphConvolution``                modules/spatial/cell_type_deconvo/dstg.py:37-100     (glorot W, optional bias, no activation)
    * STdGCN ``conGraphConvolutionlayer``      modules/spatial/cell_type_deconvo/stdgcn.py:63-90    (U(±1/√out) W and b)
    * scGNN / SpaGCN ``GraphConvolution``      scgnn2.py:479-502, spagcn.py:337-363

    One tensor-core GEMM + one SpMM (bias and activation fused into the aggregate); backward = SpMM over Âᵀ + two GEMMs."""

    def __init__(self, in_features: int, out_features: int, *, bias: bool = False, activation: Optional[str] = None, init: str = "xavier",
                 device="cuda", precision: Optional[str] = None, seed: Optional[int] = None):
        self.in_features, self.out_features, self.activation, self.precision = in_features, out_features, activation, precision
        self.device = torch.device(device)
        gen = torch.Generator().manual_seed(seed) if seed is not None else None
        if init in ("xavier", "glorot"):
            a = (6.0 / (in_features + out_features))**0.5
        elif init == "uniform_out":
            a = 1.0 / out_features**0.5
        else:
            raise ValueError("init must be xavier | glorot | uniform_out")
        self.weight = ((torch.rand((in_features, out_features), generator=gen) * 2 - 1) * a).to(self.device)
        stdv = 1.0 / out_features**0.5
        self.bias = ((torch.rand(out_features, generator=gen) * 2 - 1) * stdv).to(self.device) if bias else None
        self.grad_weight = torch.zeros_like(self.weight)
        self.grad_bias = torch.zeros_like(self.bias) if bias else None
        self._A = self._AT = None

    def bind(self, adj, symmetric: bool = False):
        """``adj``: ops.CSR or scipy sparse matrix (rows = output nodes).  ``symmetric`` skips building Âᵀ."""
        self._A = adj if isinstance(adj, ops.CSR) else ops.CSR.from_scipy(sp.csr_matrix(adj), device=self.device)
        self._AT = self._A if symmetric else ops.csr_transpose(self._A)[0]
        return self

    def forward(self, x: torch.Tensor, active: bool = True) -> torch.Tensor:
        if self._A is None:
            raise RuntimeError("bind() the adjacency first")
        self._x = x
        self._act = self.activation if active else None
        support = ops.gemm(x, self.weight, precision=self.precision)
        self._out = ops.spmm(self._A, support, act=self._act, bias=self.bias)
        return self._out

    __call__ = forward

    def backward(self, dout: torch.Tensor, need_input_grad: bool = True) -> Optional[torch.Tensor]:
        if self._act == "relu":
            dpre = ops.relu_bwd(dout, self._out)
        elif self._act is None:
            dpre = dout
        else:
            dpre, _ = ops.gat_combine_bwd(dout, self._out, 1, self.out_features, True, act=self._act)
        if self.bias is not None:
            ops.colsum(dpre, out=self.grad_bias)
        ds = ops.spmm(self._AT, dpre)
        ops.gemm(self._x, ds, transA=True, out=self.grad_weight, precision=self.precision)
        return ops.gemm(ds, self.weight, transB=True, precision=self.precision) if need_input_grad else None


class TAGConvLayer:
    """``dgl.nn.TAGConv(in, out, k)`` as used by scTAG (sctag.py:101-102, 173-174; SURVEY App. A): with
    ``Ân = D_in^-1/2 · A_w · D_in^-1/2`` (structural in-degrees clamped to ≥ 1, edge weights inside), the hop stack
    ``[X, Ân X, …, Ân^k X]`` goes through ONE Linear of width in·(k+1).  Each hop is one SpMM written straight into its column block
    of the stacked buffer; the Linear is one GEMM.  Backward walks the hops in reverse over Ânᵀ."""

    def __init__(self, in_feats: int, out_feats: int, k: int = 2, *, bias: bool = True, activation: Optional[str] = None, device="cuda",
                 precision: Optional[str] = None, seed: Optional[int] = None):
        if in_feats % 4:
            raise ValueError("in_feats must be a multiple of 4 (16-byte aligned hop blocks)")
        self.in_feats, self.out_feats, self.k, self.activation, self.precision = in_feats, out_feats, k, activation, precision
        self.device = torch.device(device)
        gen = torch.Generator().manual_seed(seed) if seed is not None else None
        fan_in, fan_out = in_feats * (k + 1), out_feats
        std = (2.0**0.5) * (2.0 / (fan_in + fan_out))**0.5           # xavier_normal_(gain=calculate_gain("relu")), TAGConv.reset_parameters
        self.weight = (torch.randn((out_feats, fan_in), generator=gen) * std).to(self.device)      # nn.Linear layout [out, in·(k+1)]
        self.bias = torch.zeros(out_feats, device=self.device) if bias else None
        self.grad_weight = torch.zeros_like(self.weight)
        self.grad_bias = torch.zeros_like(self.bias) if bias else None
        self._A = self._AT = None

    def bind(self, src, dst, num_nodes: int, edge_weight=None):
        src, dst = np.asarray(src).astype(np.int64), np.asarray(dst).astype(np.int64)
        n = int(num_nodes)
        norm = np.bincount(dst, minlength=n).clip(min=1).astype(np.float32)**-0.5
        w = np.ones(len(src), np.float32) if edge_weight is None else np.asarray(edge_weight, np.float32).reshape(-1)
        A = sp.csr_matrix((w * norm[src] * norm[dst], (dst, src)), shape=(n, n))
        A.sort_indices()
        self._A = ops.CSR.from_scipy(A, device=self.device)
        self._AT, _ = ops.csr_transpose(self._A)
        return self

    def forward(self, feat: torch.Tensor) -> torch.Tensor:
        if self._A is None:
            raise RuntimeError("bind() the graph first")
        n, f = feat.shape
        self._stack = torch.empty((n, f * (self.k + 1)), dtype=torch.float32, device=self.device)
        self._stack[:, :f].copy_(feat)
        for t in range(1, self.k + 1):
            ops.spmm(self._A, self._stack[:, (t - 1) * f:t * f], out=self._stack[:, t * f:(t + 1) * f])
        self._out = ops.gemm(self._stack, self.weight, transB=True, bias=self.bias, act=self.activation, precision=self.precision)
        return self._out

    __call__ = forward

    def backward(self, dout: torch.Tensor, need_input_grad: bool = True) -> Optional[torch.Tensor]:
        if self.activation == "relu":
            dpre = ops.relu_bwd(dout, self._out)
        elif self.activation is None:
            dpre = dout
        else:
            dpre, _ = ops.gat_combine_bwd(dout, self._out, 1, self.out_feats, True, act=self.activation)
        if self.bias is not None:
            ops.colsum(dpre, out=self.grad_bias)
        ops.gemm(dpre, self._stack, transA=True, out=self.grad_weight, precision=self.precision)
        if not need_input_grad:
            return None
        f = self.in_feats
        dstack = ops.gemm(dpre, self.weight, precision=self.precision)                     # [n, f·(k+1)]
        carry = dstack[:, self.k * f:(self.k + 1) * f].contiguous()
        for t in range(self.k, 0, -1):                                                     # d H_{t-1} += Ânᵀ · d H_t
            back = ops.spmm(self._AT, carry)
            carry = back + dstack[:, (t - 1) * f:t * f]
        return carry
