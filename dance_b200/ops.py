"""Thin torch-tensor wrappers over the C-ABI (``include/dance_b200.h``).

Every function takes CUDA tensors, hands raw pointers to the shared library on torch's
current stream and returns CUDA tensors.  Nothing here computes on the CPU and nothing
falls back to torch kernels: a missing library or a non-CUDA tensor raises.
"""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple, Optional, Tuple

import torch

from ._lib import B2Error, check
from ._lib import lib as _raw_lib

ACT = {"none": 0, None: 0, "relu": 1, "elu": 2, "tanh": 3}
# every activation code, for act / act_bwd; the GEMM / SpMM epilogues take ACT only
ACT_ALL = {**ACT, "leaky_relu": 4, "gelu": 5}
PREC = {"fp32": 0, "simt": 0, "tf32x3": 1, "tf32": 2, "bf16": 3}

_DEFAULT_PRECISION = "tf32x3"

# ---- instrumentation (bench.py): launch counter + optional per-entry-point CUDA-event timing -------------
_timing = {"on": False, "events": []}
_launch_base = [0]


class _TimedLib:
    """Proxy over the ctypes library: when timing is enabled every compute entry point is bracketed by
    CUDA events on the launching (current) stream."""

    def __getattr__(self, name):
        fn = getattr(_raw_lib(), name)
        if not _timing["on"] or name.endswith("_bytes") or name in ("b2_last_error", "b2_version", "b2_launch_count",
                                                                     "b2_device_info"):
            return fn

        def timed(*a):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            rc = fn(*a)
            e.record()
            _timing["events"].append((name[3:], s, e))
            return rc
        return timed


_proxy = _TimedLib()


def lib():
    return _proxy


def reset_counters():
    _launch_base[0] = _raw_lib().b2_launch_count()


def counters():
    return {"launches": _raw_lib().b2_launch_count() - _launch_base[0]}


def enable_kernel_timing(on: bool):
    _timing["on"] = bool(on)
    if on:
        _timing["events"] = []


def kernel_times():
    """{entry point: {"ms": total, "n": calls}} for the calls recorded since timing was enabled (synchronises)."""
    torch.cuda.synchronize()
    out = {}
    for name, s, e in _timing["events"]:
        d = out.setdefault(name, {"ms": 0.0, "n": 0})
        d["ms"] += s.elapsed_time(e)
        d["n"] += 1
    return out


def set_default_precision(p: str):
    """GEMM precision used when a call does not name one: 'fp32' | 'tf32x3' | 'tf32' | 'bf16' (see :func:`gemm`)."""
    global _DEFAULT_PRECISION
    if p not in PREC:
        raise ValueError(f"unknown precision {p!r}; choose from {sorted(PREC)}")
    _DEFAULT_PRECISION = p


def get_default_precision() -> str:
    return _DEFAULT_PRECISION


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _p(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _chk(t: torch.Tensor, dtype, name: str, ndim: Optional[int] = None):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise B2Error(f"{name}: expected a CUDA tensor (dance_b200 has no CPU path)")
    if t.dtype != dtype:
        raise B2Error(f"{name}: expected dtype {dtype}, got {t.dtype}")
    if ndim is not None and t.dim() != ndim:
        raise B2Error(f"{name}: expected {ndim}-D tensor, got shape {tuple(t.shape)}")


def _rowmajor(t: torch.Tensor, name: str) -> int:
    """Leading dimension of a 2-D row-major (possibly row-padded) tensor."""
    if t.dim() != 2 or t.stride(1) != 1:
        raise B2Error(f"{name}: must be 2-D with unit inner stride, got strides {t.stride()}")
    return t.stride(0) if t.shape[0] > 1 else max(t.stride(0), t.shape[1])


_ws_cache = {}


def _workspace(nbytes: int, device) -> torch.Tensor:
    """Per-device grow-only scratch buffer (stream-ordered use only)."""
    key = (device.index if device.index is not None else torch.cuda.current_device())
    buf = _ws_cache.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8, device=device)
        _ws_cache[key] = buf
    return buf


_PATHS = {"gae": (0, {"auto": 0, "cuda": 1, "tc": 2}), "knn": (1, {"auto": 0, "simt": 1}),
          "spmm": (2, {"auto": 0, "rowgroup": 1})}


def set_path(which: str, mode: str = "auto") -> None:
    """Select the kernel path of the decoder ("gae": auto | cuda | tc), of the kNN candidate filter ("knn": auto | simt) or
    of the aggregate ("spmm": auto | rowgroup).  All paths return the same result; the switch exists
    for A/B tests and timing."""
    sel, modes = _PATHS[which]
    check(lib().b2_set_path(sel, modes[mode]), "b2_set_path")


def set_tuning(knob: str, value: int) -> None:
    """Scheduling knob of the tensor-core decoder ("gae_splits": step ranges per 128-row block of the J sweep, 0 = automatic):
    timing experiments only."""
    check(lib().b2_set_tuning({"gae_splits": 0}[knob], int(value)), "b2_set_tuning")


def get_path(which: str) -> str:
    sel, modes = _PATHS[which]
    v = lib().b2_get_path(sel)
    return next(k for k, m in modes.items() if m == v)


def device_info() -> Tuple[int, int, int]:
    a, b, c = C.c_int(), C.c_int(), C.c_int()
    check(lib().b2_device_info(C.byref(a), C.byref(b), C.byref(c)), "b2_device_info")
    return a.value, b.value, c.value


# ----------------------------------------------------------------------------- CSR container
class CSR:
    """Device CSR matrix: int32 rowptr/colidx, optional fp32 values (None = all ones)."""

    __slots__ = ("rowptr", "colidx", "vals", "shape", "_t", "sigmas", "rhos")

    def __init__(self, rowptr, colidx, vals, shape):
        _chk(rowptr, torch.int32, "rowptr", 1)
        _chk(colidx, torch.int32, "colidx", 1)
        if vals is not None:
            _chk(vals, torch.float32, "vals", 1)
        self.rowptr, self.colidx, self.vals, self.shape = rowptr, colidx, vals, tuple(shape)
        self._t = None

    @property
    def nnz(self) -> int:
        return self.colidx.numel()

    @classmethod
    def from_scipy(cls, m, device="cuda", with_values=True):
        m = m.tocsr()
        m.sort_indices()
        return cls(torch.from_numpy(m.indptr.astype("int32")).to(device),
                   torch.from_numpy(m.indices.astype("int32")).to(device),
                   torch.from_numpy(m.data.astype("float32")).to(device) if with_values else None, m.shape)

    def to_scipy(self):
        import numpy as np
        import scipy.sparse as sp
        vals = self.vals.cpu().numpy() if self.vals is not None else np.ones(self.nnz, dtype="float32")
        return sp.csr_matrix((vals, self.colidx.cpu().numpy(), self.rowptr.cpu().numpy()), shape=self.shape)

    def transpose(self) -> "CSR":
        """Deterministic device transpose (cached)."""
        if self._t is None:
            self._t = csr_transpose(self)[0]
        return self._t


_X16 = {torch.bfloat16: ("b2_spmm_csr_bf16", 0), torch.float16: ("b2_spmm_csr_f16", 1)}


def to_x16(X: torch.Tensor, dtype=torch.bfloat16, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """fp32 → bf16 / fp16 copy of a row-major matrix (operand of the 16-bit aggregate)."""
    _chk(X, torch.float32, "X", 2)
    if dtype not in _X16:
        raise B2Error(f"to_x16: dtype must be torch.bfloat16 or torch.float16, got {dtype}")
    if out is None:
        out = torch.empty(X.shape, dtype=dtype, device=X.device)
    _chk(out, dtype, "out", 2)
    check(lib().b2_convert_f32_to_x16(_p(X), _rowmajor(X, "X"), _p(out), _rowmajor(out, "out"), X.shape[0], X.shape[1], _X16[dtype][1],
                                      _stream()), "b2_convert_f32_to_x16")
    return out


def spmm(A: CSR, X: torch.Tensor, reduce: str = "sum", act: Optional[str] = None,
         out: Optional[torch.Tensor] = None, bias: Optional[torch.Tensor] = None, out16: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``Y = act(A @ X)`` (reduce='sum') or row-mean (reduce='mean').  A bf16 / fp16 ``X`` is gathered in its 16-bit
    type (fp32 accumulation, fp32 ``out``; ``out16`` additionally receives the result in the operand's type)."""
    x16 = isinstance(X, torch.Tensor) and X.dtype in _X16
    _chk(X, X.dtype if x16 else torch.float32, "X", 2)
    n_rows, n_cols = A.shape
    if X.shape[0] != n_cols:
        raise B2Error(f"spmm: A is {A.shape} but X has {X.shape[0]} rows")
    F = X.shape[1]
    if not x16:
        out16 = None  # an fp32 operand has no 16-bit result copy
    if out is None and out16 is None:
        out = torch.empty((n_rows, F), dtype=torch.float32, device=X.device)
    if out is not None:
        _chk(out, torch.float32, "out", 2)
    if out16 is not None:
        _chk(out16, X.dtype, "out16", 2)
    colidx_ptr = _p(A.colidx) if A.nnz else _p(A.rowptr)  # an empty matrix has no colidx storage; never dereferenced
    args = [_p(A.rowptr), colidx_ptr, _p(A.vals) if A.nnz else None, _p(X), _rowmajor(X, "X"),
            _p(out), _rowmajor(out, "out") if out is not None else 0]
    if x16:
        fn = _X16[X.dtype][0]
        args += [_p(out16), _rowmajor(out16, "out16") if out16 is not None else 0]
    else:
        fn = "b2_spmm_csr_f32"
    check(getattr(lib(), fn)(*args, n_rows, n_cols, F, {"sum": 0, "mean": 1}[reduce], ACT[act], _p(bias), _stream()), fn)
    return out if out is not None else out16


def csr_transpose(A: CSR) -> Tuple[CSR, torch.Tensor]:
    n_rows, n_cols = A.shape
    nnz = A.nnz
    dev = A.rowptr.device
    t_rowptr = torch.empty(n_cols + 1, dtype=torch.int32, device=dev)
    t_colidx = torch.empty(nnz, dtype=torch.int32, device=dev)
    t_vals = torch.empty(nnz, dtype=torch.float32, device=dev) if A.vals is not None else None
    perm = torch.empty(nnz, dtype=torch.int32, device=dev)
    nbytes = lib().b2_csr_transpose_workspace_bytes(n_rows, n_cols, nnz)
    ws = _workspace(nbytes, dev)
    check(lib().b2_csr_transpose(_p(A.rowptr), _p(A.colidx), _p(A.vals), n_rows, n_cols, nnz, _p(t_rowptr), _p(t_colidx),
                                 _p(t_vals), _p(perm), _p(ws), ws.numel(), _stream()), "b2_csr_transpose")
    return CSR(t_rowptr, t_colidx, t_vals, (n_cols, n_rows)), perm


def gemm(A: torch.Tensor, B: torch.Tensor, *, transA: bool = False, transB: bool = False,
         bias: Optional[torch.Tensor] = None, act: Optional[str] = None, mask: Optional[torch.Tensor] = None,
         out: Optional[torch.Tensor] = None, accumulate: bool = False, precision: Optional[str] = None) -> torch.Tensor:
    """``C = act(op(A) @ op(B) + bias) * (mask > 0)``; ``accumulate`` adds into ``out``.

    All tensors are float32.  ``precision`` (default: :func:`set_default_precision`, initially 'tf32x3') bounds how the
    tensor cores round the operands: 'tf32x3' is fp32-accurate (3-product split), 'tf32' uses 10-bit mantissas, 'bf16'
    rounds each operand to bfloat16 (round-to-nearest-even, 8-bit mantissa) inside the kernel; all three accumulate in
    fp32.  'fp32' forces the CUDA-core kernel.  Shapes the tensor-core kernel does not take (K < 8, M·N·K < 2^18, a base
    not 16-byte aligned or a row pitch not a multiple of 4) run on the CUDA-core fp32 kernel whatever the mode."""
    _chk(A, torch.float32, "A", 2)
    _chk(B, torch.float32, "B", 2)
    lda, ldb = _rowmajor(A, "A"), _rowmajor(B, "B")
    M, K = (A.shape[1], A.shape[0]) if transA else A.shape
    Kb, N = (B.shape[1], B.shape[0]) if transB else B.shape
    if K != Kb:
        raise B2Error(f"gemm: inner dimensions differ ({K} vs {Kb})")
    if out is None:
        if accumulate:
            raise B2Error("gemm: accumulate=True needs `out`")
        out = torch.empty((M, N), dtype=torch.float32, device=A.device)
    _chk(out, torch.float32, "out", 2)
    if tuple(out.shape) != (M, N):
        raise B2Error(f"gemm: out has shape {tuple(out.shape)}, expected {(M, N)}")
    if bias is not None:
        _chk(bias, torch.float32, "bias", 1)
    ldmask = 0
    if mask is not None:
        _chk(mask, torch.float32, "mask", 2)
        ldmask = _rowmajor(mask, "mask")
    prec = PREC[precision or _DEFAULT_PRECISION]
    nbytes = lib().b2_gemm_workspace_bytes(M, N, K, int(transA), int(transB), prec)
    ws = _workspace(nbytes, A.device) if nbytes else None
    check(lib().b2_gemm_f32(_p(A), lda, int(transA), _p(B), ldb, int(transB), _p(out), _rowmajor(out, "out"), M, N, K,
                            _p(bias), ACT[act], _p(mask), ldmask, 1.0 if accumulate else 0.0, prec,
                            _p(ws), ws.numel() if ws is not None else 0, _stream()), "b2_gemm_f32")
    return out


def colsum(X: torch.Tensor, out: Optional[torch.Tensor] = None, accumulate: bool = False) -> torch.Tensor:
    _chk(X, torch.float32, "X", 2)
    if out is None:
        out = torch.empty(X.shape[1], dtype=torch.float32, device=X.device)
    nbytes = lib().b2_colsum_workspace_bytes(X.shape[0], X.shape[1])
    ws = _workspace(nbytes, X.device) if nbytes else None
    check(lib().b2_colsum_f32(_p(X), _rowmajor(X, "X"), X.shape[0], X.shape[1], _p(out), 1.0 if accumulate else 0.0,
                              _p(ws), ws.numel() if ws is not None else 0, _stream()), "b2_colsum_f32")
    return out


def mse_sum_loss_grad(recon, target, ltmg_regu=None, regu_strength=0.0, relu_mask=False, grad=None, loss_out=None):
    """Feature-AE loss; returns (loss_out[1] accumulated, grad wrt recon)."""
    _chk(recon, torch.float32, "recon")
    _chk(target, torch.float32, "target")
    if not (recon.is_contiguous() and target.is_contiguous()):
        raise B2Error("mse_sum_loss_grad: recon/target must be contiguous")
    if grad is None:
        grad = torch.empty_like(recon)
    if loss_out is None:
        loss_out = torch.zeros(1, dtype=torch.float32, device=recon.device)
    check(lib().b2_mse_sum_loss_grad_f32(_p(recon), _p(target), _p(ltmg_regu), float(regu_strength), int(relu_mask),
                                         _p(grad), _p(loss_out), recon.numel(), _stream()), "b2_mse_sum_loss_grad_f32")
    return loss_out, grad


def _gae_prepare(what, z, labels: CSR, n_rows, mu, logvar, dmu, dlogvar, loss, labels_t: Optional[CSR] = None):
    """Checks and buffers both decoder calls share; returns (n, d, n_rows, ldm, ldd, dmu, dlogvar, loss, workspace, label
    arguments).  The label arguments are the pointers of L and of Lᵀ; the library reads Lᵀ only when L has values."""
    _chk(z, torch.float32, "z", 2)
    n, d = z.shape
    n_rows = n if n_rows is None else n_rows
    if labels.shape[0] != n_rows or labels.shape[1] != n:
        raise B2Error(f"{what}: labels must be [{n_rows}, {n}] (rows of this shard x all columns), got {tuple(labels.shape)}")
    if labels.vals is not None:
        if labels_t is None or labels_t.vals is None:
            raise B2Error(f"{what}: real-valued labels need labels_t= (the same rows of Lᵀ, with values)")
        if tuple(labels_t.shape) != tuple(labels.shape):
            raise B2Error(f"{what}: labels_t must be [{n_rows}, {n}] like labels, got {tuple(labels_t.shape)}")
    ldm = ldd = 0
    if mu is not None:
        _chk(mu, torch.float32, "mu", 2)
        _chk(logvar, torch.float32, "logvar", 2)
        ldm = _rowmajor(mu, "mu")
        if _rowmajor(logvar, "logvar") != ldm:
            raise B2Error(f"{what}: mu and logvar must share a leading dimension")
        if dmu is None:
            dmu = torch.empty((n_rows, d), dtype=torch.float32, device=z.device)
            dlogvar = torch.empty((n_rows, d), dtype=torch.float32, device=z.device)
        ldd = _rowmajor(dmu, "dmu")
        if _rowmajor(dlogvar, "dlogvar") != ldd:
            raise B2Error(f"{what}: dmu and dlogvar must share a leading dimension")
    if loss is None:
        loss = torch.empty(1, dtype=torch.float32, device=z.device)
    lt = (labels_t.rowptr, labels_t.colidx, labels_t.vals) if labels_t is not None else (None, None, None)
    labs = [_p(t) for t in (labels.rowptr, labels.colidx, labels.vals, *lt)]
    return n, d, n_rows, ldm, ldd, dmu, dlogvar, loss, _workspace(lib().b2_gae_loss_workspace_bytes(n, d), z.device), labs


def gae_loss_grad(z, labels: CSR, norm: float, pos_weight: float, mu=None, logvar=None, use_pos_weight=True,
                  dz=None, dmu=None, dlogvar=None, loss=None, row_begin: int = 0, n_rows: Optional[int] = None,
                  labels_t: Optional[CSR] = None):
    """Matrix-free Graph-AE loss: returns (loss[1], dz, dmu, dlogvar).

    ``dmu``/``dlogvar`` may be column slices of one packed [n, 2d] buffer (shared leading dimension).
    ``labels.vals`` None: unit, symmetric labels.  Otherwise real-valued, possibly asymmetric labels (graph_AE_retain_weights), and
    ``labels_t`` holds the same rows of Lᵀ with their values.
    """
    n, d, n_rows, ldm, ldd, dmu, dlogvar, loss, ws, labs = _gae_prepare("gae_loss_grad", z, labels, n_rows, mu, logvar, dmu, dlogvar,
                                                                        loss, labels_t)
    if dz is None:
        dz = torch.empty((n_rows, d), dtype=torch.float32, device=z.device)
    else:
        _chk(dz, torch.float32, "dz", 2)
        if tuple(dz.shape) != (n_rows, d) or not dz.is_contiguous():
            raise B2Error(f"gae_loss_grad: dz must be a contiguous [{n_rows}, {d}] buffer, got {tuple(dz.shape)} strides {dz.stride()}")
    check(lib().b2_gae_loss_grad_f32(_p(z), _rowmajor(z, "z"), _p(mu), _p(logvar), ldm, *labs, n, d, row_begin, n_rows, float(norm),
                                     float(pos_weight), int(use_pos_weight), _p(dz), _p(dmu), _p(dlogvar), ldd, _p(loss), _p(ws),
                                     ws.numel(), _stream()), "b2_gae_loss_grad_f32")
    return loss, dz, dmu, dlogvar


def gae_sym_super_blocks(n: int) -> int:
    """Equal-work units of the pair-sharded decoder (super-block s = 128-row blocks s and nb−1−s; see gae_loss_grad_sym)."""
    return int(lib().b2_gae_sym_super_blocks(n))


def gae_loss_grad_sym(z, labels: CSR, norm: float, pos_weight: float, sb_begin: int, sb_end: int, mu=None, logvar=None,
                      use_pos_weight=True, dz_full=None, dmu=None, dlogvar=None, loss=None, row_begin: int = 0,
                      n_rows: Optional[int] = None, labels_t: Optional[CSR] = None):
    """Pair-sharded matrix-free Graph-AE loss (multi-GPU form of :func:`gae_loss_grad`): this rank evaluates super-blocks
    ``[sb_begin, sb_end)`` of the unordered block-pair schedule and the label / KLD terms of its rows.  Returns
    ``(loss_share[1], dz_full[n, d], dmu, dlogvar)``; all-reduce ``dz_full`` and ``loss_share`` over ranks.  Real-valued labels
    (``labels.vals`` set) need ``labels_t`` as in :func:`gae_loss_grad`."""
    n, d, n_rows, ldm, ldd, dmu, dlogvar, loss, ws, labs = _gae_prepare("gae_loss_grad_sym", z, labels, n_rows, mu, logvar, dmu,
                                                                        dlogvar, loss, labels_t)
    if dz_full is None:
        dz_full = torch.empty((n, d), dtype=torch.float32, device=z.device)
    _chk(dz_full, torch.float32, "dz_full", 2)
    if tuple(dz_full.shape) != (n, d) or not dz_full.is_contiguous():
        raise B2Error(f"gae_loss_grad_sym: dz_full must be a contiguous [{n}, {d}] buffer")
    check(lib().b2_gae_loss_grad_sym_f32(_p(z), _rowmajor(z, "z"), _p(mu), _p(logvar), ldm, *labs, n, d, sb_begin, sb_end,
                                         row_begin, n_rows, float(norm), float(pos_weight), int(use_pos_weight), _p(dz_full),
                                         _p(dmu), _p(dlogvar), ldd, _p(loss), _p(ws), ws.numel(), _stream()), "b2_gae_loss_grad_sym_f32")
    return loss, dz_full, dmu, dlogvar


def adam_step(param, grad, exp_avg, exp_avg_sq, step: int, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0):
    for t, nm in ((param, "param"), (grad, "grad"), (exp_avg, "exp_avg"), (exp_avg_sq, "exp_avg_sq")):
        _chk(t, torch.float32, nm)
        if not t.is_contiguous():
            raise B2Error(f"adam_step: {nm} must be contiguous")
    check(lib().b2_adam_step_f32(_p(param), _p(grad), _p(exp_avg), _p(exp_avg_sq), param.numel(), lr, beta1, beta2, eps,
                                 weight_decay, step, _stream()), "b2_adam_step_f32")


def relu_bwd(grad, y, out=None):
    _chk(grad, torch.float32, "grad")
    _chk(y, torch.float32, "y")
    if out is None:
        out = torch.empty_like(grad)
    check(lib().b2_relu_bwd_f32(_p(grad), _p(y), _p(out), grad.numel(), _stream()), "b2_relu_bwd_f32")
    return out


def reparam_fwd(mu, logvar, eps, out=None):
    n, d = mu.shape
    z = out if out is not None else torch.empty((n, d), dtype=torch.float32, device=mu.device)
    check(lib().b2_reparam_fwd_f32(_p(mu), _p(logvar), _rowmajor(mu, "mu"), _p(eps), _rowmajor(eps, "eps"), _p(z),
                                   _rowmajor(z, "z"), n, d, _stream()), "b2_reparam_fwd_f32")
    return z


def reparam_bwd(dz, logvar, eps, dmu, dlogvar):
    n, d = dz.shape
    check(lib().b2_reparam_bwd_f32(_p(dz), _rowmajor(dz, "dz"), _p(logvar), _rowmajor(logvar, "logvar"), _p(eps),
                                   _rowmajor(eps, "eps"), _p(dmu), _p(dlogvar), _rowmajor(dmu, "dmu"), n, d, _stream()),
          "b2_reparam_bwd_f32")


def knn(X: torch.Tensor, k: int, include_rank0: bool = False, q_begin: int = 0, q_end: Optional[int] = None,
        return_dist: bool = True):
    """Exact euclidean kNN of rows ``q_begin:q_end`` of X against all rows of X.

    Returns ``(idx[int32, n_q×k], dist[float64, n_q×k] or None)`` ranked by (fp64 distance, index).
    ``include_rank0=False`` drops sorted rank 0 — the reference's "self" slot (scgnn2.py:684-687).
    """
    _chk(X, torch.float32, "X", 2)
    n, d = X.shape
    q_end = n if q_end is None else q_end
    nq = q_end - q_begin
    idx = torch.empty((nq, k), dtype=torch.int32, device=X.device)
    dist = torch.empty((nq, k), dtype=torch.float64, device=X.device) if return_dist else None
    nbytes = lib().b2_knn_workspace_bytes(n, d, k, nq)
    ws = _workspace(nbytes, X.device)
    check(lib().b2_knn_l2_f32(_p(X), _rowmajor(X, "X"), n, d, k, q_begin, q_end, int(include_rank0), _p(idx), _p(dist),
                              _p(ws), ws.numel(), _stream()), "b2_knn_l2_f32")
    return idx, dist


def pairwise_l2_dense(X: torch.Tensor) -> torch.Tensor:
    _chk(X, torch.float32, "X", 2)
    n, d = X.shape
    D = torch.empty((n, n), dtype=torch.float32, device=X.device)
    check(lib().b2_pairwise_l2_dense_f32(_p(X), _rowmajor(X, "X"), n, d, _p(D), n, _stream()), "b2_pairwise_l2_dense_f32")
    return D


def knn_graph_build(knn_idx: torch.Tensor) -> CSR:
    """Union-symmetrised kNN adjacency + I with D^-1/2 (A+I) D^-1/2 values (scgnn2.py:650-672,1191-1198)."""
    _chk(knn_idx, torch.int32, "knn_idx", 2)
    if not knn_idx.is_contiguous():
        raise B2Error("knn_graph_build: knn_idx must be contiguous")
    n, k = knn_idx.shape
    cap = 2 * n * k + n
    dev = knn_idx.device
    rowptr = torch.empty(n + 1, dtype=torch.int32, device=dev)
    colidx = torch.empty(cap, dtype=torch.int32, device=dev)
    vals = torch.empty(cap, dtype=torch.float32, device=dev)
    nnz = C.c_int64(0)
    nbytes = lib().b2_knn_graph_workspace_bytes(n, k)
    ws = _workspace(nbytes, dev)
    check(lib().b2_knn_graph_build(_p(knn_idx), n, k, _p(rowptr), _p(colidx), _p(vals), cap, C.byref(nnz), _p(ws),
                                   ws.numel(), _stream()), "b2_knn_graph_build")
    m = nnz.value
    return CSR(rowptr, colidx[:m].clone(), vals[:m].clone(), (n, n))


class WeightedGraph(NamedTuple):
    """The weighted, directed kNN graph of ``graph_AE_retain_weights`` (see :func:`knn_graph_weighted_build`).  ``adj`` and
    ``labels_t`` share the target-row index arrays, ``adj_t`` and ``labels`` the source-row ones."""
    adj: CSR          # Â, rows = target: the forward aggregate
    adj_t: CSR        # Âᵀ, rows = source: the backward aggregate
    labels: CSR       # L = adj_train + I with its fp32 values, rows = source
    labels_t: CSR     # Lᵀ with its values, rows = target
    sum_w: torch.Tensor   # ΣW = adj_train.sum(), device fp64 [1]


def knn_graph_weighted_build(knn_idx: torch.Tensor, knn_dist: torch.Tensor) -> WeightedGraph:
    """feature2adj(retain_weights=True) + preprocess_graph (scgnn2.py:659-670, 1191-1198) from the kNN lists: W = 1/(d + 1e-16),
    directed, in cell order; Â = ((adj_train + I)·Dm)ᵀ·Dm with Dm = diag(rowsum^-1/2), evaluated in fp64, stored in fp32."""
    _chk(knn_idx, torch.int32, "knn_idx", 2)
    _chk(knn_dist, torch.float64, "knn_dist", 2)
    if not (knn_idx.is_contiguous() and knn_dist.is_contiguous()) or knn_idx.shape != knn_dist.shape:
        raise B2Error("knn_graph_weighted_build: knn_idx and knn_dist must be contiguous and of one shape")
    n, k = knn_idx.shape
    cap = n * (k + 1)
    dev = knn_idx.device
    i32 = lambda m: torch.empty(m, dtype=torch.int32, device=dev)
    f32 = lambda m: torch.empty(m, dtype=torch.float32, device=dev)
    rowptr, colidx, y, norm_t = i32(n + 1), i32(cap), f32(cap), f32(cap)
    t_rowptr, t_colidx, t_y, norm = i32(n + 1), i32(cap), f32(cap), f32(cap)
    sum_w = torch.empty(1, dtype=torch.float64, device=dev)
    nnz = C.c_int64(0)
    ws = _workspace(lib().b2_knn_graph_weighted_workspace_bytes(n, k), dev)
    check(lib().b2_knn_graph_weighted_build(_p(knn_idx), _p(knn_dist), n, k, _p(rowptr), _p(colidx), _p(y), _p(norm_t), _p(t_rowptr),
                                            _p(t_colidx), _p(t_y), _p(norm), _p(sum_w), cap, C.byref(nnz), _p(ws), ws.numel(),
                                            _stream()), "b2_knn_graph_weighted_build")
    m = nnz.value
    if m < cap:
        colidx, y, norm_t, t_colidx, t_y, norm = (t[:m].clone() for t in (colidx, y, norm_t, t_colidx, t_y, norm))
    return WeightedGraph(CSR(t_rowptr, t_colidx, norm, (n, n)), CSR(rowptr, colidx, norm_t, (n, n)), CSR(rowptr, colidx, y, (n, n)),
                         CSR(t_rowptr, t_colidx, t_y, (n, n)), sum_w)


def normalize_total_log1p_(X: torch.Tensor, target_sum: Optional[float] = None, max_fraction: float = 1.0,
                           normalize: bool = True, log1p: bool = True, base: Optional[float] = None) -> torch.Tensor:
    """In-place normalize_total (+log1p) on a dense CUDA matrix (cells × genes)."""
    _chk(X, torch.float32, "X", 2)
    n, g = X.shape
    nbytes = lib().b2_normalize_total_workspace_bytes(n, g)
    ws = _workspace(nbytes, X.device)
    check(lib().b2_normalize_total_log1p_f32(_p(X), _rowmajor(X, "X"), n, g, float(target_sum or 0.0), float(max_fraction),
                                             int(normalize), int(log1p), float(base or 0.0), _p(ws), ws.numel(),
                                             _stream()), "b2_normalize_total_log1p_f32")
    return X


# ----------------------------------------------------------------------------- GAT
SCORE_ACT = {"leakyrelu": 0, "sigmoid": 1}
SHIFT = {"global": 0, "segment": 1}


def _head_width(W: int, nheads: int, what: str) -> int:
    if nheads <= 0 or W % nheads:
        raise B2Error(f"{what}: width {W} is not a multiple of nheads={nheads}")
    return W // nheads


def _drop_prob(p) -> float:
    """nn.Dropout's check: a probability outside [0, 1] is a ValueError."""
    p = float(p)
    if not 0.0 <= p <= 1.0:
        raise ValueError(f"dropout probability has to be between 0 and 1, but got {p}")
    return p


def dropout(x, p: float, seed: int, key: int, out=None):
    """Inverted dropout of a 2-D (strided) matrix: ``out[r, c] = x[r, c] / (1 - p)`` where keep(seed, key, r, c), else 0.

    The keep bit is a counter-based draw (independent Bernoulli(1 - p) per element; see include/dance_b200.h), so calling this
    again with the same (seed, key) applies the same mask — which is how a backward pass drops its gradient.  ``out`` may be
    ``x`` (in place).  Over an [nnz, nheads] tensor with a GAT layer's attention key it materialises that layer's attention
    mask (scaled): entry (p, h) is the keep bit of the edge at CSR position p and head h."""
    _chk(x, torch.float32, "x", 2)
    p = _drop_prob(p)
    if out is None:
        out = torch.empty(x.shape, dtype=torch.float32, device=x.device)
    _chk(out, torch.float32, "out", 2)
    if tuple(out.shape) != tuple(x.shape):
        raise B2Error(f"dropout: out has shape {tuple(out.shape)}, expected {tuple(x.shape)}")
    check(lib().b2_dropout_f32(_p(x), _rowmajor(x, "x"), x.shape[0], x.shape[1], p, int(seed) & 0xFFFFFFFF, int(key) & 0xFFFFFFFF,
                               _p(out), _rowmajor(out, "out"), _stream()), "b2_dropout_f32")
    return out


def gat_scores(H, a_src, a_trg, nheads: int):
    """s_src[n,h] = <H[n,h,:], a_src[h,:]> (scgnn2.py:1016-1017)."""
    _chk(H, torch.float32, "H", 2)
    n, W = H.shape
    F = _head_width(W, nheads, "gat_scores")
    s_src = torch.empty((n, nheads), dtype=torch.float32, device=H.device)
    s_trg = torch.empty((n, nheads), dtype=torch.float32, device=H.device)
    check(lib().b2_gat_scores_f32(_p(H), _rowmajor(H, "H"), _p(a_src), _p(a_trg), n, nheads, F, _p(s_src), _p(s_trg), _stream()),
          "b2_gat_scores_f32")
    return s_src, s_trg


def gat_aggregate_fwd(T: CSR, H, s_src, s_trg, nheads: int, score_act="leakyrelu", slope=0.2, shift="global",
                      out=None, keep_alpha=True, dropout: float = 0.0, seed: Optional[int] = None, key: int = 0):
    """Fused edge softmax + aggregate on the target-indexed CSR ``T``; returns (out, alpha, gmax).

    ``gmax`` [1] is the global shift (``shift="global"``; -inf for a graph without edges) and is what
    :func:`gat_aggregate_bwd` needs to differentiate through it.

    ``seed`` given: attention dropout (scgnn2.py:1029) — ``out[v] = Σ drop(α)_e H[u]`` with the keep bit of (edge at CSR
    position p, head h) drawn as :func:`dropout` draws element (p, h) under (seed, key).  ``alpha`` stays undropped; pass
    the same (dropout, seed, key) to :func:`gat_aggregate_bwd`."""
    n, W = H.shape
    F = _head_width(W, nheads, "gat_aggregate_fwd")
    if seed is None and dropout:
        raise ValueError("gat_aggregate_fwd: attention dropout needs a seed")
    p = _drop_prob(dropout)
    if out is None:
        out = torch.empty((n, W), dtype=torch.float32, device=H.device)
    gmax = torch.empty(1, dtype=torch.float32, device=H.device)
    act, sm = SCORE_ACT[score_act], SHIFT[shift]
    colidx = _p(T.colidx) if T.nnz else _p(T.rowptr)  # an edgeless graph has no colidx storage; never dereferenced
    if sm == 0:
        check(lib().b2_gat_edge_max_f32(_p(T.rowptr), colidx, _p(s_src), _p(s_trg), n, nheads, act, slope, _p(gmax),
                                        _stream()), "b2_gat_edge_max_f32")
    alpha = torch.empty((T.nnz, nheads), dtype=torch.float32, device=H.device) if keep_alpha else None
    check(lib().b2_gat_aggregate_fwd_f32(_p(T.rowptr), colidx, _p(H), _rowmajor(H, "H"), _p(s_src), _p(s_trg), n, nheads, F, act, slope,
                                         sm, _p(gmax), _p(out), _rowmajor(out, "out"), _p(alpha) if T.nnz else None, p,
                                         int(seed or 0) & 0xFFFFFFFF, int(key) & 0xFFFFFFFF, _stream()), "b2_gat_aggregate_fwd_f32")
    return out, alpha, gmax


def gat_aggregate_bwd(T: CSR, Tt: CSR, t_perm, H, a_src, a_trg, s_src, s_trg, alpha, dOut, nheads: int,
                      score_act="leakyrelu", slope=0.2, H2=None, dOut2=None, want_dH2=True, gmax=None, dropout: float = 0.0,
                      seed: Optional[int] = None, key: int = 0):
    """Returns (dH, da_src, da_trg), or (dH, da_src, da_trg, dH2 | None) with a tied second layer (H2, dOut2).

    ``gmax``: the forward's global shift (third result of :func:`gat_aggregate_fwd` with ``shift="global"``), whose
    gradient the backward then includes, as the reference does not detach its max; None for ``shift="segment"``.
    ``dropout`` / ``seed`` / ``key``: the forward's attention dropout (not with a tied layer); ``alpha`` is the undropped α."""
    n, W = H.shape
    F = _head_width(W, nheads, "gat_aggregate_bwd")
    if seed is None and dropout:
        raise ValueError("gat_aggregate_bwd: attention dropout needs a seed")
    p = _drop_prob(dropout)
    dev = H.device
    dH = torch.empty((n, W), dtype=torch.float32, device=dev)
    da_src = torch.empty(W, dtype=torch.float32, device=dev)
    da_trg = torch.empty(W, dtype=torch.float32, device=dev)
    ds_s = torch.empty(n * nheads, dtype=torch.float32, device=dev)
    ds_t = torch.empty(n * nheads, dtype=torch.float32, device=dev)
    dpre = torch.empty(max(T.nnz, 1) * nheads, dtype=torch.float32, device=dev)
    shift_ws = torch.empty(2, dtype=torch.float32, device=dev) if gmax is not None else None
    # an edgeless graph has no colidx / t_perm / alpha storage: any non-NULL pointer stands in, never dereferenced
    edge = (lambda t: _p(t)) if T.nnz else (lambda t: _p(T.rowptr))
    tied = H2 is not None
    dH2 = torch.empty((n, W), dtype=torch.float32, device=dev) if tied and want_dH2 else None
    check(lib().b2_gat_aggregate_bwd_f32(_p(T.rowptr), edge(T.colidx), _p(Tt.rowptr), edge(Tt.colidx), edge(t_perm), _p(H),
                                         _rowmajor(H, "H"), _p(a_src), _p(a_trg), _p(s_src), _p(s_trg), edge(alpha), _p(dOut),
                                         _rowmajor(dOut, "dOut"), _p(H2), _rowmajor(H2, "H2") if tied else 0, _p(dOut2),
                                         _rowmajor(dOut2, "dOut2") if tied else 0, n, nheads, F, SCORE_ACT[score_act], slope, _p(gmax),
                                         _p(dH), _rowmajor(dH, "dH"), _p(dH2), _rowmajor(dH2, "dH2") if dH2 is not None else 0,
                                         _p(da_src), _p(da_trg), _p(ds_s), _p(ds_t), _p(dpre), _p(shift_ws), p,
                                         int(seed or 0) & 0xFFFFFFFF, int(key) & 0xFFFFFFFF, _stream()), "b2_gat_aggregate_bwd_f32")
    return (dH, da_src, da_trg, dH2) if tied else (dH, da_src, da_trg)


def gat_combine_fwd(agg, skip, bias, nheads: int, concat: bool, act=None, identity: bool = False):
    """``identity``: ``skip`` is the layer's raw input [n, F], added to every head (GATLayer with FIN == FOUT,
    scgnn2.py:1167-1171); otherwise ``skip`` is [n, nheads*F] or None."""
    n, W = agg.shape
    F = _head_width(W, nheads, "gat_combine_fwd")
    out = torch.empty((n, W if concat else F), dtype=torch.float32, device=agg.device)
    if identity:
        _chk(skip, torch.float32, "skip", 2)
        if tuple(skip.shape) != (n, F):
            raise B2Error(f"gat_combine_fwd: an identity skip must have shape {(n, F)}, got {tuple(skip.shape)}")
    check(lib().b2_gat_combine_fwd_f32(_p(agg), _rowmajor(agg, "agg"), _p(skip), _rowmajor(skip, "skip") if skip is not None else 0,
                                       _p(bias), n, nheads, F, int(concat), ACT[act], int(identity), _p(out), _rowmajor(out, "out"),
                                       _stream()), "b2_gat_combine_fwd_f32")
    return out


def gat_combine_bwd(dout, out, nheads: int, F: int, concat: bool, act=None, identity: bool = False, dpre=None, dx_skip=None):
    """Returns (dpre [n, nheads*F], dact [n, out width]); with ``identity`` also dx_skip [n, F] = Σ_h dpre[:, h·F:(h+1)·F],
    the identity skip's gradient of the layer input.  ``dpre`` / ``dx_skip``: optional (strided) output buffers."""
    n = dout.shape[0]
    if dpre is None:
        dpre = torch.empty((n, nheads * F), dtype=torch.float32, device=dout.device)
    dact = torch.empty_like(out)
    if not identity:
        dx_skip = None
    elif dx_skip is None:
        dx_skip = torch.empty((n, F), dtype=torch.float32, device=dout.device)
    check(lib().b2_gat_combine_bwd_f32(_p(dout), _rowmajor(dout, "dout"), _p(out), _rowmajor(out, "out"), n, nheads, F,
                                       int(concat), ACT[act], _p(dpre), _rowmajor(dpre, "dpre"), _p(dact), _rowmajor(dact, "dact"),
                                       _p(dx_skip), _rowmajor(dx_skip, "dx_skip") if identity else 0, _stream()),
          "b2_gat_combine_bwd_f32")
    return (dpre, dact, dx_skip) if identity else (dpre, dact)


# ----------------------------------------------------------------------------- scDeepSort path
def cellgene_graph(X: torch.Tensor, normalize_edges: bool = True):
    """CellFeatureGraph edge list (cell_feature_graph.py:34-79): returns (src int64, dst int64, w fp32 [E,1], nnz)."""
    _chk(X, torch.float32, "X", 2)
    n, g = X.shape
    nbytes = lib().b2_cellgene_graph_workspace_bytes(n, g)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=X.device)      # private: must survive between count and fill
    nnz = C.c_int64(0)
    check(lib().b2_cellgene_graph_count(_p(X), _rowmajor(X, "X"), n, g, C.byref(nnz), _p(ws), ws.numel(), _stream()),
          "b2_cellgene_graph_count")
    E = 2 * nnz.value + n + g
    src = torch.empty(E, dtype=torch.int64, device=X.device)
    dst = torch.empty(E, dtype=torch.int64, device=X.device)
    w = torch.empty((E, 1), dtype=torch.float32, device=X.device)
    check(lib().b2_cellgene_graph_fill(_p(X), _rowmajor(X, "X"), n, g, int(normalize_edges), nnz.value, _p(src), _p(dst), _p(w),
                                       _p(ws), ws.numel(), _stream()), "b2_cellgene_graph_fill")
    return src, dst, w, nnz.value


def sage_edge_values(T: CSR, w: torch.Tensor, alpha: torch.Tensor, n_genes: int) -> torch.Tensor:
    out = torch.empty(T.nnz, dtype=torch.float32, device=w.device)
    check(lib().b2_sage_edge_values_f32(_p(T.rowptr), _p(T.colidx), _p(w), _p(alpha), T.shape[0], n_genes, _p(out), _stream()),
          "b2_sage_edge_values_f32")
    return out


def softmax_ce_sum(logits: torch.Tensor, labels: torch.Tensor, dlogits: Optional[torch.Tensor] = None,
                   loss_out: Optional[torch.Tensor] = None, need_grad: bool = True):
    """CrossEntropyLoss(reduction='sum'): accumulates into loss_out[0]; returns (loss_out, dlogits)."""
    _chk(logits, torch.float32, "logits", 2)
    _chk(labels, torch.int64, "labels", 1)
    n, c = logits.shape
    if need_grad and dlogits is None:
        dlogits = torch.empty_like(logits)
    if loss_out is None:
        loss_out = torch.zeros(1, dtype=torch.float32, device=logits.device)
    check(lib().b2_softmax_ce_sum_f32(_p(logits), _rowmajor(logits, "logits"), _p(labels), n, c, _p(dlogits) if need_grad else None,
                                      _rowmajor(dlogits, "dlogits") if need_grad else 0, _p(loss_out), _stream()),
          "b2_softmax_ce_sum_f32")
    return loss_out, dlogits


# ----------------------------------------------------------------------------- PCA
def sym_eig(Cm: torch.Tensor, max_sweeps: int = 30, tol: float = 4e-6):
    """Eigen-decomposition of a symmetric matrix (destroyed) by parallel one-sided Jacobi.
    Returns (evals [g] descending, evecs [g,g] rows = eigenvectors in the same order, sweeps)."""
    _chk(Cm, torch.float32, "C", 2)
    g = Cm.shape[0]
    if Cm.shape[1] != g or not Cm.is_contiguous():
        raise B2Error("sym_eig: need a contiguous square matrix")
    V = torch.empty_like(Cm)
    ev = torch.empty(g, dtype=torch.float32, device=Cm.device)
    sweeps = C.c_int32(0)
    ws = _workspace(64, Cm.device)
    check(lib().b2_sym_eig_jacobi_f32(_p(Cm), _p(V), g, max_sweeps, tol, _p(ev), C.byref(sweeps), _p(ws), ws.numel(), _stream()),
          "b2_sym_eig_jacobi_f32")
    order = torch.argsort(ev, descending=True)
    return ev[order], V[order], sweeps.value


def pca(X: torch.Tensor, n_components: int, precision: Optional[str] = None):
    """PCA of X [n_samples, n_features] like sklearn.decomposition.PCA(n_components).fit_transform (centred, no whitening).

    Returns dict(scores [n,k] = U·S, components [k,f], explained_variance [k], mean [f]).  Uses the Gram matrix when
    n_samples <= n_features, the covariance matrix otherwise; signs follow sklearn's u-based svd_flip.
    """
    _chk(X, torch.float32, "X", 2)
    n, f = X.shape
    k = int(n_components)
    mean = colsum(X) / float(n)
    if n <= f:
        # Gram side: K = Xc Xcᵀ with Xc = X - 1·meanᵀ  → K = X Xᵀ - s 1ᵀ - 1 sᵀ + (m·m) 1 1ᵀ, s = X·mean
        Xc = X - mean                                        # n ≤ f: the centred copy is the small side's operand
        K = gemm(Xc, Xc, transB=True, precision=precision)
        ev, evec, _ = sym_eig(K)
        ev = ev[:k].clamp_min(0)
        U = evec[:k]                                          # rows = left singular vectors
        S = ev.sqrt()
        scores = (U * S[:, None]).t().contiguous()            # [n, k] = U·S
        comps = gemm(U, Xc, precision=precision) / S.clamp_min(1e-30)[:, None]   # Vᵀ = Σ^-1 Uᵀ Xc
    else:
        Cm = gemm(X, X, transA=True, precision=precision)     # XᵀX  [f,f]
        check(lib().b2_cov_rank1_sub_f32(_p(Cm), _p(mean), f, float(n), _stream()), "b2_cov_rank1_sub_f32")
        ev, evec, _ = sym_eig(Cm)
        ev = ev[:k].clamp_min(0)
        comps = evec[:k].contiguous()                         # [k, f]
        bias = -(comps @ mean)
        scores = gemm(X, comps, transB=True, bias=bias.contiguous(), precision=precision)   # (X - mean)·Vᵀ
    # sklearn svd_flip (u-based): make the largest-|.| entry of every score column positive
    idx = scores.abs().argmax(0)
    sign = torch.sign(scores[idx, torch.arange(k, device=X.device)])
    sign[sign == 0] = 1
    return {"scores": scores * sign, "components": comps * sign[:, None], "explained_variance": ev / max(n - 1, 1), "mean": mean}


# ----------------------------------------------------------------------------- SpaGCN (DEC head)
def dec_q(z, mu, alpha: float = 0.2):
    n, h = z.shape
    K = mu.shape[0]
    q = torch.empty((n, K), dtype=torch.float32, device=z.device)
    check(lib().b2_dec_q_f32(_p(z), _rowmajor(z, "z"), _p(mu), n, K, h, alpha, _p(q), K, _stream()), "b2_dec_q_f32")
    return q


def dec_target(q):
    n, K = q.shape
    p = torch.empty_like(q)
    cs = colsum(q)
    check(lib().b2_dec_target_f32(_p(q), _rowmajor(q, "q"), _p(cs), n, K, _p(p), K, _stream()), "b2_dec_target_f32")
    return p


def dec_kl_grad(z, mu, p, alpha: float = 0.2, dz=None, dmu=None, loss=None, q_out=None, labels_out=None):
    n, h = z.shape
    K = mu.shape[0]
    dz = torch.empty((n, h), dtype=torch.float32, device=z.device) if dz is None else dz
    dmu = torch.empty((K, h), dtype=torch.float32, device=z.device) if dmu is None else dmu
    loss = torch.empty(1, dtype=torch.float32, device=z.device) if loss is None else loss
    check(lib().b2_dec_kl_grad_f32(_p(z), _rowmajor(z, "z"), _p(mu), _p(p), _rowmajor(p, "p"), n, K, h, alpha, _p(q_out),
                                   _rowmajor(q_out, "q_out") if q_out is not None else 0, _p(dz), _rowmajor(dz, "dz"), _p(dmu), _p(loss),
                                   _p(labels_out), _stream()), "b2_dec_kl_grad_f32")
    return loss, dz, dmu


def sgd_momentum_step(param, grad, buf, step: int, lr: float, momentum: float = 0.9, weight_decay: float = 0.0):
    check(lib().b2_sgd_momentum_step_f32(_p(param), _p(grad), _p(buf), param.numel(), lr, momentum, weight_decay, step, _stream()),
          "b2_sgd_momentum_step_f32")


def exp_adj(D: torch.Tensor, l: float, want_matrix: bool = True, want_sum: bool = False):
    """exp(-D²/(2l²)) elementwise on a dense distance matrix and / or its total sum (fp64)."""
    _chk(D, torch.float32, "D")
    if not D.is_contiguous():
        raise B2Error("exp_adj: D must be contiguous")
    out = torch.empty_like(D) if want_matrix else None
    acc = torch.zeros(1, dtype=torch.float64, device=D.device) if want_sum else None
    check(lib().b2_exp_adj_f32(_p(D), _p(out), D.numel(), float(l), _p(acc), _stream()), "b2_exp_adj_f32")
    return out, acc


def clip_grad_norm_(grad: torch.Tensor, max_norm: float, pre_scale: float = 1.0, norm_out: Optional[torch.Tensor] = None):
    """In-place ``clip_grad_norm_`` over one flat bucket (after multiplying it by ``pre_scale``)."""
    _chk(grad, torch.float32, "grad")
    ws = torch.empty(1, dtype=torch.float64, device=grad.device)
    check(lib().b2_clip_grad_norm_f32(_p(grad), grad.numel(), float(pre_scale), float(max_norm), _p(ws), _p(norm_out), _stream()),
          "b2_clip_grad_norm_f32")
    return grad


def radius_graph(X: torch.Tensor, radius: float) -> "CSR":
    """Unit-weight CSR of all pairs within ``radius`` (self included); ``X`` is [n, d<=4] float64 on the device."""
    _chk(X, torch.float64, "X", 2)
    n, d = X.shape
    if n == 0:
        return CSR(torch.zeros(1, dtype=torch.int32, device=X.device), torch.empty(0, dtype=torch.int32, device=X.device),
                   torch.empty(0, dtype=torch.float32, device=X.device), (0, 0))
    ws = _workspace(lib().b2_radius_graph_workspace_bytes(n), X.device)
    rowptr = torch.empty(n + 1, dtype=torch.int32, device=X.device)
    nnz = C.c_int64(0)
    check(lib().b2_radius_graph_count(_p(X), _rowmajor(X, "X"), n, d, float(radius), _p(rowptr), C.addressof(nnz), _p(ws),
                                      ws.numel(), _stream()), "b2_radius_graph_count")
    colidx = torch.empty(max(nnz.value, 1), dtype=torch.int32, device=X.device)[:nnz.value]
    if nnz.value:
        check(lib().b2_radius_graph_fill(_p(X), _rowmajor(X, "X"), n, d, float(radius), _p(rowptr), _p(colidx), _stream()),
              "b2_radius_graph_fill")
    vals = torch.ones(nnz.value, dtype=torch.float32, device=X.device)
    return CSR(rowptr, colidx, vals, (n, n))


NORM_MODE = {"normalize": 0, "standardize": 1, "minmax": 2, "l2": 3}


def matrix_normalize(X: torch.Tensor, mode: str = "normalize", axis: int = 0, eps: float = -1.0, out: Optional[torch.Tensor] = None):
    """``dance.utils.matrix.normalize`` on a CUDA fp32 matrix (utils/matrix.py:8-67)."""
    _chk(X, torch.float32, "X", 2)
    if mode not in NORM_MODE:
        raise B2Error(f"matrix_normalize: unknown mode {mode!r}")
    if not (eps == -1 or eps > 0):
        raise ValueError(f"Invalid {eps=!r}. Must be positive or -1, the later set zero entries to one.")
    n, g = X.shape
    out = torch.empty_like(X) if out is None else out
    ws = _workspace(lib().b2_matrix_normalize_workspace_bytes(n, g, axis), X.device)
    check(lib().b2_matrix_normalize_f32(_p(X), _rowmajor(X, "X"), n, g, NORM_MODE[mode], int(axis), float(eps), _p(out),
                                        _rowmajor(out, "out"), _p(ws), ws.numel(), _stream()), "b2_matrix_normalize_f32")
    return out


def pearson_corr(X: torch.Tensor) -> torch.Tensor:
    """float32(np.corrcoef(X.T)) for X [n, g] — fp64 arithmetic on the device."""
    _chk(X, torch.float32, "X", 2)
    n, g = X.shape
    adj = torch.empty((g, g), dtype=torch.float32, device=X.device)
    ws = torch.empty(lib().b2_pearson_corr_workspace_bytes(g), dtype=torch.uint8, device=X.device)
    check(lib().b2_pearson_corr_f32(_p(X), _rowmajor(X, "X"), n, g, _p(adj), g, _p(ws), ws.numel(), _stream()), "b2_pearson_corr_f32")
    return adj


def threshold_graph(adj: torch.Tensor, threshold: float, positive_only: bool = False, normalize_edges: bool = True):
    """Edges of a dense score matrix after thresholding: (src int32, dst int32, w fp32), row-major order."""
    _chk(adj, torch.float32, "adj", 2)
    g = adj.shape[0]
    ws = torch.empty(lib().b2_threshold_graph_workspace_bytes(g), dtype=torch.uint8, device=adj.device)   # survives count → fill
    rowptr = torch.empty(g + 1, dtype=torch.int32, device=adj.device)
    nnz = C.c_int64(0)
    check(lib().b2_threshold_graph_count(_p(adj), _rowmajor(adj, "adj"), g, float(threshold), int(positive_only), _p(rowptr),
                                         C.addressof(nnz), _p(ws), ws.numel(), _stream()), "b2_threshold_graph_count")
    E = nnz.value
    src = torch.empty(max(E, 1), dtype=torch.int32, device=adj.device)[:E]
    dst = torch.empty(max(E, 1), dtype=torch.int32, device=adj.device)[:E]
    w = torch.empty(max(E, 1), dtype=torch.float32, device=adj.device)[:E]
    if E:
        check(lib().b2_threshold_graph_fill(_p(adj), _rowmajor(adj, "adj"), g, float(threshold), int(positive_only), _p(rowptr),
                                            int(normalize_edges), _p(src), _p(dst), _p(w), _p(ws), ws.numel(), _stream()),
              "b2_threshold_graph_fill")
    return src, dst, w, rowptr


def umap_connectivities(knn_idx: torch.Tensor, knn_dist: torch.Tensor) -> "CSR":
    """scanpy/umap fuzzy-simplicial-set connectivities from a kNN table whose column 0 is the cell itself."""
    _chk(knn_idx, torch.int32, "knn_idx", 2)
    _chk(knn_dist, torch.float32, "knn_dist", 2)
    n, k = knn_idx.shape
    dev = knn_idx.device
    vals = torch.empty((n, k), dtype=torch.float32, device=dev)
    sig = torch.empty(n, dtype=torch.float32, device=dev)
    rho = torch.empty(n, dtype=torch.float32, device=dev)
    acc = torch.empty(1, dtype=torch.float64, device=dev)
    check(lib().b2_umap_fuzzy_knn_f32(_p(knn_idx), _p(knn_dist), n, k, _p(vals), _p(sig), _p(rho), _p(acc), _stream()),
          "b2_umap_fuzzy_knn_f32")
    rowptr = torch.arange(0, n * k + 1, k, dtype=torch.int32, device=dev)
    A0 = CSR(rowptr, knn_idx.reshape(-1).contiguous(), vals.reshape(-1), (n, n))
    T, _ = csr_transpose(A0)          # Aᵀ, ascending columns
    A, _ = csr_transpose(T)           # A again, now with ascending columns too
    ws = torch.empty(lib().b2_fuzzy_union_workspace_bytes(n), dtype=torch.uint8, device=dev)
    rp = torch.empty(n + 1, dtype=torch.int32, device=dev)
    nnz = C.c_int64(0)
    check(lib().b2_fuzzy_union_count(_p(A.rowptr), _p(A.colidx), _p(A.vals), _p(T.rowptr), _p(T.colidx), _p(T.vals), n, _p(rp),
                                     C.addressof(nnz), _p(ws), ws.numel(), _stream()), "b2_fuzzy_union_count")
    E = nnz.value
    ci = torch.empty(max(E, 1), dtype=torch.int32, device=dev)[:E]
    cv = torch.empty(max(E, 1), dtype=torch.float32, device=dev)[:E]
    if E:
        check(lib().b2_fuzzy_union_fill(_p(A.rowptr), _p(A.colidx), _p(A.vals), _p(T.rowptr), _p(T.colidx), _p(T.vals), n, _p(rp),
                                        _p(ci), _p(cv), _stream()), "b2_fuzzy_union_fill")
    out = CSR(rp, ci, cv, (n, n))
    out.sigmas, out.rhos = sig, rho
    return out


# ----------------------------------------------------------------------------- GraphSCI path
def batchnorm_fwd(X, gamma, beta, running_mean, running_var, training: bool, momentum: float = 0.1, eps: float = 1e-5,
                  act: Optional[str] = None):
    """nn.BatchNorm1d (+ optional fused ReLU); returns (out, save_mean, save_invstd)."""
    _chk(X, torch.float32, "X", 2)
    n, c = X.shape
    out = torch.empty_like(X)
    sm = torch.empty(c, dtype=torch.float32, device=X.device)
    si = torch.empty(c, dtype=torch.float32, device=X.device)
    ws = _workspace(lib().b2_batchnorm_workspace_bytes(c), X.device)
    check(lib().b2_batchnorm_fwd_f32(_p(X), _rowmajor(X, "X"), n, c, _p(gamma), _p(beta), _p(running_mean), _p(running_var),
                                     int(training), momentum, eps, ACT[act], _p(out), _rowmajor(out, "out"), _p(sm), _p(si), _p(ws),
                                     ws.numel(), _stream()), "b2_batchnorm_fwd_f32")
    return out, sm, si


def batchnorm_bwd(dY, Y, X, gamma, save_mean, save_invstd, act: Optional[str] = None, training: bool = True, dgamma=None, dbeta=None):
    """Returns (dX, dgamma, dbeta); ``Y`` (the forward output) is only read for the fused ReLU."""
    n, c = X.shape
    dX = torch.empty_like(X)
    dgamma = torch.empty(c, dtype=torch.float32, device=X.device) if dgamma is None else dgamma
    dbeta = torch.empty(c, dtype=torch.float32, device=X.device) if dbeta is None else dbeta
    ws = _workspace(lib().b2_batchnorm_workspace_bytes(c), X.device)
    check(lib().b2_batchnorm_bwd_f32(_p(dY), _rowmajor(dY, "dY"), _p(Y), _rowmajor(Y, "Y") if Y is not None else 0, _p(X),
                                     _rowmajor(X, "X"), n, c, _p(gamma), _p(save_mean), _p(save_invstd), ACT[act], int(training), _p(dX),
                                     _rowmajor(dX, "dX"), _p(dgamma), _p(dbeta), _p(ws), ws.numel(), _stream()), "b2_batchnorm_bwd_f32")
    return dX, dgamma, dbeta


def zinb_loss_grad(a_pi, b_disp, c_mean, Y, size_factors, mask=None, le: float = 1.0, ke: float = 1.0, want_grad: bool = True,
                   want_outputs: bool = False):
    """Returns (acc3 fp64 {Σnll, Σmse, count}, (d_a, d_b, d_c) | None, (mean, disp, pi) | None)."""
    n, g = a_pi.shape
    dev = a_pi.device
    acc = torch.empty(3, dtype=torch.float64, device=dev)
    grads = tuple(torch.empty_like(a_pi) for _ in range(3)) if want_grad else (None, None, None)
    outs = tuple(torch.empty_like(a_pi) for _ in range(3)) if want_outputs else (None, None, None)
    if mask is not None:
        if mask.dtype == torch.bool:
            mask = mask.view(torch.uint8)
        _chk(mask, torch.uint8, "mask", 2)
    check(lib().b2_zinb_loss_grad_f32(_p(a_pi), _p(b_disp), _p(c_mean), _rowmajor(a_pi, "a_pi"), _p(Y), _rowmajor(Y, "Y"),
                                      _p(size_factors), _p(mask), mask.stride(0) if mask is not None else 0, n, g, le, ke, _p(grads[0]),
                                      _p(grads[1]), _p(grads[2]), g, _p(outs[0]), _p(outs[1]), _p(outs[2]), g, _p(acc), _stream()),
          "b2_zinb_loss_grad_f32")
    return acc, (grads if want_grad else None), (outs if want_outputs else None)


def adj_sample(mu, log_std, eps):
    for t, name in ((mu, "mu"), (log_std, "log_std"), (eps, "eps")):
        _chk(t, torch.float32, f"adj_sample: {name}")
        if t.numel() != mu.numel() or not t.is_contiguous():
            raise B2Error(f"adj_sample: {name} must be a contiguous tensor of {mu.numel()} elements")
    z = torch.empty_like(mu)
    check(lib().b2_adj_sample_f32(_p(mu), _p(log_std), _p(eps), mu.numel(), _p(z), _stream()), "b2_adj_sample_f32")
    return z


def adj_loss_grad(z, mu, log_std, target, class_weight, coef_ce: float = 0.0, want_grad: bool = True):
    """Returns (acc2 fp64 {Σ CE, Σ KL terms}, dz | None) for the [g, g] adjacency logits."""
    g = z.shape[0]
    acc = torch.empty(2, dtype=torch.float64, device=z.device)
    dz = torch.empty_like(z) if want_grad else None
    check(lib().b2_adj_loss_grad_f32(_p(z), _p(mu), _p(log_std), _p(target), _p(class_weight), g, coef_ce, _p(dz), _p(acc), _stream()),
          "b2_adj_loss_grad_f32")
    return acc, dz


def adj_reparam_bwd(dz, mu, log_std, eps, coef_kl: float):
    dmu, dls = torch.empty_like(mu), torch.empty_like(mu)
    check(lib().b2_adj_reparam_bwd_f32(_p(dz), _p(mu), _p(log_std), _p(eps), mu.numel(), coef_kl, _p(dmu), _p(dls), _stream()),
          "b2_adj_reparam_bwd_f32")
    return dmu, dls


# ----------------------------------------------------------------------------- scGNN EM-iteration stages (csrc/em.cu)
def kmeans(X: torch.Tensor, centers: torch.Tensor, max_iter: int = 300, tol: float = 1e-4):
    """Lloyd iterations of ``sklearn.cluster.KMeans(init=centers, n_init=1)`` on the device (scgnn2.py:186).

    ``centers`` [k, d] is updated in place.  Stops when no label changes or when ‖ΔC‖² ≤ tol·mean(var(X, axis=0)) (sklearn's
    rule), then runs a final assignment so that labels are consistent with the returned centres.
    Returns (labels int32 [n], inertia float, n_iter)."""
    _chk(X, torch.float32, "X", 2)
    _chk(centers, torch.float32, "centers", 2)
    n, d = X.shape
    k = centers.shape[0]
    if centers.shape[1] != d or not centers.is_contiguous():
        raise B2Error("kmeans: centers must be a contiguous [k, d] tensor")
    labels = torch.full((n, ), -1, dtype=torch.int32, device=X.device)
    stats = torch.zeros(3, dtype=torch.float64, device=X.device)
    nbytes = lib().b2_kmeans_workspace_bytes(k, d)
    ws = _workspace(nbytes, X.device)
    tol_abs = float(tol * X.var(dim=0, unbiased=False).mean().item())

    def step(update):
        check(lib().b2_kmeans_step_f32(_p(X), _rowmajor(X, "X"), n, d, _p(centers), k, _p(labels), int(update), _p(stats), _p(ws),
                                       ws.numel(), _stream()), "b2_kmeans_step_f32")
        return stats.tolist()

    it = 0
    for it in range(1, max_iter + 1):
        inertia, shift2, changed = step(True)
        if changed == 0 or shift2 <= tol_abs:
            break
    inertia, _, _ = step(False)
    return labels, inertia, it


def graph_regu_weights(A: CSR, labels: torch.Tensor, n_clusters: Optional[int] = None) -> torch.Tensor:
    """Per-cell column sums, inside the cell's own cluster, of the reference's "normalised" adjacency deg_j / deg_i
    (see b2_graph_regu_weights_f32): w_j = deg_j · Σ_{i ∈ cluster(j)} 1/deg_i."""
    _chk(labels, torch.int32, "labels", 1)
    n = A.shape[0]
    if n_clusters is None:
        n_clusters = int(labels.max().item()) + 1 if n else 1
    w = torch.empty(n, dtype=torch.float32, device=labels.device)
    sums = torch.empty(max(n_clusters, 1), dtype=torch.float64, device=labels.device)
    check(lib().b2_graph_regu_weights_f32(_p(A.rowptr), _p(A.colidx), _p(labels), n, int(n_clusters), _p(sums), _p(w), _stream()),
          "b2_graph_regu_weights_f32")
    return w


def graph_regu_weights_weighted(rowptr: torch.Tensor, colidx: torch.Tensor, vals: torch.Tensor, labels: torch.Tensor,
                                n_clusters: Optional[int] = None) -> torch.Tensor:
    """:func:`graph_regu_weights` for a weighted, directed adjacency (CSR with fp64 ``vals``, the ``adj`` of
    graph_AE_retain_weights): w_j = colsum_j · Σ_{i ∈ cluster(j)} 1/rowsum_i (see b2_graph_regu_weights_weighted_f32)."""
    _chk(labels, torch.int32, "labels", 1)
    _chk(rowptr, torch.int32, "rowptr", 1)
    _chk(colidx, torch.int32, "colidx", 1)
    _chk(vals, torch.float64, "vals", 1)
    n = rowptr.numel() - 1
    if labels.numel() != n or vals.numel() != colidx.numel():
        raise B2Error(f"graph_regu_weights_weighted: {n} rows but {labels.numel()} labels, or values and columns differ in length")
    if n_clusters is None:
        n_clusters = int(labels.max().item()) + 1 if n else 1
    w = torch.empty(n, dtype=torch.float32, device=labels.device)
    scratch = torch.empty(n + max(n_clusters, 1), dtype=torch.float64, device=labels.device)
    check(lib().b2_graph_regu_weights_weighted_f32(_p(rowptr), _p(colidx) if colidx.numel() else _p(rowptr),
                                                   _p(vals) if vals.numel() else _p(scratch), _p(labels), n, int(n_clusters),
                                                   _p(scratch), _p(w), _stream()), "b2_graph_regu_weights_weighted_f32")
    return w


def celltype_loss_grad(recon, target, x_dropout, row_weight, relu_mask=True, grad=None, loss_out=None):
    """loss_function_graph(regularizer_type="Celltype") (scgnn2.py:1316-1326): returns (loss_out[1] accumulated, d loss / d recon)."""
    for t, nm in ((recon, "recon"), (target, "target"), (x_dropout, "x_dropout")):
        _chk(t, torch.float32, nm, 2)
        if not t.is_contiguous():
            raise B2Error(f"celltype_loss_grad: {nm} must be contiguous")
    _chk(row_weight, torch.float32, "row_weight", 1)
    rows, cols = recon.shape
    if target.shape != recon.shape or x_dropout.shape[0] != rows or row_weight.shape[0] != rows or x_dropout.shape[1] > cols:
        raise B2Error("celltype_loss_grad: shape mismatch")
    if grad is None:
        grad = torch.empty_like(recon)
    if loss_out is None:
        loss_out = torch.zeros(1, dtype=torch.float32, device=recon.device)
    scratch = torch.empty(2, dtype=torch.float64, device=recon.device)
    check(lib().b2_celltype_loss_grad_f32(_p(recon), _p(target), _p(x_dropout), _p(row_weight), rows, cols, x_dropout.shape[1],
                                          int(relu_mask), _p(grad), _p(loss_out), _p(scratch), _stream()), "b2_celltype_loss_grad_f32")
    return loss_out, grad


def l1_grad_add(param, grad, coef: float = 1.0, l1_out=None):
    _chk(param, torch.float32, "param")
    _chk(grad, torch.float32, "grad")
    if not (param.is_contiguous() and grad.is_contiguous()) or param.numel() != grad.numel():
        raise B2Error("l1_grad_add: param / grad must be contiguous and equally sized")
    check(lib().b2_l1_grad_add_f32(_p(param), _p(grad), param.numel(), float(coef), _p(l1_out), _stream()), "b2_l1_grad_add_f32")


def louvain_host(indptr, indices, weights=None, max_levels: int = 0, min_gain: float = 1e-7):
    """Multilevel Louvain on a symmetric CSR in host memory (numpy arrays): returns (labels int32 [n], n_communities, modularity)."""
    import numpy as np
    indptr = np.ascontiguousarray(indptr, dtype=np.int64)
    indices = np.ascontiguousarray(indices, dtype=np.int32)
    w = None if weights is None else np.ascontiguousarray(weights, dtype=np.float64)
    n = indptr.shape[0] - 1
    labels = np.empty(n, dtype=np.int32)
    nc, mod = C.c_int32(), C.c_double()
    check(lib().b2_louvain_csr_host(indptr.ctypes.data, indices.ctypes.data, None if w is None else w.ctypes.data, n, labels.ctypes.data,
                                    C.byref(nc), C.byref(mod), int(max_levels), float(min_gain)), "b2_louvain_csr_host")
    return labels, nc.value, mod.value


# ----------------------------------------------------------------------------- pre-processing reductions (csrc/prep.cu)
def gene_stats(X: torch.Tensor, want_sumsq: bool = True, want_nnz: bool = True):
    """Per-gene (column) Σx, Σx², #(x>0) in fp64: returns (sum, sumsq | None, nnz | None)."""
    _chk(X, torch.float32, "X", 2)
    n, g = X.shape
    mk = lambda: torch.empty(g, dtype=torch.float64, device=X.device)
    s, q, k = mk(), (mk() if want_sumsq else None), (mk() if want_nnz else None)
    check(lib().b2_gene_stats_f32(_p(X), _rowmajor(X, "X"), n, g, _p(s), _p(q), _p(k), _stream()), "b2_gene_stats_f32")
    return s, q, k


def cell_stats(X: torch.Tensor, want_nnz: bool = True):
    """Per-cell (row) Σx and #(x>0) in fp64."""
    _chk(X, torch.float32, "X", 2)
    n, g = X.shape
    s = torch.empty(n, dtype=torch.float64, device=X.device)
    k = torch.empty(n, dtype=torch.float64, device=X.device) if want_nnz else None
    check(lib().b2_cell_stats_f32(_p(X), _rowmajor(X, "X"), n, g, _p(s), _p(k), _stream()), "b2_cell_stats_f32")
    return s, k


def subset(X: torch.Tensor, rows: Optional[torch.Tensor] = None, cols: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``X[rows][:, cols]`` as a new dense matrix (``None`` keeps the axis)."""
    _chk(X, torch.float32, "X", 2)
    if rows is not None:
        _chk(rows, torch.int64, "rows", 1)
    if cols is not None:
        _chk(cols, torch.int32, "cols", 1)
    n_out = X.shape[0] if rows is None else rows.numel()
    g_out = X.shape[1] if cols is None else cols.numel()
    out = torch.empty((n_out, g_out), dtype=torch.float32, device=X.device)
    check(lib().b2_subset_f32(_p(X), _rowmajor(X, "X"), _p(rows), _p(cols), n_out, g_out, _p(out), max(g_out, 1), _stream()), "b2_subset_f32")
    return out


def cellwise_mask(X: torch.Tensor, mask_rate: float = 0.1, min_gene_counts: int = 5, distr: str = "exp", add_test_mask: bool = False,
                  seed: int = 0):
    """CellwiseMaskData masks (train, valid, test) as bool [n, g] device tensors."""
    _chk(X, torch.float32, "X", 2)
    if distr not in ("exp", "uniform"):
        raise ValueError(f"Unknown distribution function option {distr!r}, available options are: 'exp', 'uniform'")
    n, g = X.shape
    mk = lambda: torch.empty((n, g), dtype=torch.uint8, device=X.device)
    tr, va, te = mk(), mk(), mk()
    over = torch.zeros(1, dtype=torch.int32, device=X.device)
    check(lib().b2_cellwise_mask_u8(_p(X), _rowmajor(X, "X"), n, g, float(mask_rate), int(min_gene_counts), int(distr == "exp"),
                                    int(add_test_mask), int(seed) & 0xFFFFFFFF, _p(tr), _p(va), _p(te), _p(over), _stream()),
          "b2_cellwise_mask_u8")
    return tr.view(torch.bool), va.view(torch.bool), te.view(torch.bool), int(over.item())


def locality_order(X: torch.Tensor, n_anchors: int = 64, iters: int = 4, seed: int = 0):
    """A cell order that keeps each thread block's gathers of the aggregate inside a few L2-resident row ranges: cells are grouped
    by their nearest of ``n_anchors`` centroids (a few Lloyd iterations from seeded random rows, ``b2_kmeans_step_f32``) and the
    groups laid out contiguously.  Returns (perm, inv): row i of the reordered problem is cell ``perm[i]``; ``inv[perm] = arange``.
    Relabelling a kNN index table: ``inv[idx[perm]]``.  The graph and every quantity derived from it are permutation-equivariant,
    so a model run in this order and un-permuted at the end returns the same result (up to summation order)."""
    _chk(X, torch.float32, "X", 2)
    n = X.shape[0]
    k = max(1, min(n_anchors, n))
    g = torch.Generator(device=X.device).manual_seed(seed)
    centers = X[torch.randperm(n, device=X.device, generator=g)[:k]].contiguous().clone()
    labels, _, _ = kmeans(X, centers, max_iter=iters, tol=0.0)
    perm = torch.sort(labels.long(), stable=True).indices
    inv = torch.empty_like(perm)
    inv[perm] = torch.arange(n, device=X.device)
    return perm, inv


# ---- scGNN's normalizer(X, base) and the concatenations that use it (scgnn2.py:155-157, 283-294, 543-546, 795-805) ------------
def _quantiles_launch(base: torch.Tensor, qs, out: torch.Tensor) -> None:
    """Enqueue b2_quantiles_f32 for one or two q: ``out`` (device doubles) receives the quantiles, min, max, #non-finite."""
    _chk(base, torch.float32, "base", 2)
    rows, cols = base.shape
    if rows == 0 or cols == 0:
        raise ValueError("quantiles: base is empty")
    qh = (C.c_float * len(qs))(*[float(q) for q in qs])
    nbytes = lib().b2_quantiles_workspace_bytes()
    ws = _workspace(nbytes, base.device)
    check(lib().b2_quantiles_f32(_p(base), _rowmajor(base, "base"), rows, cols, qh, len(qs), _p(out), _p(ws), ws.numel(), _stream()),
          "b2_quantiles_f32")


def quantiles(base: torch.Tensor, qs) -> "np.ndarray":
    """``np.quantile(base, q)`` (method "linear") for every q of ``qs`` over ALL elements of the (row-padded) fp32 matrix ``base``,
    bit for bit, as a float32 numpy array.  A zero comes back as +0.0 whatever its sign in ``base``.  Synchronises once per pair
    of q; a non-finite element raises ``ValueError`` (numpy would return NaN)."""
    import numpy as np
    qs = [float(np.float32(q)) for q in np.atleast_1d(np.asarray(qs, dtype=np.float64))]
    if not all(0.0 <= q <= 1.0 for q in qs):
        raise ValueError("Quantiles must be in the range [0, 1]")
    res = []
    for j in range(0, len(qs), 2):
        pair = qs[j:j + 2]
        out = torch.empty(len(pair) + 3, dtype=torch.float64, device=base.device)
        _quantiles_launch(base, pair, out)
        vals = out.tolist()
        if vals[-1] > 0:
            raise ValueError(f"quantiles: base holds {int(vals[-1])} non-finite values")
        res.extend(vals[:len(pair)])
    return np.asarray(res, dtype=np.float32)


def col_minmax(x: torch.Tensor, nonfinite: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Per-column (min, max) of a 2-D fp32 matrix ignoring NaN (np.nanmin / np.nanmax); ``nonfinite``: an optional device double
    that receives the number of non-finite elements."""
    _chk(x, torch.float32, "x", 2)
    rows, cols = x.shape
    cmin = torch.empty(cols, dtype=torch.float32, device=x.device)
    cmax = torch.empty(cols, dtype=torch.float32, device=x.device)
    ws = _workspace(lib().b2_col_minmax_workspace_bytes(cols), x.device)
    check(lib().b2_col_minmax_f32(_p(x), _rowmajor(x, "x"), rows, cols, _p(cmin), _p(cmax), _p(nonfinite), _p(ws), ws.numel(),
                                  _stream()), "b2_col_minmax_f32")
    return cmin, cmax


def _feature_range(base: torch.Tensor, upper: float, lower: float, bmin: float, bmax: float):
    """normalizer's feature range (scgnn2.py:797-804): (q0.1, q0.9) of base, or (q0, q1) when those two are equal.  q1 is the
    maximum (numpy's lerp adds a zero to it) and q0 the minimum plus (second smallest − minimum)·0 — the minimum unless that
    difference overflows, which only a second selection can settle.  Raises like MinMaxScaler for an empty range."""
    import numpy as np
    f32 = np.float32
    if f32(upper) != f32(lower):
        lo, hi = f32(lower), f32(upper)
    else:
        hi = f32(bmax) + f32(0)
        with np.errstate(over="ignore"):
            spread = f32(bmax) - f32(bmin)
        lo = f32(bmin) + f32(0) if np.isfinite(spread) else quantiles(base, [0.0])[0]
    if lo >= hi:
        raise ValueError(f"Minimum of desired feature range must be smaller than maximum. Got {(lo, hi)}.")
    return float(lo), float(hi)


def concat_normalized(left: torch.Tensor, right: torch.Tensor, base: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``[left | normalizer(right, base)]`` (scgnn2.py:795-805 then np.concatenate along columns), or ``[left | right]`` unscaled
    when ``base`` is None.  normalizer = np.quantile(base, 0.9 / 0.1) (all elements of base, exact) and sklearn's
    minmax_scale(right, feature_range, axis=0) in float32, bit for bit; a non-finite element of base or right raises
    ``ValueError``, as does an empty feature range.  Returns an [N, a + e] view of an [N, pitch] buffer whose pitch is a + e
    rounded up to a multiple of 4, so GEMMs and the kNN on it stay on their tensor-core paths.  With ``base`` it synchronises once."""
    _chk(left, torch.float32, "left", 2)
    _chk(right, torch.float32, "right", 2)
    n, a = left.shape
    e = right.shape[1]
    if right.shape[0] != n:
        raise B2Error(f"concat_normalized: left has {n} rows, right {right.shape[0]}")
    pitch = (a + e + 3) // 4 * 4
    out = torch.empty((n, pitch), dtype=torch.float32, device=left.device)
    lo = hi = 0.0
    cmin = cmax = None
    if base is not None:
        res = torch.empty(6, dtype=torch.float64, device=left.device)   # q0.9, q0.1, min, max, #non-finite base, #non-finite right
        _quantiles_launch(base, (0.9, 0.1), res[0:5])
        cmin, cmax = col_minmax(right, nonfinite=res[5:6])
        upper, lower, bmin, bmax, bad_base, bad_right = res.tolist()
        if bad_base > 0:
            raise ValueError(f"normalizer: base holds {int(bad_base)} non-finite values")
        if bad_right > 0:
            raise ValueError(f"normalizer: the matrix to scale holds {int(bad_right)} non-finite values")
        lo, hi = _feature_range(base, upper, lower, bmin, bmax)
    ws = _workspace(lib().b2_concat_scaled_workspace_bytes(e), left.device)
    check(lib().b2_concat_scaled_f32(_p(left), _rowmajor(left, "left"), a, _p(right), _rowmajor(right, "right"), e, n, _p(cmin),
                                     _p(cmax), lo, hi, int(base is not None), _p(out), pitch, _p(ws), ws.numel(), _stream()),
          "b2_concat_scaled_f32")
    return out[:, :a + e]


# ----------------------------------------------------------------------------- graph-sc mini-batch blocks (csrc/graphsc.cu)
def act(x, act: Optional[str], out=None):
    """``act(x)`` elementwise, for the activations the GEMM epilogue does not take (leaky_relu, gelu) as well as the others."""
    _chk(x, torch.float32, "x", 2)
    out = torch.empty_like(x) if out is None else out
    check(lib().b2_act_f32(_p(x), _rowmajor(x, "x"), x.shape[0], x.shape[1], ACT_ALL[act], _p(out), _rowmajor(out, "out"), _stream()),
          "b2_act_f32")
    return out


def act_bwd(dy, act: Optional[str], y=None, x=None, out=None):
    """``dy ⊙ act'``: from the output ``y`` for relu / elu / tanh / leaky_relu, from the pre-activation ``x`` for gelu."""
    _chk(dy, torch.float32, "dy", 2)
    out = torch.empty_like(dy) if out is None else out
    check(lib().b2_act_bwd_f32(_p(dy), _rowmajor(dy, "dy"), _p(y), _rowmajor(y, "y") if y is not None else 0, _p(x),
                               _rowmajor(x, "x") if x is not None else 0, dy.shape[0], dy.shape[1], ACT_ALL[act], _p(out),
                               _rowmajor(out, "out"), _stream()), "b2_act_bwd_f32")
    return out


def graphsc_block_degrees(A: CSR, dst: torch.Tensor, outdeg: Optional[torch.Tensor] = None, src_cap: int = 0):
    """Out-degrees of the block whose destinations are ``dst`` (int32, −1 = padding) over the destination-indexed CSR ``A``.
    Returns ``outdeg`` [n_nodes] int32, or with ``src_cap`` > 0 ``(outdeg, src_list [src_cap], src_pos [n_nodes])``: the block's
    source nodes (first-touch order, −1 padded) and each one's slot."""
    _chk(dst, torch.int32, "dst", 1)
    n = A.shape[0]
    dev = dst.device
    outdeg = torch.empty(n, dtype=torch.int32, device=dev) if outdeg is None else outdeg
    _chk(outdeg, torch.int32, "outdeg", 1)
    if outdeg.numel() < n:
        raise B2Error(f"graphsc_block_degrees: outdeg has {outdeg.numel()} entries, the graph {n} nodes")
    lst = pos = cnt = None
    if src_cap > 0:
        lst = torch.empty(src_cap, dtype=torch.int32, device=dev)
        pos = torch.empty(n, dtype=torch.int32, device=dev)
        cnt = torch.empty(1, dtype=torch.int32, device=dev)
    check(lib().b2_graphsc_block_degrees(_p(A.rowptr), _p(A.colidx), n, _p(dst), dst.numel(), _p(outdeg), _p(lst), _p(pos), _p(cnt),
                                         int(src_cap), _stream()), "b2_graphsc_block_degrees")
    return outdeg if src_cap <= 0 else (outdeg, lst, pos)


def graphsc_block_aggregate(A: CSR, dst: torch.Tensor, outdeg: torch.Tensor, x: torch.Tensor, agg: str = "sum", p: float = 0.0,
                            seed: int = 0, key: int = 0, x_pos: Optional[torch.Tensor] = None, transposed: bool = False,
                            out_rows: int = 0, out: Optional[torch.Tensor] = None):
    """WeightedGraphConv's normalised aggregation over a block (graphsc.py:445-477, before the product with W), with the
    layer's input dropout (rows keyed by global node id).  ``transposed``: its adjoint, from [len(dst), F] to [out_rows, F]
    rows ``x_pos[u]`` (or u).  See include/dance_b200.h."""
    _chk(dst, torch.int32, "dst", 1)
    _chk(outdeg, torch.int32, "outdeg", 1)
    _chk(x, torch.float32, "x", 2)
    if x_pos is not None:
        _chk(x_pos, torch.int32, "x_pos", 1)
    if agg not in ("sum", "mean"):
        raise ValueError(f"agg must be 'sum' or 'mean', got {agg!r}")
    F = x.shape[1]
    rows = int(out_rows) if transposed else dst.numel()
    if out is None:
        out = torch.empty((rows, F), dtype=torch.float32, device=x.device)
    _chk(out, torch.float32, "out", 2)
    check(lib().b2_graphsc_block_aggregate_f32(_p(A.rowptr), _p(A.colidx), _p(A.vals), _p(dst), dst.numel(), _p(outdeg), _p(x),
                                               _rowmajor(x, "x"), _p(x_pos), F, int(agg == "mean"), float(p), int(seed) & 0xFFFFFFFF,
                                               int(key) & 0xFFFFFFFF, int(transposed), _p(out), _rowmajor(out, "out"),
                                               out.shape[0] if transposed else 0, _stream()), "b2_graphsc_block_aggregate_f32")
    return out


def graphsc_batch_decoder(z: torch.Tensor, p: float = 0.1, seed: int = 0, key: int = 0, dz: Optional[torch.Tensor] = None,
                          loss: Optional[torch.Tensor] = None):
    """graph-sc's loss on one batch (graphsc.py:208-216 with InnerProductDecoder :408-411): ``norm · BCEWithLogits(z̃z̃ᵀ, I,
    pos_weight)`` with the decoder's own dropout (rows = batch positions).  Returns (loss [1] on the device, dz)."""
    _chk(z, torch.float32, "z", 2)
    if dz is None:
        dz = torch.empty_like(z)
    if loss is None:
        loss = torch.empty(1, dtype=torch.float32, device=z.device)
    _chk(dz, torch.float32, "dz", 2)
    _chk(loss, torch.float32, "loss")
    check(lib().b2_graphsc_batch_decoder_f32(_p(z), _rowmajor(z, "z"), z.shape[0], z.shape[1], float(p), int(seed) & 0xFFFFFFFF,
                                             int(key) & 0xFFFFFFFF, _p(dz), _rowmajor(dz, "dz"), _p(loss), _stream()),
          "b2_graphsc_batch_decoder_f32")
    return loss, dz


def graphsc_scatter_rows(x: torch.Tensor, idx: torch.Tensor, out: torch.Tensor, offset: int = 0):
    """``out[idx[i] − offset] = x[i]``."""
    _chk(x, torch.float32, "x", 2)
    _chk(idx, torch.int32, "idx", 1)
    _chk(out, torch.float32, "out", 2)
    check(lib().b2_graphsc_scatter_rows_f32(_p(x), _rowmajor(x, "x"), x.shape[0], x.shape[1], _p(idx), int(offset), _p(out),
                                            _rowmajor(out, "out"), _stream()), "b2_graphsc_scatter_rows_f32")
    return out
