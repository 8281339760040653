"""Thin torch-tensor wrappers over the C-ABI (``include/dance_b200.h``).

Every function takes CUDA tensors, hands raw pointers to the shared library on torch's
current stream and returns CUDA tensors.  Nothing here computes on the CPU and nothing
falls back to torch kernels: a missing library or a non-CUDA tensor raises.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import torch

from ._lib import B2Error, check
from ._lib import lib as _raw_lib

ACT = {"none": 0, None: 0, "relu": 1, "elu": 2, "tanh": 3}
PREC = {"fp32": 0, "simt": 0, "tf32x3": 1, "tf32": 2}

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
    """GEMM precision used when a call does not name one: 'fp32' | 'tf32x3' | 'tf32'."""
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
    """Select the kernel path of the decoder ("gae": auto | cuda | tc), of the kNN candidate filter
    ("knn": auto | simt) or of the aggregate ("spmm": auto | rowgroup).  All paths return the same result; the switch exists
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
    """``Y = act(A @ X)`` (reduce='sum') or row-mean (reduce='mean').  A bf16 / fp16 ``X`` selects the 16-bit-operand kernel
    (fp32 accumulation, fp32 ``out``; ``out16`` additionally receives the result in the operand's type)."""
    if isinstance(X, torch.Tensor) and X.dtype in _X16:
        fn, _ = _X16[X.dtype]
        _chk(X, X.dtype, "X", 2)
        n_rows, n_cols = A.shape
        if X.shape[0] != n_cols:
            raise B2Error(f"spmm: A is {A.shape} but X has {X.shape[0]} rows")
        F = X.shape[1]
        if out is None and out16 is None:
            out = torch.empty((n_rows, F), dtype=torch.float32, device=X.device)
        if out is not None:
            _chk(out, torch.float32, "out", 2)
        if out16 is not None:
            _chk(out16, X.dtype, "out16", 2)
        colidx_ptr = _p(A.colidx) if A.nnz else _p(A.rowptr)
        check(getattr(lib(), fn)(_p(A.rowptr), colidx_ptr, _p(A.vals) if A.nnz else None, _p(X), _rowmajor(X, "X"),
                                 _p(out), _rowmajor(out, "out") if out is not None else 0,
                                 _p(out16), _rowmajor(out16, "out16") if out16 is not None else 0,
                                 n_rows, n_cols, F, {"sum": 0, "mean": 1}[reduce], ACT[act], _p(bias), _stream()), fn)
        return out if out is not None else out16
    _chk(X, torch.float32, "X", 2)
    ldx = _rowmajor(X, "X")
    n_rows, n_cols = A.shape
    if X.shape[0] != n_cols:
        raise B2Error(f"spmm: A is {A.shape} but X has {X.shape[0]} rows")
    F = X.shape[1]
    if out is None:
        out = torch.empty((n_rows, F), dtype=torch.float32, device=X.device)
    _chk(out, torch.float32, "out", 2)
    colidx_ptr = _p(A.colidx) if A.nnz else _p(A.rowptr)  # an empty matrix has no colidx storage; never dereferenced
    check(lib().b2_spmm_csr_f32(_p(A.rowptr), colidx_ptr, _p(A.vals) if A.nnz else None, _p(X), ldx, _p(out), _rowmajor(out, "out"),
                                n_rows, n_cols, F, {"sum": 0, "mean": 1}[reduce], ACT[act], _p(bias), _stream()), "b2_spmm_csr_f32")
    return out


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
    """``C = act(op(A) @ op(B) + bias) * (mask > 0)``; ``accumulate`` adds into ``out``."""
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


def gae_loss_grad(z, labels: CSR, norm: float, pos_weight: float, mu=None, logvar=None, use_pos_weight=True,
                  dz=None, dmu=None, dlogvar=None, loss=None, row_begin: int = 0, n_rows: Optional[int] = None):
    """Matrix-free Graph-AE loss: returns (loss[1], dz, dmu, dlogvar).

    ``dmu``/``dlogvar`` may be column slices of one packed [n, 2d] buffer (shared leading dimension).
    """
    _chk(z, torch.float32, "z", 2)
    n, d = z.shape
    n_rows = n if n_rows is None else n_rows
    if labels.shape[0] != n_rows or labels.shape[1] != n:
        raise B2Error(f"gae_loss_grad: labels must be [{n_rows}, {n}] (rows of this shard x all columns), got {tuple(labels.shape)}")
    if dz is None:
        dz = torch.empty((n_rows, d), dtype=torch.float32, device=z.device)
    else:
        _chk(dz, torch.float32, "dz", 2)
        if tuple(dz.shape) != (n_rows, d) or not dz.is_contiguous():
            raise B2Error(f"gae_loss_grad: dz must be a contiguous [{n_rows}, {d}] buffer, got {tuple(dz.shape)} strides {dz.stride()}")
    ldm = ldd = 0
    if mu is not None:
        _chk(mu, torch.float32, "mu", 2)
        _chk(logvar, torch.float32, "logvar", 2)
        ldm = _rowmajor(mu, "mu")
        if _rowmajor(logvar, "logvar") != ldm:
            raise B2Error("gae_loss_grad: mu and logvar must share a leading dimension")
        if dmu is None:
            dmu = torch.empty((n_rows, d), dtype=torch.float32, device=z.device)
            dlogvar = torch.empty((n_rows, d), dtype=torch.float32, device=z.device)
        ldd = _rowmajor(dmu, "dmu")
        if _rowmajor(dlogvar, "dlogvar") != ldd:
            raise B2Error("gae_loss_grad: dmu and dlogvar must share a leading dimension")
    if loss is None:
        loss = torch.empty(1, dtype=torch.float32, device=z.device)
    ws = _workspace(lib().b2_gae_loss_workspace_bytes(n, d), z.device)
    check(lib().b2_gae_loss_grad_f32(_p(z), _rowmajor(z, "z"), _p(mu), _p(logvar), ldm, _p(labels.rowptr),
                                     _p(labels.colidx), n, d, row_begin, n_rows, float(norm), float(pos_weight),
                                     int(use_pos_weight),
                                     _p(dz), _p(dmu), _p(dlogvar), ldd, _p(loss), _p(ws), ws.numel(), _stream()),
          "b2_gae_loss_grad_f32")
    return loss, dz, dmu, dlogvar


def gae_sym_super_blocks(n: int) -> int:
    """Equal-work units of the pair-sharded decoder (super-block s = 128-row blocks s and nb−1−s; see gae_loss_grad_sym)."""
    return int(lib().b2_gae_sym_super_blocks(n))


def gae_loss_grad_sym(z, labels: CSR, norm: float, pos_weight: float, sb_begin: int, sb_end: int, mu=None, logvar=None,
                      use_pos_weight=True, dz_full=None, dmu=None, dlogvar=None, loss=None, row_begin: int = 0,
                      n_rows: Optional[int] = None):
    """Pair-sharded matrix-free Graph-AE loss (multi-GPU form of :func:`gae_loss_grad`): this rank evaluates super-blocks
    ``[sb_begin, sb_end)`` of the unordered block-pair schedule and the label / KLD terms of its rows.  Returns
    ``(loss_share[1], dz_full[n, d], dmu, dlogvar)``; all-reduce ``dz_full`` and ``loss_share`` over ranks."""
    _chk(z, torch.float32, "z", 2)
    n, d = z.shape
    n_rows = n if n_rows is None else n_rows
    if labels.shape[0] != n_rows or labels.shape[1] != n:
        raise B2Error(f"gae_loss_grad_sym: labels must be [{n_rows}, {n}], got {tuple(labels.shape)}")
    if dz_full is None:
        dz_full = torch.empty((n, d), dtype=torch.float32, device=z.device)
    _chk(dz_full, torch.float32, "dz_full", 2)
    if tuple(dz_full.shape) != (n, d) or not dz_full.is_contiguous():
        raise B2Error(f"gae_loss_grad_sym: dz_full must be a contiguous [{n}, {d}] buffer")
    ldm = ldd = 0
    if mu is not None:
        _chk(mu, torch.float32, "mu", 2)
        _chk(logvar, torch.float32, "logvar", 2)
        ldm = _rowmajor(mu, "mu")
        if _rowmajor(logvar, "logvar") != ldm:
            raise B2Error("gae_loss_grad_sym: mu and logvar must share a leading dimension")
        if dmu is None:
            dmu = torch.empty((n_rows, d), dtype=torch.float32, device=z.device)
            dlogvar = torch.empty((n_rows, d), dtype=torch.float32, device=z.device)
        ldd = _rowmajor(dmu, "dmu")
        if _rowmajor(dlogvar, "dlogvar") != ldd:
            raise B2Error("gae_loss_grad_sym: dmu and dlogvar must share a leading dimension")
    if loss is None:
        loss = torch.empty(1, dtype=torch.float32, device=z.device)
    ws = _workspace(lib().b2_gae_loss_workspace_bytes(n, d), z.device)
    check(lib().b2_gae_loss_grad_sym_f32(_p(z), _rowmajor(z, "z"), _p(mu), _p(logvar), ldm, _p(labels.rowptr), _p(labels.colidx), n, d,
                                         sb_begin, sb_end, row_begin, n_rows, float(norm), float(pos_weight), int(use_pos_weight),
                                         _p(dz_full), _p(dmu), _p(dlogvar), ldd, _p(loss), _p(ws), ws.numel(), _stream()),
          "b2_gae_loss_grad_sym_f32")
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


def gat_scores(H, a_src, a_trg, nheads: int):
    """s_src[n,h] = <H[n,h,:], a_src[h,:]> (scgnn2.py:1016-1017)."""
    _chk(H, torch.float32, "H", 2)
    n, W = H.shape
    F = W // nheads
    s_src = torch.empty((n, nheads), dtype=torch.float32, device=H.device)
    s_trg = torch.empty((n, nheads), dtype=torch.float32, device=H.device)
    check(lib().b2_gat_scores_f32(_p(H), _rowmajor(H, "H"), _p(a_src), _p(a_trg), n, nheads, F, _p(s_src), _p(s_trg), _stream()),
          "b2_gat_scores_f32")
    return s_src, s_trg


def gat_aggregate_fwd(T: CSR, H, s_src, s_trg, nheads: int, score_act="leakyrelu", slope=0.2, shift="global",
                      out=None, keep_alpha=True):
    """Fused edge softmax + aggregate on the target-indexed CSR ``T``; returns (out, alpha, gmax)."""
    n, W = H.shape
    F = W // nheads
    if out is None:
        out = torch.empty((n, W), dtype=torch.float32, device=H.device)
    gmax = torch.empty(1, dtype=torch.float32, device=H.device)
    act, sm = SCORE_ACT[score_act], SHIFT[shift]
    if sm == 0:
        check(lib().b2_gat_edge_max_f32(_p(T.rowptr), _p(T.colidx), _p(s_src), _p(s_trg), n, nheads, act, slope, _p(gmax),
                                        _stream()), "b2_gat_edge_max_f32")
    alpha = torch.empty((T.nnz, nheads), dtype=torch.float32, device=H.device) if keep_alpha else None
    check(lib().b2_gat_aggregate_fwd_f32(_p(T.rowptr), _p(T.colidx), _p(H), _rowmajor(H, "H"), _p(s_src), _p(s_trg), n, nheads,
                                         F, act, slope, sm, _p(gmax), _p(out), _rowmajor(out, "out"), _p(alpha), _stream()),
          "b2_gat_aggregate_fwd_f32")
    return out, alpha, gmax


def gat_aggregate_bwd(T: CSR, Tt: CSR, t_perm, H, a_src, a_trg, s_src, s_trg, alpha, dOut, nheads: int,
                      score_act="leakyrelu", slope=0.2, H2=None, dOut2=None, want_dH2=True):
    """Returns (dH, da_src, da_trg), or (dH, da_src, da_trg, dH2 | None) with a tied second layer (H2, dOut2)."""
    n, W = H.shape
    F = W // nheads
    dev = H.device
    dH = torch.empty((n, W), dtype=torch.float32, device=dev)
    da_src = torch.empty(W, dtype=torch.float32, device=dev)
    da_trg = torch.empty(W, dtype=torch.float32, device=dev)
    ds_s = torch.empty(n * nheads, dtype=torch.float32, device=dev)
    ds_t = torch.empty(n * nheads, dtype=torch.float32, device=dev)
    dpre = torch.empty(max(T.nnz, 1) * nheads, dtype=torch.float32, device=dev)
    if H2 is not None:
        dH2 = torch.empty((n, W), dtype=torch.float32, device=dev) if want_dH2 else None
        check(lib().b2_gat_aggregate_bwd_tied_f32(_p(T.rowptr), _p(T.colidx), _p(Tt.rowptr), _p(Tt.colidx), _p(t_perm), _p(H),
                                                  _rowmajor(H, "H"), _p(a_src), _p(a_trg), _p(s_src), _p(s_trg), _p(alpha), _p(dOut),
                                                  _rowmajor(dOut, "dOut"), _p(H2), _rowmajor(H2, "H2"), _p(dOut2),
                                                  _rowmajor(dOut2, "dOut2"), n, nheads, F, SCORE_ACT[score_act], slope, _p(dH),
                                                  _rowmajor(dH, "dH"), _p(dH2), _rowmajor(dH2, "dH2") if want_dH2 else 0, _p(da_src), _p(da_trg),
                                                  _p(ds_s), _p(ds_t), _p(dpre), _stream()), "b2_gat_aggregate_bwd_tied_f32")
        return dH, da_src, da_trg, dH2
    check(lib().b2_gat_aggregate_bwd_f32(_p(T.rowptr), _p(T.colidx), _p(Tt.rowptr), _p(Tt.colidx), _p(t_perm), _p(H),
                                         _rowmajor(H, "H"), _p(a_src), _p(a_trg), _p(s_src), _p(s_trg), _p(alpha), _p(dOut),
                                         _rowmajor(dOut, "dOut"), n, nheads, F, SCORE_ACT[score_act], slope, _p(dH),
                                         _rowmajor(dH, "dH"), _p(da_src), _p(da_trg), _p(ds_s), _p(ds_t), _p(dpre), _stream()),
          "b2_gat_aggregate_bwd_f32")
    return dH, da_src, da_trg


def gat_combine_fwd(agg, skip, bias, nheads: int, concat: bool, act=None):
    n, W = agg.shape
    F = W // nheads
    out = torch.empty((n, W if concat else F), dtype=torch.float32, device=agg.device)
    check(lib().b2_gat_combine_fwd_f32(_p(agg), _rowmajor(agg, "agg"), _p(skip), _rowmajor(skip, "skip") if skip is not None else 0,
                                       _p(bias), n, nheads, F, int(concat), ACT[act], _p(out), _rowmajor(out, "out"), _stream()),
          "b2_gat_combine_fwd_f32")
    return out


def gat_combine_bwd(dout, out, nheads: int, F: int, concat: bool, act=None):
    """Returns (dpre [n, nheads*F], dact [n, out width])."""
    n = dout.shape[0]
    dpre = torch.empty((n, nheads * F), dtype=torch.float32, device=dout.device)
    dact = torch.empty_like(out)
    check(lib().b2_gat_combine_bwd_f32(_p(dout), _rowmajor(dout, "dout"), _p(out), _rowmajor(out, "out"), n, nheads, F,
                                       int(concat), ACT[act], _p(dpre), _rowmajor(dpre, "dpre"), _p(dact), _rowmajor(dact, "dact"),
                                       _stream()), "b2_gat_combine_bwd_f32")
    return dpre, dact


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
