"""Thin torch-tensor wrappers over the C-ABI (``include/dance_b200.h``).

Every function takes CUDA tensors, hands raw pointers to the shared library on torch's
current stream and returns CUDA tensors.  Nothing here computes on the CPU and nothing
falls back to torch kernels: a missing library or a non-CUDA tensor raises.

The library sees pointers and sizes only, so every tensor crosses the boundary through :func:`_arg`, which checks its device,
dtype, extent and layout before any launch, and every status-returning entry point is invoked through :func:`_call`.
"""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple, Optional, Tuple

import torch

from ._lib import B2Error
from ._lib import lib as _raw_lib

ACT = {"none": 0, None: 0, "relu": 1, "elu": 2, "tanh": 3}
# every activation code, for act / act_bwd; the GEMM / SpMM epilogues take ACT only
ACT_ALL = {**ACT, "leaky_relu": 4, "gelu": 5}
PREC = {"fp32": 0, "simt": 0, "tf32x3": 1, "tf32": 2, "bf16": 3}

_DEFAULT_PRECISION = "tf32x3"

_F32, _F64, _I32, _I64, _U8 = torch.float32, torch.float64, torch.int32, torch.int64, torch.uint8

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


def _call(name: str, *args) -> None:
    """Invoke the entry point ``name`` with ``args``; a non-zero status raises B2Error with the library's message."""
    status = getattr(_proxy, name)(*args)
    if status != 0:
        raise B2Error(f"{name} failed with status {status}: {_raw_lib().b2_last_error().decode('utf-8', 'replace')}")


def _arg(t, name: str, dtype, shape=None, *, ld: bool = False, optional: bool = False, at_least: bool = False, empty=None):
    """The device pointer of ``t`` for the library, after the checks the C side cannot make.

    ``t`` must be a CUDA tensor on the current device with dtype ``dtype``.  ``shape`` is its extent: an int is the element count
    of a contiguous buffer (None: a contiguous buffer of any size), a tuple the sizes of its dimensions (None: any size),
    contiguous as well unless ``ld``.  With ``at_least`` the count, or the first size, is a minimum (a kernel that reads a
    prefix).  ``ld``: a 2-D operand passed with a leading dimension, which must have unit inner stride (its rows may be padded);
    returns ``(pointer, ld)``.  ``optional``: None is allowed and gives a NULL pointer (and ld 0).  ``empty``: the pointer that
    stands in for an empty tensor, which has no storage while the library refuses NULL; it is never dereferenced."""
    if t is None and optional:
        return (None, 0) if ld else None
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise B2Error(f"{name}: expected a CUDA tensor (dance_b200 has no CPU path)")
    if t.dtype != dtype:
        raise B2Error(f"{name}: expected dtype {dtype}, got {t.dtype}")
    if t.get_device() != torch.cuda.current_device():
        raise B2Error(f"{name}: tensor is on {t.device}, the current device is cuda:{torch.cuda.current_device()}")
    s = t.shape
    if isinstance(shape, tuple):
        if len(s) != len(shape) or any(w is not None and (v < w if at_least and i == 0 else v != w)
                                       for i, (v, w) in enumerate(zip(s, shape))):
            want = tuple("*" if w is None else w for w in shape)
            raise B2Error(f"{name}: expected shape {want}{' (rows at least)' if at_least else ''}, got {tuple(s)}")
    elif shape is not None and (t.numel() < shape if at_least else t.numel() != shape):
        raise B2Error(f"{name}: expected {'at least ' if at_least else ''}{shape} elements, got shape {tuple(s)}")
    if ld and t.stride(1) != 1:
        raise B2Error(f"{name}: must be 2-D with unit inner stride, got strides {t.stride()}")
    if not ld and not t.is_contiguous():
        raise B2Error(f"{name}: must be contiguous, got shape {tuple(s)} strides {t.stride()}")
    p = t.data_ptr() if empty is None or t.numel() else empty
    return (p, t.stride(0) if s[0] > 1 else max(t.stride(0), s[1])) if ld else p


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


_ws_cache = {}


def _workspace(nbytes: int, device) -> Tuple[int, int]:
    """(pointer, bytes) of a per-device grow-only scratch buffer (stream-ordered use only)."""
    key = (device.index if device.index is not None else torch.cuda.current_device())
    buf = _ws_cache.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(max(nbytes, 1 << 20), dtype=_U8, device=device)
        _ws_cache[key] = buf
    return _arg(buf, "workspace", _U8, buf.numel()), buf.numel()


_PATHS = {"gae": (0, {"auto": 0, "cuda": 1, "tc": 2}), "knn": (1, {"auto": 0, "simt": 1}),
          "spmm": (2, {"auto": 0, "rowgroup": 1})}


def set_path(which: str, mode: str = "auto") -> None:
    """Select the kernel path of the decoder ("gae": auto | cuda | tc), of the kNN candidate filter ("knn": auto | simt) or
    of the aggregate ("spmm": auto | rowgroup).  All paths return the same result; the switch exists
    for A/B tests and timing."""
    sel, modes = _PATHS[which]
    _call("b2_set_path", sel, modes[mode])


def set_tuning(knob: str, value: int) -> None:
    """Scheduling knob of the tensor-core decoder ("gae_splits": step ranges per 128-row block of the J sweep, 0 = automatic):
    timing experiments only."""
    _call("b2_set_tuning", {"gae_splits": 0}[knob], int(value))


def get_path(which: str) -> str:
    sel, modes = _PATHS[which]
    v = lib().b2_get_path(sel)
    return next(k for k, m in modes.items() if m == v)


def device_info() -> Tuple[int, int, int]:
    a, b, c = C.c_int(), C.c_int(), C.c_int()
    _call("b2_device_info", C.byref(a), C.byref(b), C.byref(c))
    return a.value, b.value, c.value


# ----------------------------------------------------------------------------- CSR container
class CSR:
    """Device CSR matrix: int32 rowptr/colidx, optional fp32 values (None = all ones).  Checked once, here: ``ptrs`` holds the
    pointers of (rowptr, colidx, vals) that every wrapper passes on; an edgeless matrix's colidx / vals point at rowptr."""

    __slots__ = ("rowptr", "colidx", "vals", "shape", "ptrs", "_t", "sigmas", "rhos")

    def __init__(self, rowptr, colidx, vals, shape):
        shape = tuple(shape)
        rp = _arg(rowptr, "rowptr", _I32, (shape[0] + 1, ))
        ci = _arg(colidx, "colidx", _I32, (None, ), empty=rp)
        self.ptrs = (rp, ci, _arg(vals, "vals", _F32, (colidx.numel(), ), optional=True, empty=rp))
        self.rowptr, self.colidx, self.vals, self.shape = rowptr, colidx, vals, shape
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
    x, ldx = _arg(X, "X", _F32, (None, None), ld=True)
    if dtype not in _X16:
        raise B2Error(f"to_x16: dtype must be torch.bfloat16 or torch.float16, got {dtype}")
    if out is None:
        out = torch.empty(X.shape, dtype=dtype, device=X.device)
    o, ldo = _arg(out, "out", dtype, tuple(X.shape), ld=True)
    _call("b2_convert_f32_to_x16", x, ldx, o, ldo, X.shape[0], X.shape[1], _X16[dtype][1], _stream())
    return out


def spmm(A: CSR, X: torch.Tensor, reduce: str = "sum", act: Optional[str] = None,
         out: Optional[torch.Tensor] = None, bias: Optional[torch.Tensor] = None, out16: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``Y = act(A @ X)`` (reduce='sum') or row-mean (reduce='mean').  A bf16 / fp16 ``X`` is gathered in its 16-bit
    type (fp32 accumulation, fp32 ``out``; ``out16`` additionally receives the result in the operand's type)."""
    x16 = isinstance(X, torch.Tensor) and X.dtype in _X16
    n_rows, n_cols = A.shape
    x, ldx = _arg(X, "X", X.dtype if x16 else _F32, (n_cols, None), ld=True)
    F = X.shape[1]
    if not x16:
        out16 = None  # an fp32 operand has no 16-bit result copy
    if out is None and out16 is None:
        out = torch.empty((n_rows, F), dtype=_F32, device=X.device)
    args = [*A.ptrs, x, ldx, *_arg(out, "out", _F32, (n_rows, F), ld=True, optional=True)]
    if x16:
        fn = _X16[X.dtype][0]
        args += _arg(out16, "out16", X.dtype, (n_rows, F), ld=True, optional=True)
    else:
        fn = "b2_spmm_csr_f32"
    _call(fn, *args, n_rows, n_cols, F, {"sum": 0, "mean": 1}[reduce], ACT[act], _arg(bias, "bias", _F32, F, optional=True), _stream())
    return out if out is not None else out16


def csr_transpose(A: CSR) -> Tuple[CSR, torch.Tensor]:
    n_rows, n_cols = A.shape
    nnz = A.nnz
    dev = A.rowptr.device
    t_rowptr = torch.empty(n_cols + 1, dtype=_I32, device=dev)
    t_colidx = torch.empty(nnz, dtype=_I32, device=dev)
    t_vals = torch.empty(nnz, dtype=_F32, device=dev) if A.vals is not None else None
    perm = torch.empty(nnz, dtype=_I32, device=dev)
    outs = (_arg(t_rowptr, "t_rowptr", _I32, n_cols + 1), _arg(t_colidx, "t_colidx", _I32, nnz),
            _arg(t_vals, "t_vals", _F32, nnz, optional=True), _arg(perm, "perm", _I32, nnz))
    _call("b2_csr_transpose", *A.ptrs, n_rows, n_cols, nnz, *outs, *_workspace(lib().b2_csr_transpose_workspace_bytes(n_rows, n_cols, nnz), dev),
          _stream())
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
    a, lda = _arg(A, "A", _F32, (None, None), ld=True)
    M, K = (A.shape[1], A.shape[0]) if transA else A.shape
    b, ldb = _arg(B, "B", _F32, (None, K) if transB else (K, None), ld=True)
    N = B.shape[0] if transB else B.shape[1]
    if out is None:
        if accumulate:
            raise B2Error("gemm: accumulate=True needs `out`")
        out = torch.empty((M, N), dtype=_F32, device=A.device)
    prec = PREC[precision or _DEFAULT_PRECISION]
    nbytes = lib().b2_gemm_workspace_bytes(M, N, K, int(transA), int(transB), prec)
    _call("b2_gemm_f32", a, lda, int(transA), b, ldb, int(transB), *_arg(out, "out", _F32, (M, N), ld=True), M, N, K,
          _arg(bias, "bias", _F32, (N, ), optional=True), ACT[act], *_arg(mask, "mask", _F32, (M, N), ld=True, optional=True),
          1.0 if accumulate else 0.0, prec, *(_workspace(nbytes, A.device) if nbytes else (None, 0)), _stream())
    return out


def colsum(X: torch.Tensor, out: Optional[torch.Tensor] = None, accumulate: bool = False) -> torch.Tensor:
    x, ldx = _arg(X, "X", _F32, (None, None), ld=True)
    M, N = X.shape
    if out is None:
        out = torch.empty(N, dtype=_F32, device=X.device)
    nbytes = lib().b2_colsum_workspace_bytes(M, N)
    _call("b2_colsum_f32", x, ldx, M, N, _arg(out, "out", _F32, N), 1.0 if accumulate else 0.0,
          *(_workspace(nbytes, X.device) if nbytes else (None, 0)), _stream())
    return out


def mse_sum_loss_grad(recon, target, ltmg_regu=None, regu_strength=0.0, relu_mask=False, grad=None, loss_out=None):
    """Feature-AE loss; returns (loss_out[1] accumulated, grad wrt recon)."""
    r = _arg(recon, "recon", _F32, None)
    n = recon.numel()
    if grad is None:
        grad = torch.empty_like(recon)
    if loss_out is None:
        loss_out = torch.zeros(1, dtype=_F32, device=recon.device)
    _call("b2_mse_sum_loss_grad_f32", r, _arg(target, "target", _F32, n), _arg(ltmg_regu, "ltmg_regu", _F32, n, optional=True),
          float(regu_strength), int(relu_mask), _arg(grad, "grad", _F32, n), _arg(loss_out, "loss_out", _F32, 1), n, _stream())
    return loss_out, grad


def _gae_prepare(what, z, labels: CSR, n_rows, mu, logvar, dmu, dlogvar, loss, labels_t: Optional[CSR] = None):
    """Checks and buffers both decoder calls share.  Returns (n, d, n_rows, head, tail, dmu, dlogvar, loss): ``head`` are the
    arguments from z up to and including n and d, ``tail`` those from dmu on; the label arguments in ``head`` are the pointers of
    L and of Lᵀ, and the library reads Lᵀ only when L has values."""
    zp, ldz = _arg(z, "z", _F32, (None, None), ld=True)
    n, d = z.shape
    n_rows = n if n_rows is None else n_rows
    if labels.shape[0] != n_rows or labels.shape[1] != n:
        raise B2Error(f"{what}: labels must be [{n_rows}, {n}] (rows of this shard x all columns), got {tuple(labels.shape)}")
    if labels.vals is not None:
        if labels_t is None or labels_t.vals is None:
            raise B2Error(f"{what}: real-valued labels need labels_t= (the same rows of Lᵀ, with values)")
        if tuple(labels_t.shape) != tuple(labels.shape):
            raise B2Error(f"{what}: labels_t must be [{n_rows}, {n}] like labels, got {tuple(labels_t.shape)}")
    m = lv = dm = dl = None
    ldm = ldd = 0
    if mu is not None:
        m, ldm = _arg(mu, "mu", _F32, (n_rows, d), ld=True)
        lv, ldl = _arg(logvar, "logvar", _F32, (n_rows, d), ld=True)
        if ldl != ldm:
            raise B2Error(f"{what}: mu and logvar must share a leading dimension")
        if dmu is None:
            dmu = torch.empty((n_rows, d), dtype=_F32, device=z.device)
            dlogvar = torch.empty((n_rows, d), dtype=_F32, device=z.device)
        dm, ldd = _arg(dmu, "dmu", _F32, (n_rows, d), ld=True)
        dl, ldl = _arg(dlogvar, "dlogvar", _F32, (n_rows, d), ld=True)
        if ldl != ldd:
            raise B2Error(f"{what}: dmu and dlogvar must share a leading dimension")
    if loss is None:
        loss = torch.empty(1, dtype=_F32, device=z.device)
    head = (zp, ldz, m, lv, ldm, *labels.ptrs, *(labels_t.ptrs if labels_t is not None else (None, None, None)), n, d)
    tail = (dm, dl, ldd, _arg(loss, "loss", _F32, 1), *_workspace(lib().b2_gae_loss_workspace_bytes(n, d), z.device), _stream())
    return n, d, n_rows, head, tail, dmu, dlogvar, loss


def gae_loss_grad(z, labels: CSR, norm: float, pos_weight: float, mu=None, logvar=None, use_pos_weight=True,
                  dz=None, dmu=None, dlogvar=None, loss=None, row_begin: int = 0, n_rows: Optional[int] = None,
                  labels_t: Optional[CSR] = None):
    """Matrix-free Graph-AE loss: returns (loss[1], dz, dmu, dlogvar).

    ``dmu``/``dlogvar`` may be column slices of one packed [n, 2d] buffer (shared leading dimension).
    ``labels.vals`` None: unit, symmetric labels.  Otherwise real-valued, possibly asymmetric labels (graph_AE_retain_weights), and
    ``labels_t`` holds the same rows of Lᵀ with their values.
    """
    n, d, n_rows, head, tail, dmu, dlogvar, loss = _gae_prepare("gae_loss_grad", z, labels, n_rows, mu, logvar, dmu, dlogvar, loss,
                                                                labels_t)
    if dz is None:
        dz = torch.empty((n_rows, d), dtype=_F32, device=z.device)
    _call("b2_gae_loss_grad_f32", *head, row_begin, n_rows, float(norm), float(pos_weight), int(use_pos_weight),
          _arg(dz, "dz", _F32, (n_rows, d)), *tail)
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
    n, d, n_rows, head, tail, dmu, dlogvar, loss = _gae_prepare("gae_loss_grad_sym", z, labels, n_rows, mu, logvar, dmu, dlogvar,
                                                                loss, labels_t)
    if dz_full is None:
        dz_full = torch.empty((n, d), dtype=_F32, device=z.device)
    _call("b2_gae_loss_grad_sym_f32", *head, sb_begin, sb_end, row_begin, n_rows, float(norm), float(pos_weight),
          int(use_pos_weight), _arg(dz_full, "dz_full", _F32, (n, d)), *tail)
    return loss, dz_full, dmu, dlogvar


def adam_step(param, grad, exp_avg, exp_avg_sq, step: int, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0):
    p = _arg(param, "param", _F32, None)
    n = param.numel()
    _call("b2_adam_step_f32", p, _arg(grad, "grad", _F32, n), _arg(exp_avg, "exp_avg", _F32, n),
          _arg(exp_avg_sq, "exp_avg_sq", _F32, n), n, lr, beta1, beta2, eps, weight_decay, step, _stream())


def act(x, act: Optional[str], out=None):
    """``act(x)`` elementwise, for the activations the GEMM epilogue does not take (leaky_relu, gelu) as well as the others."""
    xp, ldx = _arg(x, "x", _F32, (None, None), ld=True)
    out = torch.empty_like(x) if out is None else out
    _call("b2_act_f32", xp, ldx, x.shape[0], x.shape[1], ACT_ALL[act], *_arg(out, "out", _F32, tuple(x.shape), ld=True), _stream())
    return out


def act_bwd(dy, act: Optional[str], y=None, x=None, out=None):
    """``dy ⊙ act'``: from the output ``y`` for relu / elu / tanh / leaky_relu, from the pre-activation ``x`` for gelu."""
    g, ldg = _arg(dy, "dy", _F32, (None, None), ld=True)
    shape = tuple(dy.shape)
    out = torch.empty_like(dy) if out is None else out
    _call("b2_act_bwd_f32", g, ldg, *_arg(y, "y", _F32, shape, ld=True, optional=True), *_arg(x, "x", _F32, shape, ld=True, optional=True),
          shape[0], shape[1], ACT_ALL[act], *_arg(out, "out", _F32, shape, ld=True), _stream())
    return out


def reparam_fwd(mu, logvar, eps, out=None):
    m, ldm = _arg(mu, "mu", _F32, (None, None), ld=True)
    n, d = mu.shape
    lv, ldl = _arg(logvar, "logvar", _F32, (n, d), ld=True)
    if ldl != ldm:
        raise B2Error("reparam_fwd: mu and logvar must share a leading dimension")
    z = out if out is not None else torch.empty((n, d), dtype=_F32, device=mu.device)
    _call("b2_reparam_fwd_f32", m, lv, ldm, *_arg(eps, "eps", _F32, (n, d), ld=True), *_arg(z, "out", _F32, (n, d), ld=True), n, d,
          _stream())
    return z


def reparam_bwd(dz, logvar, eps, dmu, dlogvar):
    g, ldg = _arg(dz, "dz", _F32, (None, None), ld=True)
    n, d = dz.shape
    dm, ldd = _arg(dmu, "dmu", _F32, (n, d), ld=True)
    dl, ldl = _arg(dlogvar, "dlogvar", _F32, (n, d), ld=True)
    if ldl != ldd:
        raise B2Error("reparam_bwd: dmu and dlogvar must share a leading dimension")
    _call("b2_reparam_bwd_f32", g, ldg, *_arg(logvar, "logvar", _F32, (n, d), ld=True), *_arg(eps, "eps", _F32, (n, d), ld=True),
          dm, dl, ldd, n, d, _stream())


def knn(X: torch.Tensor, k: int, include_rank0: bool = False, q_begin: int = 0, q_end: Optional[int] = None,
        return_dist: bool = True):
    """Exact euclidean kNN of rows ``q_begin:q_end`` of X against all rows of X.

    Returns ``(idx[int32, n_q×k], dist[float64, n_q×k] or None)`` ranked by (fp64 distance, index).
    ``include_rank0=False`` drops sorted rank 0 — the reference's "self" slot (scgnn2.py:684-687).
    """
    x, ldx = _arg(X, "X", _F32, (None, None), ld=True)
    n, d = X.shape
    q_end = n if q_end is None else q_end
    nq = q_end - q_begin
    idx = torch.empty((nq, k), dtype=_I32, device=X.device)
    dist = torch.empty((nq, k), dtype=_F64, device=X.device) if return_dist else None
    ws = _workspace(lib().b2_knn_workspace_bytes(n, d, k, nq), X.device)
    _call("b2_knn_l2_f32", x, ldx, n, d, k, q_begin, q_end, int(include_rank0), _arg(idx, "idx", _I32, (nq, k)),
          _arg(dist, "dist", _F64, (nq, k), optional=True), *ws, _stream())
    return idx, dist


def pairwise_l2_dense(X: torch.Tensor) -> torch.Tensor:
    x, ldx = _arg(X, "X", _F32, (None, None), ld=True)
    n, d = X.shape
    D = torch.empty((n, n), dtype=_F32, device=X.device)
    _call("b2_pairwise_l2_dense_f32", x, ldx, n, d, _arg(D, "D", _F32, (n, n)), n, _stream())
    return D


def knn_graph_build(knn_idx: torch.Tensor) -> CSR:
    """Union-symmetrised kNN adjacency + I with D^-1/2 (A+I) D^-1/2 values (scgnn2.py:650-672,1191-1198)."""
    ki = _arg(knn_idx, "knn_idx", _I32, (None, None))
    n, k = knn_idx.shape
    cap = 2 * n * k + n
    dev = knn_idx.device
    rowptr = torch.empty(n + 1, dtype=_I32, device=dev)
    colidx = torch.empty(cap, dtype=_I32, device=dev)
    vals = torch.empty(cap, dtype=_F32, device=dev)
    nnz = C.c_int64(0)
    ws = _workspace(lib().b2_knn_graph_workspace_bytes(n, k), dev)
    _call("b2_knn_graph_build", ki, n, k, _arg(rowptr, "rowptr", _I32, n + 1), _arg(colidx, "colidx", _I32, cap),
          _arg(vals, "vals", _F32, cap), cap, C.byref(nnz), *ws, _stream())
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
    ki = _arg(knn_idx, "knn_idx", _I32, (None, None))
    n, k = knn_idx.shape
    kd = _arg(knn_dist, "knn_dist", _F64, (n, k))
    cap = n * (k + 1)
    dev = knn_idx.device
    i32 = lambda m: torch.empty(m, dtype=_I32, device=dev)
    f32 = lambda m: torch.empty(m, dtype=_F32, device=dev)
    rowptr, colidx, y, norm_t = i32(n + 1), i32(cap), f32(cap), f32(cap)
    t_rowptr, t_colidx, t_y, norm = i32(n + 1), i32(cap), f32(cap), f32(cap)
    sum_w = torch.empty(1, dtype=_F64, device=dev)
    nnz = C.c_int64(0)
    ws = _workspace(lib().b2_knn_graph_weighted_workspace_bytes(n, k), dev)
    _call("b2_knn_graph_weighted_build", ki, kd, n, k, _arg(rowptr, "rowptr", _I32, n + 1), _arg(colidx, "colidx", _I32, cap),
          _arg(y, "y", _F32, cap), _arg(norm_t, "norm_t", _F32, cap), _arg(t_rowptr, "t_rowptr", _I32, n + 1),
          _arg(t_colidx, "t_colidx", _I32, cap), _arg(t_y, "t_y", _F32, cap), _arg(norm, "norm", _F32, cap),
          _arg(sum_w, "sum_w", _F64, 1), cap, C.byref(nnz), *ws, _stream())
    m = nnz.value
    if m < cap:
        colidx, y, norm_t, t_colidx, t_y, norm = (t[:m].clone() for t in (colidx, y, norm_t, t_colidx, t_y, norm))
    return WeightedGraph(CSR(t_rowptr, t_colidx, norm, (n, n)), CSR(rowptr, colidx, norm_t, (n, n)), CSR(rowptr, colidx, y, (n, n)),
                         CSR(t_rowptr, t_colidx, t_y, (n, n)), sum_w)


def normalize_total_log1p_(X: torch.Tensor, target_sum: Optional[float] = None, max_fraction: float = 1.0,
                           normalize: bool = True, log1p: bool = True, base: Optional[float] = None) -> torch.Tensor:
    """In-place normalize_total (+log1p) on a dense CUDA matrix (cells × genes)."""
    x, ldx = _arg(X, "X", _F32, (None, None), ld=True)
    n, g = X.shape
    ws = _workspace(lib().b2_normalize_total_workspace_bytes(n, g), X.device)
    _call("b2_normalize_total_log1p_f32", x, ldx, n, g, float(target_sum or 0.0), float(max_fraction), int(normalize), int(log1p),
          float(base or 0.0), *ws, _stream())
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
    xp, ldx = _arg(x, "x", _F32, (None, None), ld=True)
    p = _drop_prob(p)
    if out is None:
        out = torch.empty(x.shape, dtype=_F32, device=x.device)
    _call("b2_dropout_f32", xp, ldx, x.shape[0], x.shape[1], p, int(seed) & 0xFFFFFFFF, int(key) & 0xFFFFFFFF,
          *_arg(out, "out", _F32, tuple(x.shape), ld=True), _stream())
    return out


def gat_scores(H, a_src, a_trg, nheads: int):
    """s_src[n,h] = <H[n,h,:], a_src[h,:]> (scgnn2.py:1016-1017)."""
    h, ldh = _arg(H, "H", _F32, (None, None), ld=True)
    n, W = H.shape
    F = _head_width(W, nheads, "gat_scores")
    s_src = torch.empty((n, nheads), dtype=_F32, device=H.device)
    s_trg = torch.empty((n, nheads), dtype=_F32, device=H.device)
    _call("b2_gat_scores_f32", h, ldh, _arg(a_src, "a_src", _F32, W), _arg(a_trg, "a_trg", _F32, W), n, nheads, F,
          _arg(s_src, "s_src", _F32, (n, nheads)), _arg(s_trg, "s_trg", _F32, (n, nheads)), _stream())
    return s_src, s_trg


def gat_aggregate_fwd(T: CSR, H, s_src, s_trg, nheads: int, score_act="leakyrelu", slope=0.2, shift="global",
                      out=None, keep_alpha=True, dropout: float = 0.0, seed: Optional[int] = None, key: int = 0):
    """Fused edge softmax + aggregate on the target-indexed CSR ``T``; returns (out, alpha, gmax).

    ``gmax`` [1] is the global shift (``shift="global"``; -inf for a graph without edges) and is what
    :func:`gat_aggregate_bwd` needs to differentiate through it.

    ``seed`` given: attention dropout (scgnn2.py:1029) — ``out[v] = Σ drop(α)_e H[u]`` with the keep bit of (edge at CSR
    position p, head h) drawn as :func:`dropout` draws element (p, h) under (seed, key).  ``alpha`` stays undropped; pass
    the same (dropout, seed, key) to :func:`gat_aggregate_bwd`."""
    h, ldh = _arg(H, "H", _F32, (T.shape[0], None), ld=True)
    n, W = H.shape
    F = _head_width(W, nheads, "gat_aggregate_fwd")
    if seed is None and dropout:
        raise ValueError("gat_aggregate_fwd: attention dropout needs a seed")
    p = _drop_prob(dropout)
    ss, st = _arg(s_src, "s_src", _F32, (n, nheads)), _arg(s_trg, "s_trg", _F32, (n, nheads))
    if out is None:
        out = torch.empty((n, W), dtype=_F32, device=H.device)
    o, ldo = _arg(out, "out", _F32, (n, W), ld=True)
    gmax = torch.empty(1, dtype=_F32, device=H.device)
    g = _arg(gmax, "gmax", _F32, 1)
    act, sm = SCORE_ACT[score_act], SHIFT[shift]
    alpha = torch.empty((T.nnz, nheads), dtype=_F32, device=H.device) if keep_alpha else None
    a = _arg(alpha, "alpha", _F32, (T.nnz, nheads), optional=True, empty=T.ptrs[0])
    if sm == 0:
        _call("b2_gat_edge_max_f32", *T.ptrs[:2], ss, st, n, nheads, act, slope, g, _stream())
    _call("b2_gat_aggregate_fwd_f32", *T.ptrs[:2], h, ldh, ss, st, n, nheads, F, act, slope, sm, g, o, ldo, a, p,
          int(seed or 0) & 0xFFFFFFFF, int(key) & 0xFFFFFFFF, _stream())
    return out, alpha, gmax


def gat_aggregate_bwd(T: CSR, Tt: CSR, t_perm, H, a_src, a_trg, s_src, s_trg, alpha, dOut, nheads: int,
                      score_act="leakyrelu", slope=0.2, H2=None, dOut2=None, want_dH2=True, gmax=None, dropout: float = 0.0,
                      seed: Optional[int] = None, key: int = 0):
    """Returns (dH, da_src, da_trg), or (dH, da_src, da_trg, dH2 | None) with a tied second layer (H2, dOut2).

    ``gmax``: the forward's global shift (third result of :func:`gat_aggregate_fwd` with ``shift="global"``), whose
    gradient the backward then includes, as the reference does not detach its max; None for ``shift="segment"``.
    ``dropout`` / ``seed`` / ``key``: the forward's attention dropout (not with a tied layer); ``alpha`` is the undropped α."""
    h, ldh = _arg(H, "H", _F32, (T.shape[0], None), ld=True)
    n, W = H.shape
    F = _head_width(W, nheads, "gat_aggregate_bwd")
    if seed is None and dropout:
        raise ValueError("gat_aggregate_bwd: attention dropout needs a seed")
    p = _drop_prob(dropout)
    if Tt.shape != (n, n) or Tt.nnz != T.nnz:
        raise B2Error(f"gat_aggregate_bwd: Tt must be the [{n}, {n}] transpose of T with its {T.nnz} edges, got {Tt.shape}, {Tt.nnz}")
    nnz, tied = T.nnz, H2 is not None
    dev = H.device
    dH = torch.empty((n, W), dtype=_F32, device=dev)
    da_src = torch.empty(W, dtype=_F32, device=dev)
    da_trg = torch.empty(W, dtype=_F32, device=dev)
    ds_s = torch.empty(n * nheads, dtype=_F32, device=dev)
    ds_t = torch.empty(n * nheads, dtype=_F32, device=dev)
    dpre = torch.empty(max(nnz, 1) * nheads, dtype=_F32, device=dev)
    shift_ws = torch.empty(2, dtype=_F32, device=dev) if gmax is not None else None
    dH2 = torch.empty((n, W), dtype=_F32, device=dev) if tied and want_dH2 else None
    # an edgeless graph has no t_perm / alpha storage: T's stand-in pointer takes their place
    _call("b2_gat_aggregate_bwd_f32", *T.ptrs[:2], *Tt.ptrs[:2], _arg(t_perm, "t_perm", _I32, nnz, empty=T.ptrs[0]), h, ldh,
          _arg(a_src, "a_src", _F32, W), _arg(a_trg, "a_trg", _F32, W), _arg(s_src, "s_src", _F32, (n, nheads)),
          _arg(s_trg, "s_trg", _F32, (n, nheads)), _arg(alpha, "alpha", _F32, (nnz, nheads), empty=T.ptrs[0]),
          *_arg(dOut, "dOut", _F32, (n, W), ld=True), *_arg(H2, "H2", _F32, (n, W), ld=True, optional=True),
          *_arg(dOut2 if tied else None, "dOut2", _F32, (n, W), ld=True, optional=not tied), n, nheads, F, SCORE_ACT[score_act],
          slope, _arg(gmax, "gmax", _F32, 1, optional=True), *_arg(dH, "dH", _F32, (n, W), ld=True),
          *_arg(dH2, "dH2", _F32, (n, W), ld=True, optional=True), _arg(da_src, "da_src", _F32, W), _arg(da_trg, "da_trg", _F32, W),
          _arg(ds_s, "ds_src", _F32, n * nheads), _arg(ds_t, "ds_trg", _F32, n * nheads), _arg(dpre, "dpre", _F32, dpre.numel()),
          _arg(shift_ws, "shift_ws", _F32, 2, optional=True), p, int(seed or 0) & 0xFFFFFFFF, int(key) & 0xFFFFFFFF, _stream())
    return (dH, da_src, da_trg, dH2) if tied else (dH, da_src, da_trg)


def gat_combine_fwd(agg, skip, bias, nheads: int, concat: bool, act=None, identity: bool = False):
    """``identity``: ``skip`` is the layer's raw input [n, F], added to every head (GATLayer with FIN == FOUT,
    scgnn2.py:1167-1171); otherwise ``skip`` is [n, nheads*F] or None."""
    a, lda = _arg(agg, "agg", _F32, (None, None), ld=True)
    n, W = agg.shape
    F = _head_width(W, nheads, "gat_combine_fwd")
    OW = W if concat else F
    out = torch.empty((n, OW), dtype=_F32, device=agg.device)
    _call("b2_gat_combine_fwd_f32", a, lda, *_arg(skip, "skip", _F32, (n, F if identity else W), ld=True, optional=not identity),
          _arg(bias, "bias", _F32, OW, optional=True), n, nheads, F, int(concat), ACT[act], int(identity),
          *_arg(out, "out", _F32, (n, OW), ld=True), _stream())
    return out


def gat_combine_bwd(dout, out, nheads: int, F: int, concat: bool, act=None, identity: bool = False, dpre=None, dx_skip=None):
    """Returns (dpre [n, nheads*F], dact [n, out width]); with ``identity`` also dx_skip [n, F] = Σ_h dpre[:, h·F:(h+1)·F],
    the identity skip's gradient of the layer input.  ``dpre`` / ``dx_skip``: optional (strided) output buffers."""
    OW = nheads * F if concat else F
    g, ldg = _arg(dout, "dout", _F32, (None, OW), ld=True)
    n = dout.shape[0]
    o, ldo = _arg(out, "out", _F32, (n, OW), ld=True)
    if dpre is None:
        dpre = torch.empty((n, nheads * F), dtype=_F32, device=dout.device)
    dact = torch.empty((n, OW), dtype=_F32, device=dout.device)
    if not identity:
        dx_skip = None
    elif dx_skip is None:
        dx_skip = torch.empty((n, F), dtype=_F32, device=dout.device)
    _call("b2_gat_combine_bwd_f32", g, ldg, o, ldo, n, nheads, F, int(concat), ACT[act], *_arg(dpre, "dpre", _F32, (n, nheads * F), ld=True),
          *_arg(dact, "dact", _F32, (n, OW), ld=True), *_arg(dx_skip, "dx_skip", _F32, (n, F), ld=True, optional=not identity),
          _stream())
    return (dpre, dact, dx_skip) if identity else (dpre, dact)


# ----------------------------------------------------------------------------- scDeepSort path
def cellgene_graph(X: torch.Tensor, normalize_edges: bool = True):
    """CellFeatureGraph edge list (cell_feature_graph.py:34-79): returns (src int64, dst int64, w fp32 [E,1], nnz)."""
    x, ldx = _arg(X, "X", _F32, (None, None), ld=True)
    n, g = X.shape
    nbytes = lib().b2_cellgene_graph_workspace_bytes(n, g)
    ws = torch.empty(nbytes, dtype=_U8, device=X.device)      # private: must survive between count and fill
    wsp = _arg(ws, "workspace", _U8, nbytes)
    nnz = C.c_int64(0)
    _call("b2_cellgene_graph_count", x, ldx, n, g, C.byref(nnz), wsp, nbytes, _stream())
    E = 2 * nnz.value + n + g
    src = torch.empty(E, dtype=_I64, device=X.device)
    dst = torch.empty(E, dtype=_I64, device=X.device)
    w = torch.empty((E, 1), dtype=_F32, device=X.device)
    _call("b2_cellgene_graph_fill", x, ldx, n, g, int(normalize_edges), nnz.value, _arg(src, "src", _I64, E), _arg(dst, "dst", _I64, E),
          _arg(w, "w", _F32, E), wsp, nbytes, _stream())
    return src, dst, w, nnz.value


def sage_edge_values(T: CSR, w: torch.Tensor, alpha: torch.Tensor, n_genes: int) -> torch.Tensor:
    """AdaptiveSAGE's edge scalars ``out[p] = w[p] · alpha[idx(p)]``; ``alpha`` holds the n_genes gene weights, then the gene and
    the cell self-loop weights."""
    wp = _arg(w, "w", _F32, T.nnz)
    out = torch.empty(T.nnz, dtype=_F32, device=w.device)
    _call("b2_sage_edge_values_f32", *T.ptrs[:2], wp, _arg(alpha, "alpha", _F32, n_genes + 2), T.shape[0], n_genes,
          _arg(out, "out", _F32, T.nnz), _stream())
    return out


def softmax_ce_sum(logits: torch.Tensor, labels: torch.Tensor, dlogits: Optional[torch.Tensor] = None,
                   loss_out: Optional[torch.Tensor] = None, need_grad: bool = True):
    """CrossEntropyLoss(reduction='sum'): accumulates into loss_out[0]; returns (loss_out, dlogits)."""
    lg, ldl = _arg(logits, "logits", _F32, (None, None), ld=True)
    n, c = logits.shape
    if need_grad and dlogits is None:
        dlogits = torch.empty_like(logits)
    if loss_out is None:
        loss_out = torch.zeros(1, dtype=_F32, device=logits.device)
    _call("b2_softmax_ce_sum_f32", lg, ldl, _arg(labels, "labels", _I64, (n, )), n, c,
          *_arg(dlogits if need_grad else None, "dlogits", _F32, (n, c), ld=True, optional=not need_grad),
          _arg(loss_out, "loss_out", _F32, 1), _stream())
    return loss_out, dlogits


# ----------------------------------------------------------------------------- PCA
def sym_eig(Cm: torch.Tensor, max_sweeps: int = 30, tol: float = 4e-6):
    """Eigen-decomposition of a symmetric matrix (destroyed) by parallel one-sided Jacobi.
    Returns (evals [g] descending, evecs [g,g] rows = eigenvectors in the same order, sweeps)."""
    c = _arg(Cm, "C", _F32, (None, None))
    g = Cm.shape[0]
    if Cm.shape[1] != g:
        raise B2Error("sym_eig: need a contiguous square matrix")
    V = torch.empty_like(Cm)
    ev = torch.empty(g, dtype=_F32, device=Cm.device)
    sweeps = C.c_int32(0)
    _call("b2_sym_eig_jacobi_f32", c, _arg(V, "V", _F32, (g, g)), g, max_sweeps, tol, _arg(ev, "evals", _F32, g), C.byref(sweeps),
          *_workspace(64, Cm.device), _stream())
    order = torch.argsort(ev, descending=True)
    return ev[order], V[order], sweeps.value


def pca(X: torch.Tensor, n_components: int, precision: Optional[str] = None):
    """PCA of X [n_samples, n_features] like sklearn.decomposition.PCA(n_components).fit_transform (centred, no whitening).

    Returns dict(scores [n,k] = U·S, components [k,f], explained_variance [k], mean [f]).  Uses the Gram matrix when
    n_samples <= n_features, the covariance matrix otherwise; signs follow sklearn's u-based svd_flip.
    """
    _arg(X, "X", _F32, (None, None), ld=True)
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
        _call("b2_cov_rank1_sub_f32", _arg(Cm, "C", _F32, (f, f)), _arg(mean, "mean", _F32, f), f, float(n), _stream())
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
    zp, ldz = _arg(z, "z", _F32, (None, None), ld=True)
    n, h = z.shape
    m = _arg(mu, "mu", _F32, (None, h))
    K = mu.shape[0]
    q = torch.empty((n, K), dtype=_F32, device=z.device)
    _call("b2_dec_q_f32", zp, ldz, m, n, K, h, alpha, *_arg(q, "q", _F32, (n, K), ld=True), _stream())
    return q


def dec_target(q):
    qp, ldq = _arg(q, "q", _F32, (None, None), ld=True)
    n, K = q.shape
    p = torch.empty((n, K), dtype=_F32, device=q.device)
    cs = colsum(q)
    _call("b2_dec_target_f32", qp, ldq, _arg(cs, "colsum", _F32, K), n, K, *_arg(p, "p", _F32, (n, K), ld=True), _stream())
    return p


def dec_kl_grad(z, mu, p, alpha: float = 0.2, dz=None, dmu=None, loss=None, q_out=None, labels_out=None):
    zp, ldz = _arg(z, "z", _F32, (None, None), ld=True)
    n, h = z.shape
    m = _arg(mu, "mu", _F32, (None, h))
    K = mu.shape[0]
    dz = torch.empty((n, h), dtype=_F32, device=z.device) if dz is None else dz
    dmu = torch.empty((K, h), dtype=_F32, device=z.device) if dmu is None else dmu
    loss = torch.empty(1, dtype=_F32, device=z.device) if loss is None else loss
    _call("b2_dec_kl_grad_f32", zp, ldz, m, *_arg(p, "p", _F32, (n, K), ld=True), n, K, h, alpha,
          *_arg(q_out, "q_out", _F32, (n, K), ld=True, optional=True), *_arg(dz, "dz", _F32, (n, h), ld=True),
          _arg(dmu, "dmu", _F32, (K, h)), _arg(loss, "loss", _F32, 1), _arg(labels_out, "labels_out", _I32, n, optional=True),
          _stream())
    return loss, dz, dmu


def sgd_momentum_step(param, grad, buf, step: int, lr: float, momentum: float = 0.9, weight_decay: float = 0.0):
    p = _arg(param, "param", _F32, None)
    n = param.numel()
    _call("b2_sgd_momentum_step_f32", p, _arg(grad, "grad", _F32, n), _arg(buf, "buf", _F32, n), n, lr, momentum, weight_decay, step,
          _stream())


def exp_adj(D: torch.Tensor, l: float, want_matrix: bool = True, want_sum: bool = False):
    """exp(-D²/(2l²)) elementwise on a dense distance matrix and / or its total sum (fp64)."""
    d = _arg(D, "D", _F32, None)
    n = D.numel()
    out = torch.empty_like(D) if want_matrix else None
    acc = torch.zeros(1, dtype=_F64, device=D.device) if want_sum else None
    _call("b2_exp_adj_f32", d, _arg(out, "out", _F32, n, optional=True), n, float(l), _arg(acc, "sum", _F64, 1, optional=True),
          _stream())
    return out, acc


def clip_grad_norm_(grad: torch.Tensor, max_norm: float, pre_scale: float = 1.0, norm_out: Optional[torch.Tensor] = None):
    """In-place ``clip_grad_norm_`` over one flat bucket (after multiplying it by ``pre_scale``)."""
    g = _arg(grad, "grad", _F32, None)
    ws = torch.empty(1, dtype=_F64, device=grad.device)
    _call("b2_clip_grad_norm_f32", g, grad.numel(), float(pre_scale), float(max_norm), _arg(ws, "sumsq", _F64, 1),
          _arg(norm_out, "norm_out", _F32, 1, optional=True), _stream())
    return grad


def radius_graph(X: torch.Tensor, radius: float) -> "CSR":
    """Unit-weight CSR of all pairs within ``radius`` (self included); ``X`` is [n, d<=4] float64 on the device."""
    x, ldx = _arg(X, "X", _F64, (None, None), ld=True)
    n, d = X.shape
    if n == 0:
        return CSR(torch.zeros(1, dtype=_I32, device=X.device), torch.empty(0, dtype=_I32, device=X.device),
                   torch.empty(0, dtype=_F32, device=X.device), (0, 0))
    ws = _workspace(lib().b2_radius_graph_workspace_bytes(n), X.device)
    rowptr = torch.empty(n + 1, dtype=_I32, device=X.device)
    rp = _arg(rowptr, "rowptr", _I32, n + 1)
    nnz = C.c_int64(0)
    _call("b2_radius_graph_count", x, ldx, n, d, float(radius), rp, C.addressof(nnz), *ws, _stream())
    colidx = torch.empty(nnz.value, dtype=_I32, device=X.device)
    if nnz.value:
        _call("b2_radius_graph_fill", x, ldx, n, d, float(radius), rp, _arg(colidx, "colidx", _I32, nnz.value), _stream())
    vals = torch.ones(nnz.value, dtype=_F32, device=X.device)
    return CSR(rowptr, colidx, vals, (n, n))


NORM_MODE = {"normalize": 0, "standardize": 1, "minmax": 2, "l2": 3}


def matrix_normalize(X: torch.Tensor, mode: str = "normalize", axis: int = 0, eps: float = -1.0, out: Optional[torch.Tensor] = None):
    """``dance.utils.matrix.normalize`` on a CUDA fp32 matrix (utils/matrix.py:8-67)."""
    x, ldx = _arg(X, "X", _F32, (None, None), ld=True)
    if mode not in NORM_MODE:
        raise B2Error(f"matrix_normalize: unknown mode {mode!r}")
    if not (eps == -1 or eps > 0):
        raise ValueError(f"Invalid {eps=!r}. Must be positive or -1, the later set zero entries to one.")
    n, g = X.shape
    out = torch.empty_like(X) if out is None else out
    ws = _workspace(lib().b2_matrix_normalize_workspace_bytes(n, g, axis), X.device)
    _call("b2_matrix_normalize_f32", x, ldx, n, g, NORM_MODE[mode], int(axis), float(eps), *_arg(out, "out", _F32, (n, g), ld=True),
          *ws, _stream())
    return out


def pearson_corr(X: torch.Tensor) -> torch.Tensor:
    """float32(np.corrcoef(X.T)) for X [n, g] — fp64 arithmetic on the device."""
    x, ldx = _arg(X, "X", _F32, (None, None), ld=True)
    n, g = X.shape
    adj = torch.empty((g, g), dtype=_F32, device=X.device)
    nbytes = lib().b2_pearson_corr_workspace_bytes(g)
    ws = torch.empty(nbytes, dtype=_U8, device=X.device)
    _call("b2_pearson_corr_f32", x, ldx, n, g, _arg(adj, "adj", _F32, (g, g)), g, _arg(ws, "workspace", _U8, nbytes), nbytes, _stream())
    return adj


def threshold_graph(adj: torch.Tensor, threshold: float, positive_only: bool = False, normalize_edges: bool = True):
    """Edges of a dense score matrix after thresholding: (src int32, dst int32, w fp32), row-major order."""
    a, lda = _arg(adj, "adj", _F32, (None, None), ld=True)
    g = adj.shape[0]
    if adj.shape[1] != g:
        raise B2Error(f"threshold_graph: adj must be square, got {tuple(adj.shape)}")
    nbytes = lib().b2_threshold_graph_workspace_bytes(g)
    ws = torch.empty(nbytes, dtype=_U8, device=adj.device)   # survives count → fill
    wsp = _arg(ws, "workspace", _U8, nbytes)
    rowptr = torch.empty(g + 1, dtype=_I32, device=adj.device)
    rp = _arg(rowptr, "rowptr", _I32, g + 1)
    nnz = C.c_int64(0)
    _call("b2_threshold_graph_count", a, lda, g, float(threshold), int(positive_only), rp, C.addressof(nnz), wsp, nbytes, _stream())
    E = nnz.value
    src = torch.empty(E, dtype=_I32, device=adj.device)
    dst = torch.empty(E, dtype=_I32, device=adj.device)
    w = torch.empty(E, dtype=_F32, device=adj.device)
    if E:
        _call("b2_threshold_graph_fill", a, lda, g, float(threshold), int(positive_only), rp, int(normalize_edges),
              _arg(src, "src", _I32, E), _arg(dst, "dst", _I32, E), _arg(w, "w", _F32, E), wsp, nbytes, _stream())
    return src, dst, w, rowptr


def umap_connectivities(knn_idx: torch.Tensor, knn_dist: torch.Tensor) -> "CSR":
    """scanpy/umap fuzzy-simplicial-set connectivities from a kNN table whose column 0 is the cell itself."""
    ki = _arg(knn_idx, "knn_idx", _I32, (None, None))
    n, k = knn_idx.shape
    kd = _arg(knn_dist, "knn_dist", _F32, (n, k))
    dev = knn_idx.device
    vals = torch.empty((n, k), dtype=_F32, device=dev)
    sig = torch.empty(n, dtype=_F32, device=dev)
    rho = torch.empty(n, dtype=_F32, device=dev)
    acc = torch.empty(1, dtype=_F64, device=dev)
    _call("b2_umap_fuzzy_knn_f32", ki, kd, n, k, _arg(vals, "vals", _F32, (n, k)), _arg(sig, "sigmas", _F32, n),
          _arg(rho, "rhos", _F32, n), _arg(acc, "sum", _F64, 1), _stream())
    rowptr = torch.arange(0, n * k + 1, k, dtype=_I32, device=dev)
    A0 = CSR(rowptr, knn_idx.reshape(-1).contiguous(), vals.reshape(-1), (n, n))
    T, _ = csr_transpose(A0)          # Aᵀ, ascending columns
    A, _ = csr_transpose(T)           # A again, now with ascending columns too
    nbytes = lib().b2_fuzzy_union_workspace_bytes(n)
    ws = torch.empty(nbytes, dtype=_U8, device=dev)
    wsp = _arg(ws, "workspace", _U8, nbytes)
    rp = torch.empty(n + 1, dtype=_I32, device=dev)
    rpp = _arg(rp, "rowptr", _I32, n + 1)
    nnz = C.c_int64(0)
    _call("b2_fuzzy_union_count", *A.ptrs, *T.ptrs, n, rpp, C.addressof(nnz), wsp, nbytes, _stream())
    E = nnz.value
    ci = torch.empty(E, dtype=_I32, device=dev)
    cv = torch.empty(E, dtype=_F32, device=dev)
    if E:
        _call("b2_fuzzy_union_fill", *A.ptrs, *T.ptrs, n, rpp, _arg(ci, "colidx", _I32, E), _arg(cv, "vals", _F32, E), _stream())
    out = CSR(rp, ci, cv, (n, n))
    out.sigmas, out.rhos = sig, rho
    return out


# ----------------------------------------------------------------------------- GraphSCI path
def batchnorm_fwd(X, gamma, beta, running_mean, running_var, training: bool, momentum: float = 0.1, eps: float = 1e-5,
                  act: Optional[str] = None):
    """nn.BatchNorm1d (+ optional fused ReLU); returns (out, save_mean, save_invstd)."""
    x, ldx = _arg(X, "X", _F32, (None, None), ld=True)
    n, c = X.shape
    out = torch.empty((n, c), dtype=_F32, device=X.device)
    sm = torch.empty(c, dtype=_F32, device=X.device)
    si = torch.empty(c, dtype=_F32, device=X.device)
    ws = _workspace(lib().b2_batchnorm_workspace_bytes(c), X.device)
    _call("b2_batchnorm_fwd_f32", x, ldx, n, c, _arg(gamma, "gamma", _F32, c), _arg(beta, "beta", _F32, c),
          _arg(running_mean, "running_mean", _F32, c), _arg(running_var, "running_var", _F32, c), int(training), momentum, eps, ACT[act],
          *_arg(out, "out", _F32, (n, c), ld=True), _arg(sm, "save_mean", _F32, c), _arg(si, "save_invstd", _F32, c), *ws, _stream())
    return out, sm, si


def batchnorm_bwd(dY, Y, X, gamma, save_mean, save_invstd, act: Optional[str] = None, training: bool = True, dgamma=None, dbeta=None):
    """Returns (dX, dgamma, dbeta); ``Y`` (the forward output) is only read for the fused ReLU."""
    x, ldx = _arg(X, "X", _F32, (None, None), ld=True)
    n, c = X.shape
    dX = torch.empty((n, c), dtype=_F32, device=X.device)
    dgamma = torch.empty(c, dtype=_F32, device=X.device) if dgamma is None else dgamma
    dbeta = torch.empty(c, dtype=_F32, device=X.device) if dbeta is None else dbeta
    ws = _workspace(lib().b2_batchnorm_workspace_bytes(c), X.device)
    _call("b2_batchnorm_bwd_f32", *_arg(dY, "dY", _F32, (n, c), ld=True), *_arg(Y, "Y", _F32, (n, c), ld=True, optional=True), x, ldx,
          n, c, _arg(gamma, "gamma", _F32, c), _arg(save_mean, "save_mean", _F32, c), _arg(save_invstd, "save_invstd", _F32, c),
          ACT[act], int(training), *_arg(dX, "dX", _F32, (n, c), ld=True), _arg(dgamma, "dgamma", _F32, c),
          _arg(dbeta, "dbeta", _F32, c), *ws, _stream())
    return dX, dgamma, dbeta


def zinb_loss_grad(a_pi, b_disp, c_mean, Y, size_factors, mask=None, le: float = 1.0, ke: float = 1.0, want_grad: bool = True,
                   want_outputs: bool = False):
    """Returns (acc3 fp64 {Σnll, Σmse, count}, (d_a, d_b, d_c) | None, (mean, disp, pi) | None)."""
    a, ld = _arg(a_pi, "a_pi", _F32, (None, None), ld=True)
    n, g = a_pi.shape
    b, ldb = _arg(b_disp, "b_disp", _F32, (n, g), ld=True)
    c, ldc = _arg(c_mean, "c_mean", _F32, (n, g), ld=True)
    if ldb != ld or ldc != ld:
        raise B2Error("zinb_loss_grad: a_pi, b_disp and c_mean must share a leading dimension")
    dev = a_pi.device
    acc = torch.empty(3, dtype=_F64, device=dev)
    grads = tuple(torch.empty((n, g), dtype=_F32, device=dev) for _ in range(3)) if want_grad else (None, None, None)
    outs = tuple(torch.empty((n, g), dtype=_F32, device=dev) for _ in range(3)) if want_outputs else (None, None, None)
    if isinstance(mask, torch.Tensor) and mask.dtype == torch.bool:
        mask = mask.view(_U8)
    _call("b2_zinb_loss_grad_f32", a, b, c, ld, *_arg(Y, "Y", _F32, (n, g), ld=True), _arg(size_factors, "size_factors", _F32, n),
          *_arg(mask, "mask", _U8, (n, g), ld=True, optional=True), n, g, le, ke,
          *(_arg(t, "grad", _F32, (n, g), optional=True) for t in grads), g,
          *(_arg(t, "output", _F32, (n, g), optional=True) for t in outs), g, _arg(acc, "acc", _F64, 3), _stream())
    return acc, (grads if want_grad else None), (outs if want_outputs else None)


def adj_sample(mu, log_std, eps):
    m = _arg(mu, "adj_sample: mu", _F32, None)
    n = mu.numel()
    z = torch.empty_like(mu)
    _call("b2_adj_sample_f32", m, _arg(log_std, "adj_sample: log_std", _F32, n), _arg(eps, "adj_sample: eps", _F32, n), n,
          _arg(z, "z", _F32, n), _stream())
    return z


def adj_loss_grad(z, mu, log_std, target, class_weight, coef_ce: float = 0.0, want_grad: bool = True):
    """Returns (acc2 fp64 {Σ CE, Σ KL terms}, dz | None) for the [g, g] adjacency logits."""
    zp = _arg(z, "z", _F32, (None, None))
    g = z.shape[0]
    if z.shape[1] != g:
        raise B2Error(f"adj_loss_grad: z must be square, got {tuple(z.shape)}")
    acc = torch.empty(2, dtype=_F64, device=z.device)
    dz = torch.empty_like(z) if want_grad else None
    _call("b2_adj_loss_grad_f32", zp, _arg(mu, "mu", _F32, g * g), _arg(log_std, "log_std", _F32, g * g),
          _arg(target, "target", _F32, g * g), _arg(class_weight, "class_weight", _F32, g), g, coef_ce,
          _arg(dz, "dz", _F32, g * g, optional=True), _arg(acc, "acc", _F64, 2), _stream())
    return acc, dz


def adj_reparam_bwd(dz, mu, log_std, eps, coef_kl: float):
    m = _arg(mu, "mu", _F32, None)
    n = mu.numel()
    dmu, dls = torch.empty_like(mu), torch.empty_like(mu)
    _call("b2_adj_reparam_bwd_f32", _arg(dz, "dz", _F32, n), m, _arg(log_std, "log_std", _F32, n), _arg(eps, "eps", _F32, n), n, coef_kl,
          _arg(dmu, "dmu", _F32, n), _arg(dls, "dlog_std", _F32, n), _stream())
    return dmu, dls


# ----------------------------------------------------------------------------- scGNN EM-iteration stages (csrc/em.cu)
def kmeans(X: torch.Tensor, centers: torch.Tensor, max_iter: int = 300, tol: float = 1e-4):
    """Lloyd iterations of ``sklearn.cluster.KMeans(init=centers, n_init=1)`` on the device (scgnn2.py:186).

    ``centers`` [k, d] is updated in place.  Stops when no label changes or when ‖ΔC‖² ≤ tol·mean(var(X, axis=0)) (sklearn's
    rule), then runs a final assignment so that labels are consistent with the returned centres.
    Returns (labels int32 [n], inertia float, n_iter)."""
    x, ldx = _arg(X, "X", _F32, (None, None), ld=True)
    n, d = X.shape
    cp = _arg(centers, "centers", _F32, (None, d))
    k = centers.shape[0]
    labels = torch.full((n, ), -1, dtype=_I32, device=X.device)
    stats = torch.zeros(3, dtype=_F64, device=X.device)
    args = (cp, k, _arg(labels, "labels", _I32, n))
    tail = (_arg(stats, "stats", _F64, 3), *_workspace(lib().b2_kmeans_workspace_bytes(k, d), X.device), _stream())
    tol_abs = float(tol * X.var(dim=0, unbiased=False).mean().item())

    def step(update):
        _call("b2_kmeans_step_f32", x, ldx, n, d, *args, int(update), *tail)
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
    n = A.shape[0]
    lab = _arg(labels, "labels", _I32, (n, ))
    if n_clusters is None:
        n_clusters = int(labels.max().item()) + 1 if n else 1
    w = torch.empty(n, dtype=_F32, device=labels.device)
    sums = torch.empty(max(n_clusters, 1), dtype=_F64, device=labels.device)
    _call("b2_graph_regu_weights_f32", *A.ptrs[:2], lab, n, int(n_clusters), _arg(sums, "cluster_sums", _F64, sums.numel()),
          _arg(w, "w", _F32, n), _stream())
    return w


def graph_regu_weights_weighted(rowptr: torch.Tensor, colidx: torch.Tensor, vals: torch.Tensor, labels: torch.Tensor,
                                n_clusters: Optional[int] = None) -> torch.Tensor:
    """:func:`graph_regu_weights` for a weighted, directed adjacency (CSR with fp64 ``vals``, the ``adj`` of
    graph_AE_retain_weights): w_j = colsum_j · Σ_{i ∈ cluster(j)} 1/rowsum_i (see b2_graph_regu_weights_weighted_f32)."""
    rp = _arg(rowptr, "rowptr", _I32, (None, ))
    n = rowptr.numel() - 1
    ci = _arg(colidx, "colidx", _I32, (None, ), empty=rp)
    v = _arg(vals, "vals", _F64, (colidx.numel(), ), empty=rp)
    lab = _arg(labels, "labels", _I32, (n, ))
    if n_clusters is None:
        n_clusters = int(labels.max().item()) + 1 if n else 1
    w = torch.empty(n, dtype=_F32, device=labels.device)
    scratch = torch.empty(n + max(n_clusters, 1), dtype=_F64, device=labels.device)
    _call("b2_graph_regu_weights_weighted_f32", rp, ci, v, lab, n, int(n_clusters), _arg(scratch, "scratch", _F64, scratch.numel()),
          _arg(w, "w", _F32, n), _stream())
    return w


def celltype_loss_grad(recon, target, x_dropout, row_weight, relu_mask=True, grad=None, loss_out=None):
    """loss_function_graph(regularizer_type="Celltype") (scgnn2.py:1316-1326): returns (loss_out[1] accumulated, d loss / d recon)."""
    r = _arg(recon, "recon", _F32, (None, None))
    rows, cols = recon.shape
    xd = _arg(x_dropout, "x_dropout", _F32, (rows, None))
    if x_dropout.shape[1] > cols:
        raise B2Error("celltype_loss_grad: x_dropout has more columns than recon")
    if grad is None:
        grad = torch.empty_like(recon)
    if loss_out is None:
        loss_out = torch.zeros(1, dtype=_F32, device=recon.device)
    scratch = torch.empty(2, dtype=_F64, device=recon.device)
    _call("b2_celltype_loss_grad_f32", r, _arg(target, "target", _F32, (rows, cols)), xd, _arg(row_weight, "row_weight", _F32, (rows, )),
          rows, cols, x_dropout.shape[1], int(relu_mask), _arg(grad, "grad", _F32, rows * cols), _arg(loss_out, "loss_out", _F32, 1),
          _arg(scratch, "scratch", _F64, 2), _stream())
    return loss_out, grad


def l1_grad_add(param, grad, coef: float = 1.0, l1_out=None):
    p = _arg(param, "param", _F32, None)
    n = param.numel()
    _call("b2_l1_grad_add_f32", p, _arg(grad, "grad", _F32, n), n, float(coef), _arg(l1_out, "l1_out", _F32, 1, optional=True), _stream())


def louvain_host(indptr, indices, weights=None, max_levels: int = 0, min_gain: float = 1e-7):
    """Multilevel Louvain on a symmetric CSR in host memory (numpy arrays): returns (labels int32 [n], n_communities, modularity)."""
    import numpy as np
    indptr = np.ascontiguousarray(indptr, dtype=np.int64)
    indices = np.ascontiguousarray(indices, dtype=np.int32)
    w = None if weights is None else np.ascontiguousarray(weights, dtype=np.float64)
    n = indptr.shape[0] - 1
    labels = np.empty(n, dtype=np.int32)
    nc, mod = C.c_int32(), C.c_double()
    _call("b2_louvain_csr_host", indptr.ctypes.data, indices.ctypes.data, None if w is None else w.ctypes.data, n, labels.ctypes.data,
          C.byref(nc), C.byref(mod), int(max_levels), float(min_gain))
    return labels, nc.value, mod.value


# ----------------------------------------------------------------------------- pre-processing reductions (csrc/prep.cu)
def gene_stats(X: torch.Tensor, want_sumsq: bool = True, want_nnz: bool = True):
    """Per-gene (column) Σx, Σx², #(x>0) in fp64: returns (sum, sumsq | None, nnz | None)."""
    x, ldx = _arg(X, "X", _F32, (None, None), ld=True)
    n, g = X.shape
    mk = lambda: torch.empty(g, dtype=_F64, device=X.device)
    s, q, k = mk(), (mk() if want_sumsq else None), (mk() if want_nnz else None)
    _call("b2_gene_stats_f32", x, ldx, n, g, _arg(s, "sum", _F64, g), _arg(q, "sumsq", _F64, g, optional=True),
          _arg(k, "nnz", _F64, g, optional=True), _stream())
    return s, q, k


def cell_stats(X: torch.Tensor, want_nnz: bool = True):
    """Per-cell (row) Σx and #(x>0) in fp64."""
    x, ldx = _arg(X, "X", _F32, (None, None), ld=True)
    n, g = X.shape
    s = torch.empty(n, dtype=_F64, device=X.device)
    k = torch.empty(n, dtype=_F64, device=X.device) if want_nnz else None
    _call("b2_cell_stats_f32", x, ldx, n, g, _arg(s, "sum", _F64, n), _arg(k, "nnz", _F64, n, optional=True), _stream())
    return s, k


def subset(X: torch.Tensor, rows: Optional[torch.Tensor] = None, cols: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``X[rows][:, cols]`` as a new dense matrix (``None`` keeps the axis)."""
    x, ldx = _arg(X, "X", _F32, (None, None), ld=True)
    r = _arg(rows, "rows", _I64, (None, ), optional=True)
    c = _arg(cols, "cols", _I32, (None, ), optional=True)
    n_out = X.shape[0] if rows is None else rows.numel()
    g_out = X.shape[1] if cols is None else cols.numel()
    out = torch.empty((n_out, g_out), dtype=_F32, device=X.device)
    _call("b2_subset_f32", x, ldx, r, c, n_out, g_out, _arg(out, "out", _F32, (n_out, g_out)), max(g_out, 1), _stream())
    return out


def cellwise_mask(X: torch.Tensor, mask_rate: float = 0.1, min_gene_counts: int = 5, distr: str = "exp", add_test_mask: bool = False,
                  seed: int = 0):
    """CellwiseMaskData masks (train, valid, test) as bool [n, g] device tensors."""
    x, ldx = _arg(X, "X", _F32, (None, None), ld=True)
    if distr not in ("exp", "uniform"):
        raise ValueError(f"Unknown distribution function option {distr!r}, available options are: 'exp', 'uniform'")
    n, g = X.shape
    masks = [torch.empty((n, g), dtype=_U8, device=X.device) for _ in range(3)]
    over = torch.zeros(1, dtype=_I32, device=X.device)
    _call("b2_cellwise_mask_u8", x, ldx, n, g, float(mask_rate), int(min_gene_counts), int(distr == "exp"), int(add_test_mask),
          int(seed) & 0xFFFFFFFF, *(_arg(m, "mask", _U8, (n, g)) for m in masks), _arg(over, "overflow_rows", _I32, 1), _stream())
    tr, va, te = masks
    return tr.view(torch.bool), va.view(torch.bool), te.view(torch.bool), int(over.item())


def locality_order(X: torch.Tensor, n_anchors: int = 64, iters: int = 4, seed: int = 0):
    """A cell order that keeps each thread block's gathers of the aggregate inside a few L2-resident row ranges: cells are grouped
    by their nearest of ``n_anchors`` centroids (a few Lloyd iterations from seeded random rows, ``b2_kmeans_step_f32``) and the
    groups laid out contiguously.  Returns (perm, inv): row i of the reordered problem is cell ``perm[i]``; ``inv[perm] = arange``.
    Relabelling a kNN index table: ``inv[idx[perm]]``.  The graph and every quantity derived from it are permutation-equivariant,
    so a model run in this order and un-permuted at the end returns the same result (up to summation order)."""
    _arg(X, "X", _F32, (None, None), ld=True)
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
    b, ldb = _arg(base, "base", _F32, (None, None), ld=True)
    rows, cols = base.shape
    if rows == 0 or cols == 0:
        raise ValueError("quantiles: base is empty")
    qh = (C.c_float * len(qs))(*[float(q) for q in qs])
    ws = _workspace(lib().b2_quantiles_workspace_bytes(), base.device)
    _call("b2_quantiles_f32", b, ldb, rows, cols, qh, len(qs), _arg(out, "out", _F64, len(qs) + 3), *ws, _stream())


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
    xp, ldx = _arg(x, "x", _F32, (None, None), ld=True)
    rows, cols = x.shape
    cmin = torch.empty(cols, dtype=_F32, device=x.device)
    cmax = torch.empty(cols, dtype=_F32, device=x.device)
    ws = _workspace(lib().b2_col_minmax_workspace_bytes(cols), x.device)
    _call("b2_col_minmax_f32", xp, ldx, rows, cols, _arg(cmin, "cmin", _F32, cols), _arg(cmax, "cmax", _F32, cols),
          _arg(nonfinite, "nonfinite", _F64, 1, optional=True), *ws, _stream())
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
    lp, ldl = _arg(left, "left", _F32, (None, None), ld=True)
    n, a = left.shape
    rp, ldr = _arg(right, "right", _F32, (n, None), ld=True)
    e = right.shape[1]
    pitch = (a + e + 3) // 4 * 4
    out = torch.empty((n, pitch), dtype=_F32, device=left.device)
    lo = hi = 0.0
    cmin = cmax = None
    if base is not None:
        res = torch.empty(6, dtype=_F64, device=left.device)   # q0.9, q0.1, min, max, #non-finite base, #non-finite right
        _quantiles_launch(base, (0.9, 0.1), res[0:5])
        cmin, cmax = col_minmax(right, nonfinite=res[5:6])
        upper, lower, bmin, bmax, bad_base, bad_right = res.tolist()
        if bad_base > 0:
            raise ValueError(f"normalizer: base holds {int(bad_base)} non-finite values")
        if bad_right > 0:
            raise ValueError(f"normalizer: the matrix to scale holds {int(bad_right)} non-finite values")
        lo, hi = _feature_range(base, upper, lower, bmin, bmax)
    ws = _workspace(lib().b2_concat_scaled_workspace_bytes(e), left.device)
    _call("b2_concat_scaled_f32", lp, ldl, a, rp, ldr, e, n, _arg(cmin, "cmin", _F32, e, optional=True),
          _arg(cmax, "cmax", _F32, e, optional=True), lo, hi, int(base is not None), _arg(out, "out", _F32, (n, pitch)), pitch, *ws,
          _stream())
    return out[:, :a + e]


# ----------------------------------------------------------------------------- graph-sc mini-batch blocks (csrc/graphsc.cu)
def graphsc_block_degrees(A: CSR, dst: torch.Tensor, outdeg: Optional[torch.Tensor] = None, src_cap: int = 0):
    """Out-degrees of the block whose destinations are ``dst`` (int32, −1 = padding) over the destination-indexed CSR ``A``.
    Returns ``outdeg`` [n_nodes] int32, or with ``src_cap`` > 0 ``(outdeg, src_list [src_cap], src_pos [n_nodes])``: the block's
    source nodes (first-touch order, −1 padded) and each one's slot."""
    d = _arg(dst, "dst", _I32, (None, ))
    n = A.shape[0]
    dev = dst.device
    outdeg = torch.empty(n, dtype=_I32, device=dev) if outdeg is None else outdeg
    lst = pos = cnt = None
    if src_cap > 0:
        lst = torch.empty(src_cap, dtype=_I32, device=dev)
        pos = torch.empty(n, dtype=_I32, device=dev)
        cnt = torch.empty(1, dtype=_I32, device=dev)
    _call("b2_graphsc_block_degrees", *A.ptrs[:2], n, d, dst.numel(), _arg(outdeg, "outdeg", _I32, (n, ), at_least=True),
          _arg(lst, "src_list", _I32, src_cap, optional=True), _arg(pos, "src_pos", _I32, n, optional=True),
          _arg(cnt, "n_src", _I32, 1, optional=True), int(src_cap), _stream())
    return outdeg if src_cap <= 0 else (outdeg, lst, pos)


def graphsc_block_aggregate(A: CSR, dst: torch.Tensor, outdeg: torch.Tensor, x: torch.Tensor, agg: str = "sum", p: float = 0.0,
                            seed: int = 0, key: int = 0, x_pos: Optional[torch.Tensor] = None, transposed: bool = False,
                            out_rows: int = 0, out: Optional[torch.Tensor] = None):
    """WeightedGraphConv's normalised aggregation over a block (graphsc.py:445-477, before the product with W), with the
    layer's input dropout (rows keyed by global node id).  ``transposed``: its adjoint, from [len(dst), F] to [out_rows, F]
    rows ``x_pos[u]`` (or u).  See include/dance_b200.h.  Without ``x_pos`` the node-side operand (``x``, or ``out`` when
    transposed) has a row for every node of the graph."""
    d = _arg(dst, "dst", _I32, (None, ))
    n, n_dst = A.shape[0], dst.numel()
    deg = _arg(outdeg, "outdeg", _I32, (n, ), at_least=True)
    xpos = _arg(x_pos, "x_pos", _I32, (n, ), at_least=True, optional=True)
    if agg not in ("sum", "mean"):
        raise ValueError(f"agg must be 'sum' or 'mean', got {agg!r}")
    node_rows = n if x_pos is None else None
    xp, ldx = _arg(x, "x", _F32, (n_dst, None) if transposed else (node_rows, None), ld=True, at_least=not transposed)
    F = x.shape[1]
    if out is None:
        out = torch.empty((int(out_rows) if transposed else n_dst, F), dtype=_F32, device=x.device)
    o, ldo = _arg(out, "out", _F32, (node_rows, F) if transposed else (n_dst, F), ld=True, at_least=transposed)
    _call("b2_graphsc_block_aggregate_f32", *A.ptrs, d, n_dst, deg, xp, ldx, xpos, F, int(agg == "mean"), float(p), int(seed) & 0xFFFFFFFF,
          int(key) & 0xFFFFFFFF, int(transposed), o, ldo, out.shape[0] if transposed else 0, _stream())
    return out


def graphsc_batch_decoder(z: torch.Tensor, p: float = 0.1, seed: int = 0, key: int = 0, dz: Optional[torch.Tensor] = None,
                          loss: Optional[torch.Tensor] = None):
    """graph-sc's loss on one batch (graphsc.py:208-216 with InnerProductDecoder :408-411): ``norm · BCEWithLogits(z̃z̃ᵀ, I,
    pos_weight)`` with the decoder's own dropout (rows = batch positions).  Returns (loss [1] on the device, dz)."""
    zp, ldz = _arg(z, "z", _F32, (None, None), ld=True)
    if dz is None:
        dz = torch.empty_like(z)
    if loss is None:
        loss = torch.empty(1, dtype=_F32, device=z.device)
    _call("b2_graphsc_batch_decoder_f32", zp, ldz, z.shape[0], z.shape[1], float(p), int(seed) & 0xFFFFFFFF, int(key) & 0xFFFFFFFF,
          *_arg(dz, "dz", _F32, tuple(z.shape), ld=True), _arg(loss, "loss", _F32, 1), _stream())
    return loss, dz


def graphsc_scatter_rows(x: torch.Tensor, idx: torch.Tensor, out: torch.Tensor, offset: int = 0):
    """``out[idx[i] − offset] = x[i]``."""
    xp, ldx = _arg(x, "x", _F32, (None, None), ld=True)
    rows, cols = x.shape
    _call("b2_graphsc_scatter_rows_f32", xp, ldx, rows, cols, _arg(idx, "idx", _I32, (rows, )), int(offset),
          *_arg(out, "out", _F32, (None, cols), ld=True), _stream())
    return out
