"""Mirror of ``dance/utils/matrix.py`` for the functions on the hot path: ``normalize`` (:8-67) and ``pairwise_distance``
(:164-180), executed by the device kernels, and ``SpotDistance``, the coordinate-backed form of the spot distance matrix."""
from __future__ import annotations

import hashlib

import numpy as np
import torch

from . import ops


def normalize(mat, *, mode: str = "normalize", axis: int = 0, eps: float = -1.0):
    """Same contract as the reference: numpy in → numpy out, torch in → torch (CUDA) out; 2-D fp32."""
    if isinstance(mat, torch.Tensor):
        is_torch = True
    elif not isinstance(mat, np.ndarray):
        raise TypeError(f"Invalid type for input matrix: {type(mat)}")
    else:
        is_torch = False
    if mode not in ops.NORM_MODE:       # the reference silently returns mat / 1 for unknown modes (denom = None → 1)
        if not (eps == -1 or eps > 0):
            raise ValueError(f"Invalid {eps=!r}. Must be positive or -1, the later set zero entries to one.")
        return mat / 1
    X = mat if is_torch else torch.as_tensor(np.ascontiguousarray(mat, dtype=np.float32))
    X = X.to(device="cuda", dtype=torch.float32).contiguous()
    if X.dim() != 2:
        raise ValueError("normalize: 2-D input expected")
    out = ops.matrix_normalize(X, mode, axis % 2, eps)
    return out if is_torch else out.cpu().numpy()


def pairwise_distance(x: np.ndarray, dist_func_id: int = 0) -> np.ndarray:
    if dist_func_id != 0:
        raise NotImplementedError("only the euclidean distance (dist_func_id=0) is built")
    X = torch.as_tensor(np.ascontiguousarray(x, dtype=np.float32)).cuda()
    return ops.pairwise_l2_dense(X).cpu().numpy()


def _frozen(a) -> np.ndarray:
    """A read-only C-contiguous fp32 copy of ``a``."""
    out = np.array(a, dtype=np.float32, order="C", copy=True)
    out.flags.writeable = False
    return out


class SpotDistance:
    """The euclidean distance matrix between a row and a column set of spot coordinates, held as the coordinates.

    What ``pairwise_distance`` stores in ``obsp`` for SpaGCN is 4·N² bytes; this is the same matrix as 4·d·N: ``toarray()`` /
    ``np.asarray`` give ``ops.pairwise_l2_dense``'s entries bit for bit, and the SpaGCN consumers (``calculate_p`` /
    ``search_l``, ``SimpleGCDEC.bind``, ``refine``) sweep the coordinates on the device instead.  With ``l`` set it stands for the
    exponentiated matrix ``exp(-D²/(2 l²))`` that ``SpaGCN.calc_adj_exp`` returns.  ``m[rows]``, ``m[:, cols]`` and
    ``m[rows][:, cols]`` subset the coordinate sets, as ``Data`` filtering and split access do to ``obsp`` entries.  The host
    coordinates are read-only fp32 numpy copies made on construction, so the object pickles and its content cannot change
    under the device copies, which are cached per device and not pickled."""

    dtype = np.dtype(np.float32)
    ndim = 2

    def __init__(self, rows, cols=None, l=None):
        rows = _frozen(rows)
        cols = rows if cols is None else _frozen(cols)
        if rows.ndim != 2 or cols.ndim != 2 or rows.shape[1] != cols.shape[1] or not 1 <= rows.shape[1] <= 4:
            raise ValueError(f"SpotDistance: coordinate sets [n, d] with the same 1 <= d <= 4 expected, got {rows.shape} and {cols.shape}")
        if l is not None and not float(l) > 0:
            raise ValueError(f"SpotDistance: l must be positive, got {l}")
        self.rows, self.cols, self.l = rows, cols, None if l is None else float(l)
        self._dev = {}

    @property
    def shape(self):
        return (self.rows.shape[0], self.cols.shape[0])

    def exp(self, l) -> "SpotDistance":
        """The exponentiated form ``exp(-D²/(2 l²))`` of this distance matrix (shares the device copy)."""
        if self.l is not None:
            raise ValueError("SpotDistance.exp: the matrix is already exponentiated")
        out = SpotDistance.__new__(SpotDistance)
        out.rows, out.cols, out.l, out._dev = self.rows, self.cols, float(l), self._dev   # same coordinates, same uploads
        if not out.l > 0:
            raise ValueError(f"SpotDistance: l must be positive, got {l}")
        return out

    def device_coords(self, device=None):
        """(rows, cols) as fp32 tensors on ``device`` (default: the current CUDA device), uploaded once per device."""
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if dev.type == "cuda" and dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        if dev not in self._dev:
            r = torch.tensor(self.rows, device=dev)
            self._dev[dev] = (r, r if self.cols is self.rows else torch.tensor(self.cols, device=dev))
        return self._dev[dev]

    def fingerprint(self) -> tuple:
        """Content key of the matrix: the coordinates' digest and ``l``."""
        h = hashlib.sha1(self.rows.tobytes())
        h.update(b"|" if self.cols is self.rows else self.cols.tobytes())
        return (self.shape, self.rows.shape[1], h.hexdigest(), self.l)

    def to_device(self) -> torch.Tensor:
        """The materialised matrix as a CUDA tensor (``pairwise_l2_dense``, then ``exp_adj`` when ``l`` is set)."""
        r, c = self.device_coords()
        if r is c:
            D = ops.pairwise_l2_dense(r)
        else:   # each entry depends on its own pair only, so the rows × cols block of the joint matrix is the same bits
            D = ops.pairwise_l2_dense(torch.cat([r, c]))[:r.shape[0], r.shape[0]:].contiguous()
        return D if self.l is None else ops.exp_adj(D, self.l)[0]

    def toarray(self) -> np.ndarray:
        return self.to_device().cpu().numpy()

    def __array__(self, dtype=None, copy=None):
        a = self.toarray()
        return a if dtype is None else a.astype(dtype)

    def __getitem__(self, key):
        r, c = key if isinstance(key, tuple) else (key, slice(None))
        full = lambda k: isinstance(k, slice) and k == slice(None)
        rows = self.rows if full(r) else self.rows[r]
        cols = self.cols if full(c) else self.cols[c]
        if rows.ndim != 2 or cols.ndim != 2:
            raise IndexError("SpotDistance takes row and column subsets (slices, index arrays, masks), not single entries")
        if full(r) and full(c):
            return self
        out = SpotDistance.__new__(SpotDistance)
        out.rows = self.rows if full(r) else _frozen(rows)
        out.cols = self.cols if full(c) else _frozen(cols)
        out.l, out._dev = self.l, {}
        return out

    def __getstate__(self):
        return {"rows": self.rows, "cols": self.cols, "l": self.l, "same": self.cols is self.rows}

    def __setstate__(self, state):
        self.rows, self.l, self._dev = _frozen(state["rows"]), state["l"], {}
        self.cols = self.rows if state["same"] else _frozen(state["cols"])

    def __repr__(self):
        kind = "distance" if self.l is None else f"exp(-D²/2l²), l={self.l!r}"
        return f"SpotDistance({self.shape[0]} x {self.shape[1]}, d={self.rows.shape[1]}, {kind})"
