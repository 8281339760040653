"""numpy restatement of scGNN's ``normalizer(X, base)`` (scgnn2.py:795-805) with every float32 rounding step spelled out
(test infrastructure).  It is the specification ``ops.quantiles`` / ``ops.concat_normalized`` are checked against bit for bit.

* :func:`quantile` — ``np.quantile(base, q)`` (method "linear") over all elements of a float32 array.  numpy casts q to float32, so
  the virtual index ``(n − 1)·q`` is a float32 product with n − 1 rounded to float32 (numpy/lib/_function_base_impl.py,
  ``_get_indexes``: at or past the last index both neighbours are the maximum); the weight is the exact fractional part, and
  ``_lerp`` is ``a + (b−a)·t``, or ``b − (b−a)·(1−t)`` when t ≥ 0.5, each operation rounded to float32.  A zero order statistic
  is taken as +0.0: numpy's partition does not order −0.0 against +0.0.
* :func:`normalizer` — feature range (q0.1, q0.9) of base, or (q0, q1) when they are equal, then sklearn's
  ``minmax_scale(X, feature_range, axis=0)`` in float32 (MinMaxScaler.partial_fit: scale_ = (hi − lo) / range with ranges below
  10·eps set to 1, min_ = lo − data_min·scale_; transform ``X *= scale_; X += min_``).  An empty range raises like sklearn.
"""
from __future__ import annotations

import numpy as np

f32 = np.float32


def plan(n: int, q: float):
    """(previous index, next index, weight) numpy's quantile uses for n values."""
    nm1 = f32(n - 1)
    v = nm1 * f32(q)
    if v >= nm1:
        return n - 1, n - 1, f32(0)
    prev = int(np.floor(v))
    return prev, min(prev + 1, n - 1), f32(float(v) - prev)


def lerp(a, b, t):
    a, b, t = f32(a), f32(b), f32(t)
    d = b - a
    return b - d * (f32(1) - t) if t >= f32(0.5) else a + d * t


def quantile(base, q: float) -> np.float32:
    a = np.asarray(base, dtype=np.float32).ravel()
    prev, nxt, t = plan(a.size, q)
    part = np.partition(a, sorted({prev, nxt}))
    with np.errstate(over="ignore", invalid="ignore"):
        return lerp(part[prev] + f32(0), part[nxt] + f32(0), t)


def feature_range(base):
    upper, lower = quantile(base, 0.9), quantile(base, 0.1)
    lo, hi = (lower, upper) if upper != lower else (quantile(base, 0.0), quantile(base, 1.0))
    if lo >= hi:
        raise ValueError(f"Minimum of desired feature range must be smaller than maximum. Got {(lo, hi)}.")
    return lo, hi


def minmax_scale(X, lo, hi):
    X = np.array(X, dtype=np.float32)
    dmin, dmax = np.nanmin(X, axis=0), np.nanmax(X, axis=0)
    rng = dmax - dmin
    rng[rng < f32(10) * np.finfo(np.float32).eps] = f32(1)
    scale = (f32(hi) - f32(lo)) / rng
    shift = f32(lo) - dmin * scale
    X *= scale
    X += shift
    return X


def normalizer(X, base):
    lo, hi = feature_range(base)
    return minmax_scale(X, lo, hi)


def concat_normalized(left, right, base=None):
    right = np.asarray(right, dtype=np.float32) if base is None else normalizer(right, base)
    return np.concatenate((np.asarray(left, dtype=np.float32), right), axis=1)
