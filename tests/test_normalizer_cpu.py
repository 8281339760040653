"""scGNN's normalizer without a GPU: the float32 restatement in ``normalizer_ref`` against the reference's own ``normalizer``
(numpy quantile + sklearn minmax_scale), bit for bit, and argument validation of the new C entry points (rejected before any CUDA
call, so stand-in pointers are never dereferenced).

Outputs are compared as bit patterns after adding +0.0, which makes −0.0 and +0.0 one value: which of two equal zeros numpy's
partition leaves at an index is not specified, and the restatement takes +0.0."""
import ctypes

import numpy as np
import pytest

import normalizer_ref as nr
from oracle import ref_loader

P = 1 << 20          # a 16-byte aligned stand-in address
f32 = np.float32

needs_ref = pytest.mark.skipif(not ref_loader.available(), reason="reference sources not present")


def bits(a):
    return (np.asarray(a, dtype=np.float32) + f32(0)).view(np.uint32)


def _ref_normalizer():
    return ref_loader.scgnn2().normalizer


def _cases():
    rng = np.random.default_rng(11)
    yield "negative_zeros_ties", (rng.integers(-3, 4, size=(37, 5)).astype(np.float32) * f32(0.5)), \
        np.where(rng.random((53, 7)) < 0.2, f32(-0.0), rng.integers(-4, 5, size=(53, 7)).astype(np.float32))
    yield "t_at_least_half", rng.standard_normal((20, 3)).astype(np.float32), rng.standard_normal((7, 1)).astype(np.float32)
    near = rng.standard_normal((40, 4)).astype(np.float32)
    near[:, 1] = f32(1.0)
    near[::2, 1] = np.nextafter(f32(1.0), f32(2.0))                # range 1.2e-7 < 10·eps: scale set to 1
    yield "near_constant_column", near, rng.standard_normal((30, 30)).astype(np.float32)
    sparse = np.where(rng.random((200, 50)) < 0.95, f32(0), rng.gamma(2.0, 1.0, size=(200, 50)).astype(np.float32))
    yield "upper_equals_lower", rng.standard_normal((200, 16)).astype(np.float32), sparse


@needs_ref
@pytest.mark.parametrize("name,X,base", list(_cases()), ids=[c[0] for c in _cases()])
def test_restatement_equals_reference_normalizer(name, X, base):
    ref = _ref_normalizer()(X, base=base, axis=0)
    assert ref.dtype == np.float32
    mine = nr.normalizer(X, base)
    assert np.array_equal(bits(mine), bits(ref))
    if name == "upper_equals_lower":
        assert np.quantile(base, 0.9) == np.quantile(base, 0.1)
    if name == "t_at_least_half":
        assert nr.plan(base.size, 0.1)[2] >= 0.5 and nr.plan(base.size, 0.9)[2] < 0.5


def test_quantile_index_is_a_float32_product():
    """Above 2²⁴ values (n − 1)·q is rounded to float32, and numpy picks its neighbours from the rounded index."""
    n = (1 << 24) + 11
    base = np.random.default_rng(3).permutation(n).astype(np.float32)     # distinct exact integers 0 … n−1 (below 2²⁵)
    prev, nxt, t = nr.plan(n, 0.9)
    assert prev != int(np.floor((n - 1) * 0.9)) or t != f32(((n - 1) * 0.9) % 1.0)   # the float64 index would differ
    for q in (0.1, 0.9):
        assert bits(nr.quantile(base, q)) == bits(np.quantile(base, q))


@needs_ref
def test_restatement_equals_reference_above_2_24_values():
    rng = np.random.default_rng(5)
    base = rng.standard_normal(((1 << 24) // 64 + 3, 64)).astype(np.float32)
    X = rng.standard_normal((100, 16)).astype(np.float32)
    assert base.size > (1 << 24)
    assert np.array_equal(bits(nr.normalizer(X, base)), bits(_ref_normalizer()(X, base=base, axis=0)))


@needs_ref
def test_degenerate_base_raises_like_reference():
    X = np.ones((5, 2), dtype=np.float32)
    base = np.full((4, 3), 2.5, dtype=np.float32)
    with pytest.raises(ValueError, match="Minimum of desired feature range must be smaller than maximum"):
        _ref_normalizer()(X, base=base, axis=0)
    with pytest.raises(ValueError, match="Minimum of desired feature range must be smaller than maximum"):
        nr.normalizer(X, base)


def test_quantile_matches_numpy_on_small_sizes():
    rng = np.random.default_rng(8)
    for n in (1, 2, 3, 5, 10, 11, 101, 1000, 4097):
        a = rng.standard_normal(n).astype(np.float32)
        for q in (0.0, 0.1, 0.5, 0.9, 1.0):
            assert bits(nr.quantile(a, q)) == bits(np.quantile(a, q)), (n, q)


def _lib():
    from dance_b200 import _lib
    return _lib.lib()


def test_quantiles_validation():
    lib = _lib()
    ws = lib.b2_quantiles_workspace_bytes()
    qs = (ctypes.c_float * 2)(0.9, 0.1)
    ok = dict(base=P, ldb=8, rows=4, cols=8, qs=qs, nq=2, out=P, ws=P, wsb=ws)
    bad = [dict(base=None), dict(rows=0), dict(cols=0), dict(ldb=7), dict(nq=0), dict(nq=3), dict(out=None), dict(wsb=ws - 1),
           dict(qs=(ctypes.c_float * 2)(1.5, 0.1))]
    for b in bad:
        a = {**ok, **b}
        assert lib.b2_quantiles_f32(a["base"], a["ldb"], a["rows"], a["cols"], a["qs"], a["nq"], a["out"], a["ws"], a["wsb"], None) == -1, b


def test_col_minmax_and_concat_validation():
    lib = _lib()
    ws = lib.b2_col_minmax_workspace_bytes(16)
    assert lib.b2_col_minmax_f32(P, 16, 0, 16, P, P, None, P, ws, None) == -1
    assert lib.b2_col_minmax_f32(P, 15, 4, 16, P, P, None, P, ws, None) == -1
    assert lib.b2_col_minmax_f32(P, 16, 4, 16, P, P, None, P, ws - 1, None) == -1
    cw = lib.b2_concat_scaled_workspace_bytes(16)
    call = lambda ldo, out=P, scale=1, wsb=cw: lib.b2_concat_scaled_f32(P, 128, 128, P, 16, 16, 10, P, P, 0.0, 1.0, scale, out, ldo,
                                                                         P, wsb, None)
    assert call(146) == -1                  # pitch not a multiple of 4
    assert call(140) == -1                  # pitch below a + e
    assert call(144, out=P + 4) == -1       # out not 16-byte aligned
    assert call(144, wsb=cw - 1) == -1      # scaling without its workspace


def test_fixture_inputs_are_the_restated_concatenations(golden):
    """The widened matrices the reference's handlers trained on (recorded in the fixture) are [X | normalizer(graph_embed, X)],
    [X | feature_embed] and [X_embed | normalizer(graph_embed, X_embed)] of the restatement, bit for bit."""
    g = golden("scgnn_concat_prev_embed")
    X, ge, fe, xe = g["X"], g["graph_embed"], g["feature_embed"], g["x_embed"]
    for e in (1, 2):
        assert np.array_equal(bits(g[f"fae.graph.e{e}.X"]), bits(nr.concat_normalized(X, ge, X)))
        assert np.array_equal(bits(g[f"fae.feature.e{e}.X"]), bits(nr.concat_normalized(X, fe)))
    for branch in ("gcn", "gat"):
        assert np.array_equal(bits(g[f"gae.{branch}.e1.X"]), bits(nr.concat_normalized(xe, ge, xe)))
        assert np.array_equal(bits(g[f"gae.{branch}.e0.X"]), bits(xe))
    assert [str(g[f"fae.graph.e{e}.loaded"]) for e in (0, 1, 2)] == ["none", "none", "model_concat"]
