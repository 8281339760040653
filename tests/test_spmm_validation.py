"""Argument validation of the three SpMM entry points (no GPU needed).

Validation returns before any CUDA call and n_rows = 0 returns B2_OK right after it, so every case below runs on a machine
without a device; the pointers are never dereferenced.  The one case with n_rows > 0, fp32 F = 516, is turned down by the
nnz-stream dispatch and the row-group ladder on the host before anything is launched."""
import pytest

OK, INVALID, UNSUPPORTED = 0, -1, -3
P = 1 << 20          # a 16-byte aligned stand-in address
F32, BF16, F16 = "b2_spmm_csr_f32", "b2_spmm_csr_bf16", "b2_spmm_csr_f16"


def _args(fn, **kw):
    a = dict(rowptr=P, colidx=P, vals=None, X=P, ldx=64, Y=P, ldy=64, Y16=None, ldy16=0, n_rows=0, n_cols=0, F=64, reduce=0,
             act=0, bias=None)
    a.update(kw)
    order = ["rowptr", "colidx", "vals", "X", "ldx", "Y", "ldy"] + ([] if fn == F32 else ["Y16", "ldy16"]) + \
            ["n_rows", "n_cols", "F", "reduce", "act", "bias"]
    return [a[k] for k in order] + [None]


CASES = [
    # every entry point: a valid call, and what all three reject alike
    *[(fn, {}, OK) for fn in (F32, BF16, F16)],
    *[(fn, {"reduce": 1, "act": 3, "vals": P, "bias": P}, OK) for fn in (F32, BF16, F16)],
    *[(fn, {k: None}, INVALID) for fn in (F32, BF16, F16) for k in ("rowptr", "colidx", "X")],
    *[(fn, {"n_rows": -1}, INVALID) for fn in (F32, BF16, F16)],
    *[(fn, {"n_cols": -1}, INVALID) for fn in (F32, BF16, F16)],
    *[(fn, {"F": 0}, INVALID) for fn in (F32, BF16, F16)],
    *[(fn, {"reduce": 2}, INVALID) for fn in (F32, BF16, F16)],
    *[(fn, {"ldx": 56}, INVALID) for fn in (F32, BF16, F16)],
    *[(fn, {"ldy": 56}, INVALID) for fn in (F32, BF16, F16)],
    *[(fn, {"ldy": 66}, INVALID) for fn in (F32, BF16, F16)],
    *[(fn, {"X": P + 4}, INVALID) for fn in (F32, BF16, F16)],
    *[(fn, {"Y": P + 8}, INVALID) for fn in (F32, BF16, F16)],
    # fp32: F % 4, F <= 512 (wider is unsupported, checked after the n_rows == 0 return), Y required, 16-byte aligned bias
    (F32, {"F": 6, "ldx": 8, "ldy": 8}, INVALID),
    (F32, {"F": 12, "ldx": 12, "ldy": 12}, OK),
    (F32, {"ldx": 68}, OK),
    (F32, {"ldx": 66}, INVALID),
    (F32, {"F": 512, "ldx": 512, "ldy": 512}, OK),
    (F32, {"F": 516, "ldx": 516, "ldy": 516}, OK),
    (F32, {"F": 516, "ldx": 516, "ldy": 516, "n_rows": 1, "n_cols": 1}, UNSUPPORTED),
    (F32, {"Y": None}, INVALID),
    (F32, {"bias": P + 4}, INVALID),
    # bf16 / fp16: F % 8, F <= 256, Y may be NULL when Y16 is given, any 4-byte aligned bias
    *[(fn, kw, st) for fn in (BF16, F16) for kw, st in (
        ({"F": 12, "ldx": 16, "ldy": 16}, INVALID),
        ({"F": 8, "ldx": 8, "ldy": 8}, OK),
        ({"F": 104, "ldx": 104, "ldy": 104}, OK),
        ({"ldx": 68}, INVALID),
        ({"ldx": 72}, OK),
        ({"F": 256, "ldx": 256, "ldy": 256}, OK),
        ({"F": 264, "ldx": 264, "ldy": 264}, INVALID),
        ({"F": 264, "ldx": 264, "ldy": 264, "n_rows": 1, "n_cols": 1}, INVALID),
        ({"Y": None, "Y16": P, "ldy16": 64}, OK),
        ({"Y": None, "Y16": None}, INVALID),
        ({"Y16": P, "ldy16": 64}, OK),
        ({"Y16": P, "ldy16": 56}, INVALID),
        ({"Y16": P, "ldy16": 68}, INVALID),
        ({"Y16": P + 8, "ldy16": 64}, INVALID),
        ({"bias": P + 4}, OK),
    )],
]


@pytest.mark.parametrize("fn,kw,status", CASES, ids=[f"{c[0][12:]}-{'-'.join(f'{k}={v}' for k, v in c[1].items()) or 'valid'}"
                                                     for c in CASES])
def test_spmm_entry_point_validation(fn, kw, status):
    from dance_b200 import _lib
    assert getattr(_lib.lib(), fn)(*_args(fn, **kw)) == status
