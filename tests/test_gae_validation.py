"""Argument validation of the two Graph-AE decoder entry points (no GPU needed), with unit labels (vals NULL) and with
real-valued labels (vals and the transposed labels t_* set).

Every case below is rejected before any CUDA call, so it runs on a machine without a device and the stand-in pointers are
never dereferenced.  That includes an embedding size the label kernels are not built for: it is refused up front, before dz
is zeroed or anything is launched."""
import pytest

INVALID, UNSUPPORTED = -1, -3
P = 1 << 20          # a 16-byte aligned stand-in address
ROWS, SYM = "b2_gae_loss_grad_f32", "b2_gae_loss_grad_sym_f32"
N = 1000             # 8 row blocks, 4 super-blocks


def _args(fn, vals, **kw):
    from dance_b200 import _lib
    t = P if vals else None          # unit labels pass no transposed labels
    a = dict(z=P, ldz=64, mu=None, logvar=None, ldm=0, rowptr=P, colidx=P, vals=vals, t_rowptr=t, t_colidx=t, t_vals=t, n=N, d=16,
             sb_begin=0, sb_end=_lib.lib().b2_gae_sym_super_blocks(N), row_begin=0, n_rows=N, norm=1.0, pw=1.0, use_pw=1, dz=P,
             dmu=None, dlogvar=None, ldd=0, loss=P, ws=P, ws_bytes=1 << 30)
    a.update(kw)
    order = ["z", "ldz", "mu", "logvar", "ldm", "rowptr", "colidx", "vals", "t_rowptr", "t_colidx", "t_vals", "n", "d"] + \
            (["sb_begin", "sb_end"] if fn == SYM else []) + \
            ["row_begin", "n_rows", "norm", "pw", "use_pw", "dz", "dmu", "dlogvar", "ldd", "loss", "ws", "ws_bytes"]
    return [a[k] for k in order] + [None]


KLD = {"mu": P, "logvar": P, "ldm": 16, "dmu": P, "dlogvar": P, "ldd": 16}

COMMON = [
    # both entry points alike
    *[(fn, {k: None}, INVALID) for fn in (ROWS, SYM) for k in ("z", "rowptr", "colidx", "dz", "loss")],
    *[(fn, kw, INVALID) for fn in (ROWS, SYM) for kw in (
        {"n": 0}, {"n": -1}, {"d": 0}, {"d": -8}, {"ldz": 15},
        {"row_begin": -1}, {"n_rows": -1}, {"row_begin": 500, "n_rows": 501},
        {"ws": None}, {"ws_bytes": 255},
        {"mu": P}, {"logvar": P},
        {**KLD, "dmu": None}, {**KLD, "dlogvar": None}, {**KLD, "ldm": 15}, {**KLD, "ldd": 15},
    )],
    # pair-sharded form: d <= 16, the super-block range, the tensor-core workspace
    (SYM, {"d": 32}, INVALID),
    (SYM, {"sb_begin": -1}, INVALID),
    (SYM, {"sb_begin": 3, "sb_end": 2}, INVALID),
    (SYM, {"sb_end": 5}, INVALID),
    (SYM, {"ws_bytes": 256}, INVALID),
    # embedding sizes without a label kernel
    (ROWS, {"d": 12}, UNSUPPORTED),
    (ROWS, {"d": 40}, UNSUPPORTED),
    (SYM, {"d": 12}, UNSUPPORTED),
]
CASES = [(fn, vals, kw, status) for vals in (None, P) for fn, kw, status in COMMON] + \
        [(fn, P, {k: None}, INVALID) for fn in (ROWS, SYM) for k in ("t_rowptr", "t_colidx", "t_vals")]   # values need Lᵀ


@pytest.mark.parametrize("fn,vals,kw,status", CASES,
                         ids=[f"{'sym' if c[0] == SYM else 'rows'}-{'vals' if c[1] else 'unit'}-{'-'.join(f'{k}={v}' for k, v in c[2].items())}"
                              for c in CASES])
def test_gae_entry_point_validation(fn, vals, kw, status):
    from dance_b200 import _lib
    lib = _lib.lib()
    assert getattr(lib, fn)(*_args(fn, vals, **kw)) == status
    assert lib.b2_last_error().decode().startswith(fn + ":")
