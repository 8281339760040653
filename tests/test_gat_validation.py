"""Argument validation of the GAT aggregate and combine entry points' options (no GPU needed): attention dropout, the tied
second layer, the identity skip and the combine's activation code.  Every case is rejected before any CUDA call, so the
stand-in pointers are never dereferenced."""
import pytest

INVALID = -1
P = 1 << 20          # a 16-byte aligned stand-in address
N, NH, F = 1000, 2, 16
FWD, BWD = "b2_gat_aggregate_fwd_f32", "b2_gat_aggregate_bwd_f32"
CFWD, CBWD = "b2_gat_combine_fwd_f32", "b2_gat_combine_bwd_f32"
W = NH * F


def _args(fn, **kw):
    a = dict(rowptr=P, colidx=P, t_rowptr=P, t_colidx=P, t_perm=P, H=P, ldh=W, a_src=P, a_trg=P, s_src=P, s_trg=P, alpha=P, dOut=P,
             lddo=W, H2=None, ldh2=0, dOut2=None, lddo2=0, n=N, nheads=NH, F=F, act=0, slope=0.2, shift_mode=0, gmax=P, out=P, ldo=W,
             dH=P, lddh=W, dH2=None, lddh2=0, da_src=P, da_trg=P, ds_src=P, ds_trg=P, dpre=P, shift_ws=P, drop_p=0.0, seed=1, key=2,
             agg=P, ldagg=W, skip=P, ldskip=F, bias=None, concat=1, identity_skip=1, dout=P, ldp=W, dact=None, ldact=0, dx_skip=P, ldx=F)
    a.update(kw)
    order = {
        FWD: ["rowptr", "colidx", "H", "ldh", "s_src", "s_trg", "n", "nheads", "F", "act", "slope", "shift_mode", "gmax", "out", "ldo",
              "alpha", "drop_p", "seed", "key"],
        BWD: ["rowptr", "colidx", "t_rowptr", "t_colidx", "t_perm", "H", "ldh", "a_src", "a_trg", "s_src", "s_trg", "alpha", "dOut",
              "lddo", "H2", "ldh2", "dOut2", "lddo2", "n", "nheads", "F", "act", "slope", "gmax", "dH", "lddh", "dH2", "lddh2",
              "da_src", "da_trg", "ds_src", "ds_trg", "dpre", "shift_ws", "drop_p", "seed", "key"],
        CFWD: ["agg", "ldagg", "skip", "ldskip", "bias", "n", "nheads", "F", "concat", "act", "identity_skip", "out", "ldo"],
        CBWD: ["dout", "lddo", "out", "ldo", "n", "nheads", "F", "concat", "act", "dpre", "ldp", "dact", "ldact", "dx_skip", "ldx"],
    }[fn]
    return [a[k] for k in order] + [None]


TIED = {"H2": P, "ldh2": W, "dOut2": P, "lddo2": W}
CASES = [
    # attention dropout: a probability in [0, 1]; more than 32 heads only without it
    *[(fn, {"drop_p": p}) for fn in (FWD, BWD) for p in (float("nan"), -0.1, 1.5)],
    (FWD, {"drop_p": 0.5, "nheads": 33, "F": 8, "ldh": 264, "ldo": 264}),
    # the tied second layer needs its upstream gradient and takes no attention dropout
    (BWD, {**TIED, "dOut2": None}),
    (BWD, {**TIED, "drop_p": 0.5}),
    # an identity skip is the [n, F] input itself
    (CFWD, {"skip": None}),
    (CFWD, {"ldskip": F - 1}),
    (CBWD, {"ldx": F - 1}),
    # the combine's activation is an epilogue code (NONE..TANH)
    *[(fn, {"act": a}) for fn in (CFWD, CBWD) for a in (-1, 4, 5)],
]


@pytest.mark.parametrize("fn,kw", CASES, ids=[f"{c[0][7:-4]}-{'-'.join(f'{k}={v}' for k, v in c[1].items())}" for c in CASES])
def test_gat_entry_point_validation(fn, kw):
    from dance_b200 import _lib
    lib = _lib.lib()
    assert getattr(lib, fn)(*_args(fn, **kw)) == INVALID
    assert lib.b2_last_error().decode().startswith(fn + ":")
