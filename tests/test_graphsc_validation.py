"""Argument validation of the graph-sc entry points and of the activation pair b2_act_f32 / b2_act_bwd_f32 (no GPU needed):
every case is rejected before any CUDA call, so it runs on a machine without a device and the stand-in pointers are never
dereferenced."""
import pytest

INVALID = -1
P = 1 << 20          # a 16-byte aligned stand-in address

DEG = "b2_graphsc_block_degrees"
AGG = "b2_graphsc_block_aggregate_f32"
DEC = "b2_graphsc_batch_decoder_f32"
ACT = "b2_act_bwd_f32"
FWD = "b2_act_f32"
SCAT = "b2_graphsc_scatter_rows_f32"

ORDER = {
    DEG: ["rowptr", "colidx", "n_nodes", "dst", "n_dst", "outdeg", "src_list", "src_pos", "n_src", "src_cap"],
    AGG: ["rowptr", "colidx", "weights", "dst", "n_dst", "outdeg", "x", "ldx", "x_pos", "F", "agg_mean", "p", "seed", "key",
          "transposed", "out", "ldo", "out_rows"],
    DEC: ["z", "ldz", "B", "d", "p", "seed", "key", "dz", "lddz", "loss"],
    ACT: ["dy", "lddy", "y", "ldy", "x", "ldx", "rows", "cols", "act", "dx", "lddx"],
    SCAT: ["x", "ldx", "rows", "cols", "idx", "offset", "out", "ldo"],
    FWD: ["x", "ldx", "rows", "cols", "act", "y", "ldy"],
}
DEFAULTS = {
    DEG: dict(rowptr=P, colidx=P, n_nodes=100, dst=P, n_dst=10, outdeg=P, src_list=None, src_pos=None, n_src=None, src_cap=0),
    AGG: dict(rowptr=P, colidx=P, weights=P, dst=P, n_dst=10, outdeg=P, x=P, ldx=50, x_pos=None, F=50, agg_mean=0, p=0.1, seed=0,
              key=0, transposed=0, out=P, ldo=50, out_rows=0),
    DEC: dict(z=P, ldz=300, B=128, d=300, p=0.1, seed=0, key=0, dz=P, lddz=300, loss=P),
    ACT: dict(dy=P, lddy=8, y=P, ldy=8, x=P, ldx=8, rows=4, cols=8, act=1, dx=P, lddx=8),
    SCAT: dict(x=P, ldx=8, rows=4, cols=8, idx=P, offset=0, out=P, ldo=8),
    FWD: dict(x=P, ldx=8, rows=4, cols=8, act=5, y=P, ldy=8),
}
CASES = [
    *[(DEG, {k: None}) for k in ("rowptr", "colidx", "outdeg", "dst")],
    (DEG, {"n_nodes": 0}), (DEG, {"n_dst": -1}),
    (DEG, {"src_list": P}), (DEG, {"src_list": P, "src_pos": P, "n_src": P}), (DEG, {"src_pos": P, "n_src": P, "src_cap": 5}),
    *[(AGG, {k: None}) for k in ("rowptr", "colidx", "dst", "outdeg", "x", "out")],
    (AGG, {"F": 0}), (AGG, {"ldx": 49}), (AGG, {"ldo": 49}), (AGG, {"n_dst": -1}), (AGG, {"agg_mean": 2}), (AGG, {"p": 1.0}),
    (AGG, {"p": -0.1}), (AGG, {"transposed": 2}), (AGG, {"transposed": 1}), (AGG, {"out_rows": -1}),
    *[(DEC, {k: None}) for k in ("z", "dz", "loss")],
    (DEC, {"B": 0}), (DEC, {"d": 0}), (DEC, {"d": 1025, "ldz": 1025, "lddz": 1025}), (DEC, {"ldz": 299}), (DEC, {"lddz": 299}),
    (DEC, {"p": 1.0}), (DEC, {"p": -0.5}),
    (ACT, {"dy": None}), (ACT, {"dx": None}), (ACT, {"act": 6}), (ACT, {"act": -1}), (ACT, {"y": None}), (ACT, {"act": 5, "x": None}),
    (ACT, {"lddy": 7}), (ACT, {"lddx": 7}), (ACT, {"ldy": 7}), (ACT, {"rows": -1}),
    *[(SCAT, {k: None}) for k in ("x", "idx", "out")],
    (SCAT, {"ldx": 7}), (SCAT, {"ldo": 7}), (SCAT, {"rows": -1}),
    (FWD, {"x": None}), (FWD, {"y": None}), (FWD, {"act": 6}), (FWD, {"ldx": 7}), (FWD, {"ldy": 7}),
]


@pytest.mark.parametrize("fn,kw", CASES, ids=[f"{c[0][3:]}-{'-'.join(f'{k}={v}' for k, v in c[1].items())}" for c in CASES])
def test_graphsc_entry_point_validation(fn, kw):
    from dance_b200 import _lib
    lib = _lib.lib()
    a = dict(DEFAULTS[fn], **kw)
    assert getattr(lib, fn)(*[a[k] for k in ORDER[fn]], None) == INVALID
    assert lib.b2_last_error().decode().startswith(fn + ":")


def test_activation_codes_are_additions():
    """leaky_relu and gelu take new codes for the elementwise entry points; the epilogues' table is unchanged."""
    from dance_b200 import ops
    assert ops.ACT == {"none": 0, None: 0, "relu": 1, "elu": 2, "tanh": 3}
    assert ops.ACT_ALL == {**ops.ACT, "leaky_relu": 4, "gelu": 5}
