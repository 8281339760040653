"""Argument validation of the fused GraphSCI heads entry points and of the BatchNorm statistics entry point (no GPU needed):
every case is rejected before any CUDA call, so the stand-in pointers are never dereferenced."""
import pytest

INVALID = -1
P = 1 << 20          # a 16-byte aligned stand-in address

STATS = "b2_batchnorm_stats_f32"
TRAIN = "b2_graphsci_heads_train_f32"
EVAL = "b2_graphsci_heads_eval_f32"
HEAD = ["pre_pi", "pre_disp", "pre_mean", "ldp", "gamma", "beta", "mean", "invstd", "Y", "ldy", "size_factors", "mask", "ldm", "n", "g"]
ORDER = {
    STATS: ["X", "ldx", "n", "c", "running_mean", "running_var", "training", "momentum", "eps", "save_mean", "save_invstd",
            "workspace", "workspace_bytes"],
    TRAIN: HEAD + ["le", "ke", "dgamma", "dbeta", "acc3", "workspace", "workspace_bytes"],
    EVAL: HEAD + ["accumulate", "acc3", "z_exp", "ldz"],
}
HEAD_OK = dict(pre_pi=P, pre_disp=P, pre_mean=P, ldp=50, gamma=P, beta=P, mean=P, invstd=P, Y=P, ldy=50, size_factors=P, mask=P,
               ldm=50, n=100, g=50)
DEFAULTS = {
    STATS: dict(X=P, ldx=50, n=100, c=50, running_mean=P, running_var=P, training=1, momentum=0.1, eps=1e-5, save_mean=P,
                save_invstd=P, workspace=P, workspace_bytes=1 << 20),
    TRAIN: dict(HEAD_OK, le=1.0, ke=1.0, dgamma=P, dbeta=P, acc3=P, workspace=P, workspace_bytes=1 << 20),
    EVAL: dict(HEAD_OK, accumulate=0, acc3=P, z_exp=P, ldz=50),
}
CASES = [
    *[(STATS, {k: None}) for k in ("running_mean", "running_var", "save_mean", "save_invstd", "X", "workspace")],
    (STATS, {"n": 0}), (STATS, {"c": 0}), (STATS, {"c": -1}), (STATS, {"ldx": 49}), (STATS, {"workspace_bytes": 16}),
    *[(fn, {k: None}) for fn in (TRAIN, EVAL) for k in ("pre_pi", "pre_disp", "pre_mean", "gamma", "beta", "mean", "invstd", "Y",
                                                        "size_factors", "acc3")],
    *[(fn, {k: 0}) for fn in (TRAIN, EVAL) for k in ("n", "g")],
    *[(fn, {k: -3}) for fn in (TRAIN, EVAL) for k in ("n", "g")],
    *[(fn, {k: 49}) for fn in (TRAIN, EVAL) for k in ("ldp", "ldy", "ldm")],
    (TRAIN, {"dgamma": None}), (TRAIN, {"dbeta": None}), (TRAIN, {"workspace": None}), (TRAIN, {"workspace_bytes": 16}),
    (EVAL, {"ldz": 49}),
]


@pytest.mark.parametrize("fn,kw", CASES, ids=[f"{c[0][3:]}-{'-'.join(f'{k}={v}' for k, v in c[1].items())}" for c in CASES])
def test_graphsci_heads_entry_point_validation(fn, kw):
    from dance_b200 import _lib
    lib = _lib.lib()
    a = dict(DEFAULTS[fn], **kw)
    assert getattr(lib, fn)(*[a[k] for k in ORDER[fn]], None) == INVALID
    msg = lib.b2_last_error().decode()
    assert msg.startswith(fn + ":") and len(msg) > len(fn) + 2, msg


def test_eval_statistics_need_no_matrix():
    """Eval-mode statistics come from the running statistics: X may be NULL (rejected only for the workspace here)."""
    from dance_b200 import _lib
    lib = _lib.lib()
    a = dict(DEFAULTS[STATS], X=None, ldx=0, training=0, workspace=None)
    assert lib.b2_batchnorm_stats_f32(*[a[k] for k in ORDER[STATS]], None) == INVALID
    assert "workspace" in lib.b2_last_error().decode()


def test_bindings_refuse_cpu_tensors(monkeypatch):
    """dance_b200.graphsci_ops checks every tensor at the ops boundary: CPU tensors are refused before the library is reached."""
    import torch

    from dance_b200 import graphsci_ops, ops
    from dance_b200._lib import B2Error

    def no_library():
        raise AssertionError("the library was reached")
    monkeypatch.setattr(ops, "_raw_lib", no_library)
    n, g = 4, 5
    pre = [torch.zeros(n, g) for _ in range(3)]
    vec = [torch.zeros(3, g) for _ in range(4)]
    calls = [lambda: graphsci_ops.batchnorm_stats(torch.zeros(n, g), torch.zeros(g), torch.ones(g), True),
             lambda: graphsci_ops.heads_train(pre, *vec, torch.zeros(n, g), torch.ones(n)),
             lambda: graphsci_ops.heads_eval(pre, *vec, torch.zeros(n, g), torch.ones(n))]
    for call in calls:
        with pytest.raises(B2Error, match="expected a CUDA tensor"):
            call()
