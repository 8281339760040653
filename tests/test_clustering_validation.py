"""Argument validation of the clustering entry points (no GPU needed): the DEC head's b2_dec_q_f32, b2_dec_target_f32 and
b2_dec_kl_grad_f32, and b2_kmeans_step_f32.  Every case is rejected before any CUDA call, so it runs on a machine without a
device and the stand-in pointers are never dereferenced."""
import pytest

INVALID = -1
P = 1 << 20          # a 16-byte aligned stand-in address
N, K, H = 100, 10, 50

DEC_Q = ["z", "ldz", "mu", "n", "K", "h", "alpha", "q", "ldq"]
DEC_Q_CASES = [{"z": None}, {"mu": None}, {"q": None}, {"n": -1}, {"K": 0}, {"K": 65}, {"h": 0}, {"ldz": H - 1}, {"ldq": K - 1}]

DEC_TARGET = ["q", "ldq", "colsum", "n", "K", "p", "ldp"]
DEC_TARGET_CASES = [{"q": None}, {"colsum": None}, {"p": None}, {"n": -1}, {"K": 0}, {"K": 65}, {"ldq": K - 1}, {"ldp": K - 1}]

DEC_KL = ["z", "ldz", "mu", "p", "ldp", "n", "K", "h", "alpha", "q_out", "ldq", "dz", "lddz", "dmu", "loss", "labels"]
DEC_KL_CASES = [*[{k: None} for k in ("z", "mu", "p", "dz", "dmu", "loss")], {"n": 0}, {"n": -1}, {"K": 0}, {"K": 65}, {"h": 0},
                {"ldz": H - 1}, {"ldp": K - 1}, {"lddz": H - 1}, {"ldq": K - 1}, {"ldq": 0}]

KMEANS = ["X", "ldx", "n", "d", "C", "k", "labels", "update", "stats", "workspace", "workspace_bytes"]
# k·d·4 = 96 KB + 4 bytes: one float more than the centroids' shared-memory stage holds
KMEANS_CASES = [*[{k: None} for k in ("X", "C", "labels", "stats", "workspace")], {"n": 0}, {"d": 0}, {"k": 0}, {"ldx": 15},
                {"workspace_bytes": "short"}, {"k": 7, "d": 3511, "ldx": 3511}]


def _ids(cases):
    return ["-".join(f"{k}={v}" for k, v in c.items()) for c in cases]


def _expect_invalid(fn, args, name):
    from dance_b200 import _lib
    assert fn(*args, None) == INVALID
    assert _lib.lib().b2_last_error().decode().startswith(f"{name}:")


@pytest.mark.parametrize("kw", DEC_Q_CASES, ids=_ids(DEC_Q_CASES))
def test_dec_q_validation(kw):
    from dance_b200 import _lib
    a = dict(dict(z=P, ldz=H, mu=P, n=N, K=K, h=H, alpha=0.2, q=P, ldq=K), **kw)
    _expect_invalid(_lib.lib().b2_dec_q_f32, [a[k] for k in DEC_Q], "b2_dec_q_f32")


@pytest.mark.parametrize("kw", DEC_TARGET_CASES, ids=_ids(DEC_TARGET_CASES))
def test_dec_target_validation(kw):
    from dance_b200 import _lib
    a = dict(dict(q=P, ldq=K, colsum=P, n=N, K=K, p=P, ldp=K), **kw)
    _expect_invalid(_lib.lib().b2_dec_target_f32, [a[k] for k in DEC_TARGET], "b2_dec_target_f32")


@pytest.mark.parametrize("kw", DEC_KL_CASES, ids=_ids(DEC_KL_CASES))
def test_dec_kl_grad_validation(kw):
    """Every leading dimension is checked: ldz >= h, ldp >= K, lddz >= h, and ldq >= K when q_out is given."""
    from dance_b200 import _lib
    a = dict(dict(z=P, ldz=H, mu=P, p=P, ldp=K, n=N, K=K, h=H, alpha=0.2, q_out=P, ldq=K, dz=P, lddz=H, dmu=P, loss=P, labels=P),
             **kw)
    _expect_invalid(_lib.lib().b2_dec_kl_grad_f32, [a[k] for k in DEC_KL], "b2_dec_kl_grad_f32")


@pytest.mark.parametrize("kw", KMEANS_CASES, ids=_ids(KMEANS_CASES))
def test_kmeans_step_validation(kw):
    from dance_b200 import _lib
    lib = _lib.lib()
    a = dict(dict(X=P, ldx=16, n=N, d=16, C=P, k=8, labels=P, update=1, stats=P, workspace=P, workspace_bytes=None), **kw)
    need = lib.b2_kmeans_workspace_bytes(a["k"], a["d"])
    a["workspace_bytes"] = need - 1 if a["workspace_bytes"] == "short" else need
    _expect_invalid(lib.b2_kmeans_step_f32, [a[k] for k in KMEANS], "b2_kmeans_step_f32")
