"""Models trained with precision="bf16": the string reaches every GEMM, and a step matches a float64 restatement whose products
round their operands to bf16 the way the kernel does (tests/bf16_ref.py)."""
import numpy as np
import pytest
import torch

from bf16_ref import feature_ae_step_bf16
from conftest import rel_err
from oracle.scgnn_step_ref import FEATURE_AE_PARAMS

pytestmark = pytest.mark.gpu

# Bounds, about 5x the errors measured on an H100 80 GB HBM3 at a 700 W power limit.  The bf16 restatement rounds float64
# activations and the engine rounds its float32 ones, so an operand within ~1e-7 of a bf16 rounding boundary can land one bf16
# ulp (2^-8) apart; the weight gradients are, besides, ill-conditioned at initialisation (see test_gpu_scgnn_step.py).
# Measured: loss 4.8e-7; z / recon 2.3e-5 / 1.3e-4, worst row 2.6e-3; weight gradients 2.1e-4, worst row 2.4e-2 (fc3).
TOL_FAE = dict(loss=3e-6, act=6e-4, act_row=1.2e-2, grad=1e-3, grad_row=1.2e-1)
# GraphSCI after one epoch, bf16 against tf32x3 (the same model, the same noise).  Measured: train_loss and kl 2.2e-2 (the kl
# term is a difference of two near-equal terms), the other losses at most 4.5e-4; weight matrices at most 1.1e-2 (conv1).
# Vectors (biases, BatchNorm affine) are bounded element-wise by the optimiser step instead: a first Adam step moves each
# parameter by about lr·sign(g), and the biases in front of a BatchNorm have gradients at rounding level in any precision.
TOL_GRAPHSCI = dict(loss=1e-1, loss_other=3e-3, weights=5e-2, vector_step=2.5)


def row_rel_err(a, ref):
    """Worst row of ‖a_i − ref_i‖ / ‖ref_i‖, with rows below 1e-3 of the RMS row norm measured against that floor."""
    a, ref = torch.as_tensor(a).double(), torch.as_tensor(ref).double().to(a.device)
    a, ref = a.reshape(a.shape[0], -1), ref.reshape(ref.shape[0], -1)
    den = ref.norm(dim=1)
    floor = 1e-3 * float(den.pow(2).mean().sqrt())
    return float(((a - ref).norm(dim=1) / den.clamp(min=max(floor, 1e-300))).max())


class _Checks:
    """Every comparison of a test, asserted together at the end so that a failure reports all of them."""

    def __init__(self):
        self.rows = []

    def __call__(self, what, err, tol):
        self.rows.append((what, float(err), tol))
        print(f"bf16 model error {what}: {err:.3g}")

    def done(self):
        bad = [f"{w}: {e:.3g} > {t:.3g}" for w, e, t in self.rows if not e < t]
        assert not bad, "\n".join(bad)


def test_feature_ae_step_bf16(cuda):
    """One 12 800 × 2 000 Feature-AE batch in bf16 (split-K weight gradients, BN = 128 tiles), against the bf16 restatement."""
    from dance_b200 import ops, synth
    from dance_b200.engine import FeatureAEEngine
    n, genes = 12800, 2000
    X = synth.expression_counts(n, genes, seed=0, density=0.10, device=cuda)
    ops.normalize_total_log1p_(X, target_sum=1e4, max_fraction=1.0)
    assert ops.lib().b2_gemm_workspace_bytes(genes, FeatureAEEngine.HID, n, 1, 0, ops.PREC["bf16"]) > 0     # split-K fc1 gradient
    eng = FeatureAEEngine(genes, device=cuda, lr=1e-3, precision="bf16", seed=0)
    steps = []
    eng.grad_hook = lambda g: steps.append((eng.params.flat.clone(), g.clone()))
    z_all = torch.empty(n, FeatureAEEngine.EMB, device=cuda)
    r_all = torch.empty_like(X)
    loss = eng.train_epoch(X, n, "LTMG", 0.9, None, z_all, r_all).item()
    assert len(steps) == 1
    flat, grad = steps[0]
    _check = _Checks()
    base = eng.params.flat.storage_offset()

    def views(buf):
        return {k: buf[v.storage_offset() - base:v.storage_offset() - base + v.numel()].view(v.shape) for k, v in eng.params.p.items()}
    ref = feature_ae_step_bf16(X, views(flat), "LTMG", 0.9, None)
    _check("loss", abs(loss - ref["loss"].item()) / abs(ref["loss"].item()), TOL_FAE["loss"])
    for name, got in (("z", z_all), ("recon", r_all)):
        _check(name, rel_err(got, ref[name]), TOL_FAE["act"])
        _check(name + " rows", row_rel_err(got, ref[name]), TOL_FAE["act_row"])
    g = views(grad)
    for k in FEATURE_AE_PARAMS:
        _check("d " + k, rel_err(g[k], ref["grads"][k]), TOL_FAE["grad"])
        if g[k].dim() == 2:
            _check("d " + k + " rows", row_rel_err(g[k], ref["grads"][k]), TOL_FAE["grad_row"])
    _check.done()


def _graphsci(cuda, precision, X, Xraw, graph):
    from dance_b200.modules.graphsci import GraphSCI
    N, G = X.shape
    model = GraphSCI(num_cells=N, num_genes=G, dataset="synthetic", dropout=0.0, gpu=0, seed=0, precision=precision)
    model._bind_graph(graph)
    n_counts = Xraw.sum(1)
    model.size_factors = (n_counts / torch.median(n_counts)).contiguous()
    model.lr, model.weight_decay = 1e-3, 1e-5
    return model


def test_graphsci_epoch_bf16(cuda, monkeypatch):
    """One GraphSCI training epoch at 4 096 cells × 512 genes, where every GEMM of the epoch qualifies for the tensor cores:
    every ops.gemm call carries "bf16", and the losses and weights after the epoch are close to the same epoch in tf32x3."""
    from dance_b200 import ops, synth
    from dance_b200.data import AnnDataLite, Data
    from dance_b200.transforms import FeatureFeatureGraph
    N, G = 4096, 512
    Xraw = synth.expression_counts(N, G, seed=1, density=0.10, device=cuda)
    X = Xraw.clone()
    ops.normalize_total_log1p_(X, normalize=False, log1p=True)
    sample = Data(AnnDataLite(X.cpu().numpy()))
    FeatureFeatureGraph(threshold=0.05, normalize_edges=True)(sample)
    graph = sample.data.uns["FeatureFeatureGraph"]
    graph.ndata["feat"] = X.t().contiguous()
    tm = torch.ones(N, G, dtype=torch.uint8, device=cuda)

    calls = []
    real_gemm = ops.gemm

    def recording_gemm(A, B, *, transA=False, transB=False, precision=None, **kw):
        M, K = (A.shape[1], A.shape[0]) if transA else A.shape
        n_out = B.shape[0] if transB else B.shape[1]
        on_tc = (K >= 8 and M * n_out * K >= (1 << 18) and A.stride(0) % 4 == 0 and B.stride(0) % 4 == 0
                 and A.data_ptr() % 16 == 0 and B.data_ptr() % 16 == 0)
        calls.append((precision, (M, n_out, K), on_tc))
        return real_gemm(A, B, transA=transA, transB=transB, precision=precision, **kw)

    out = {}
    for precision in ("bf16", "tf32x3"):
        model = _graphsci(cuda, precision, X, Xraw, graph)
        calls.clear()
        monkeypatch.setattr(ops, "gemm", recording_gemm)
        model.train(X, Xraw, graph, tm, tm, le=1, la=1e-9, ke=1e2, ka=1)
        monkeypatch.setattr(ops, "gemm", real_gemm)
        torch.cuda.synchronize()
        assert calls and all(c[0] == precision for c in calls), sorted({c[0] for c in calls})
        assert all(c[2] for c in calls), [c[1] for c in calls if not c[2]]
        out[precision] = (model, len(calls))
    (mb, nb), (mr, nr) = out["bf16"], out["tf32x3"]
    assert nb == nr
    _check = _Checks()
    for name in ("train_loss", "valid_loss", "loss_adj", "loss_exp", "kl"):
        a, b = getattr(mb, name), getattr(mr, name)
        _check("graphsci " + name, abs(a - b) / max(abs(b), 1e-30), TOL_GRAPHSCI["loss" if name in ("train_loss", "kl") else "loss_other"])
    for k, w in mr.params.p.items():
        if w.dim() == 2:
            _check("graphsci weight " + k, rel_err(mb.params.p[k], w), TOL_GRAPHSCI["weights"])
        else:
            _check("graphsci vector max|diff|/lr " + k, float((mb.params.p[k] - w).abs().max()) / mr.lr, TOL_GRAPHSCI["vector_step"])
    _check.done()
    assert not np.isclose(rel_err(mb.params.p["aemodel.mul_layer.fc_layer.weight"], mr.params.p["aemodel.mul_layer.fc_layer.weight"]), 0.0)
