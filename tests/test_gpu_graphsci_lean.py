"""GraphSCI's lean training schedule (dance_b200/modules/graphsci.py: ``_train_lean``, ``_evaluate_lean``) and its fused heads
kernels (csrc/graphsci.cu: b2_graphsci_heads_train_f32 / _eval_f32).

* Against the float64 step restatement (oracle/graphsci_step_ref.py) at configuration 3's gene count and at an unaligned
  shape, with and without dropout, in tf32x3 and bf16, with the tolerances of tests/test_gpu_graphsci_step.py.  The lean
  schedule draws its masks from the counter-based hash, so the restatement is fed those masks, materialised with
  ``ops.dropout`` on ones under the same (seed, key).
* Against the materialising schedule at dropout 0 (same data, same ε): the two differ only in summation order (and, in bf16,
  in what that does to the rounded operands).
* Evaluation in row chunks of any size gives the same loss and z_exp.
* Configuration 3 at its full 500 000 cells × 3 000 genes: the lean schedule is chosen, train() and fit() finish within the
  memory bound below, and the fused training kernel is checked against float64 over all 500 000 rows for sampled genes.
"""
import math

import pytest
import torch
import torch.nn.functional as F

import test_gpu_graphsci_step as S
from bf16_ref import Bf16MatMul
from conftest import rel_err
from oracle import graphsci_step_ref as R

pytestmark = pytest.mark.gpu

# Peak of torch.cuda.max_memory_allocated() for two train() steps, and separately for fit(n_epochs=2), of configuration 3 at
# 500 000 × 3 000 (bf16, dropout 0.1) including the caller's X, Xraw, Xᵀ and mask: 64 GiB.  The materialising schedule would
# need about 176 GB (graphsci.schedule_bytes).
FULL_SIZE_PEAK = 64 * 2**30


@pytest.fixture
def schedule(monkeypatch):
    from dance_b200.modules import graphsci

    def set_(name):
        monkeypatch.setattr(graphsci, "SCHEDULE", name)
    return set_


def _model(N, G, precision, dropout, seed, graph, sf):
    from dance_b200.modules.graphsci import GraphSCI
    model = GraphSCI(num_cells=N, num_genes=G, dataset="synthetic", dropout=dropout, gpu=0, seed=seed, precision=precision)
    model._bind_graph(graph)
    model.size_factors = sf
    model.lr, model.weight_decay = S.LR, S.WD
    return model


def _hash_masks(model, N, G, cuda):
    """The keep-masks (scaled by 1 / (1 − p)) the lean schedule's next train() step draws, keyed by restatement site."""
    from dance_b200 import ops
    shapes = {"feat": (G, N), "h1": (G, 256), "h2_mean": (G, 256), "h2_log_std": (G, 256), "X": (N, G), "enc.1": (N, G),
              "enc.5": (N, 256), **{h: (N, 256) for h in R.HEADS}}
    return {site: ops.dropout(torch.ones(shape, device=cuda), model.dropout, model.drop_seed, model.drop_key(site))
            for site, shape in shapes.items()}


def _capture_lean_z_exp(model, cap):
    """train() evaluates without z_exp in the lean schedule; have it write z_exp so that it can be compared."""
    real = model._evaluate_lean

    def evaluate_lean(*a, want_z_exp=True, **kw):
        out = real(*a, want_z_exp=True, **kw)
        cap["z_exp"] = out[2]
        return out
    model._evaluate_lean = evaluate_lean


# bf16 at 4 099 × 1 001 is left to test_lean_matches_materialising below: at 1 001 genes the G-pitched products run on the
# CUDA cores in fp32 while the others round to bf16, so neither the rounded nor the unrounded restatement describes that step
# (tests/test_gpu_graphsci_step.py covers that shape in fp32 / tf32x3 only, for the same reason).
@pytest.mark.parametrize("N,G,precision", [(20012, 3000, "tf32x3"), (20012, 3000, "bf16"), (4099, 1001, "tf32x3")])
@pytest.mark.parametrize("dropout", [0.0, 0.1])
def test_lean_step_against_float64(cuda, schedule, N, G, precision, dropout):
    schedule("lean")
    seed = 0 if G == 3000 else 1
    case = f"lean {N}x{G} {precision} dropout={dropout}"
    Xm, Xraw, graph, train_mask, valid_mask, sf, eps = S._data(cuda, N, G, seed)
    model = _model(N, G, precision, dropout, seed, graph, sf)
    assert model.schedule() == "lean"
    gene_graph = R.GeneGraph(*graph.edges(), G, cuda)
    cap = {}
    _capture_lean_z_exp(model, cap)
    tm, vm = train_mask.view(torch.uint8), valid_mask.view(torch.uint8)
    for step in range(2):
        at = f"{case} step {step + 1}"
        flat0 = model.params.flat.clone()
        run0 = {k: (b.running_mean.clone(), b.running_var.clone()) for k, b in model.bn.items()}
        masks = _hash_masks(model, N, G, cuda) if dropout else None
        model.train(Xm, Xraw, graph, tm, vm, eps_train=eps[2 * step], eps_eval=eps[2 * step + 1], **S.COEF)
        torch.cuda.synchronize()
        grads = S._views(model.params, model.params.grad.clone())
        ref = R.train_step(S._views(model.params, flat0), run0, Xm, Xraw, sf, gene_graph, train_mask, valid_mask,
                           eps_train=eps[2 * step], eps_eval=eps[2 * step + 1], masks=masks,
                           mm=Bf16MatMul.apply if precision == "bf16" else torch.matmul, **S.COEF)
        S._compare_step(at, model, ref, grads, cap.pop("z_exp"), S.TOL[precision])
        del ref, masks, grads
    assert model.drop_step == 2 and model.params.step == 2


# biases in front of a BatchNorm: exact gradient 0, rounding noise in both schedules
ZERO_GRAD = ("aemodel.enc.1.bias", "aemodel.enc.5.bias") + tuple(f"aemodel.{h}.1.bias" for h in R.HEADS)
# Lean against materialising at dropout 0.  The two differ in the heads only: the fused kernel forms the BatchNorm backward's
# column sums from the loss gradient at unit mask count and divides once, zinb_kernel scales each element first, so the heads'
# gradients differ in the last bits.  In tf32x3 that stays at rounding level (measured on an H100 80 GB HBM3 at 700 W: at most
# 5.2e-7 on a gradient); bf16 rounds every GEMM operand to 8 bits, so a last-bit difference can move an operand by one bf16
# ulp, and the gradient bound is wider (measured 9.2e-4, in the conv1 weight at 3 000 genes).  Each step starts both models
# from the same weights, Adam moments and running statistics: Adam moves every bias in front of a BatchNorm by about ±lr on
# its first step, with the sign of a gradient that is rounding noise, so free-running models part after one step.
TOL_SCHEDULES = {"tf32x3": dict(loss=1e-6, grad=1e-5, zero_grad=1e-5, run=1e-5, zexp=1e-5),
                 "bf16": dict(loss=1e-6, grad=3e-3, zero_grad=1e-5, run=1e-5, zexp=1e-5)}


def _copy_state(src, dst):
    for name in ("flat", "exp_avg", "exp_avg_sq"):
        getattr(dst.params, name).copy_(getattr(src.params, name))
    dst.params.step = src.params.step
    for k, b in src.bn.items():
        dst.bn[k].running_mean.copy_(b.running_mean)
        dst.bn[k].running_var.copy_(b.running_var)
        dst.bn[k].num_batches_tracked = b.num_batches_tracked


def _schedule_errors(a, b, grads_a, grads_b, zexp_a, zexp_b):
    """{(kind, name): error} of the lean model b against the materialising model a after the same step."""
    err = {}
    for k in ("loss_adj", "loss_exp", "kl", "train_loss", "valid_loss"):
        err["loss", k] = abs(getattr(b, k) - getattr(a, k)) / abs(getattr(a, k))
    gmax = max(float(v.abs().max()) for v in grads_a.values())
    for k in R.PARAMS:
        if k in ZERO_GRAD:
            err["zero_grad", k] = float((grads_b[k] - grads_a[k]).abs().max()) / gmax
        else:
            err["grad", k] = rel_err(grads_b[k], grads_a[k])
    for k in a.bn:
        err["run", f"running_mean {k}"] = rel_err(b.bn[k].running_mean, a.bn[k].running_mean)
        err["run", f"running_var {k}"] = rel_err(b.bn[k].running_var, a.bn[k].running_var)
    err["zexp", "z_exp"] = rel_err(zexp_b, zexp_a)
    return err


@pytest.mark.parametrize("N,G,precision", [(20012, 3000, "tf32x3"), (20012, 3000, "bf16"), (4099, 1001, "tf32x3"),
                                           (4099, 1001, "bf16")])
def test_lean_matches_materialising(cuda, schedule, N, G, precision):
    """Dropout 0, same data and ε, two steps, each from the same state: the lean schedule against the materialising one."""
    seed = 0 if G == 3000 else 1
    Xm, Xraw, graph, train_mask, valid_mask, sf, eps = S._data(cuda, N, G, seed)
    tm, vm = train_mask.view(torch.uint8), valid_mask.view(torch.uint8)
    models = {s: _model(N, G, precision, 0.0, seed, graph, sf) for s in ("materialise", "lean")}
    cap = {"materialise": {}, "lean": {}}
    real_eval = models["materialise"].evaluate

    def evaluate(*a, **kw):
        out = real_eval(*a, **kw)
        cap["materialise"]["z_exp"] = out[2]
        return out
    models["materialise"].evaluate = evaluate
    _capture_lean_z_exp(models["lean"], cap["lean"])
    tol = TOL_SCHEDULES[precision]
    for step in range(2):
        _copy_state(models["materialise"], models["lean"])
        out = {}
        for s, model in models.items():
            schedule(s)
            assert model.schedule() == s
            model.train(Xm, Xraw, graph, tm, vm, eps_train=eps[2 * step], eps_eval=eps[2 * step + 1], **S.COEF)
            out[s] = (S._views(model.params, model.params.grad.clone()), cap[s].pop("z_exp"))
        torch.cuda.synchronize()
        err = _schedule_errors(models["materialise"], models["lean"], out["materialise"][0], out["lean"][0], out["materialise"][1],
                               out["lean"][1])
        worst = {kind: max((e, n) for (kd, n), e in err.items() if kd == kind) for kind in tol}
        print(f"\nlean vs materialise {N}x{G} {precision} step {step + 1}: " +
              ", ".join(f"{kind} {e:.3g} ({n})" for kind, (e, n) in worst.items()))
        bad = {key: e for key, e in err.items() if not e < tol[key[0]]}
        assert not bad, (precision, step, bad)


def test_evaluation_chunks_agree(cuda, schedule, monkeypatch):
    from dance_b200.modules import graphsci
    schedule("lean")
    N, G = 4099, 1001
    Xm, Xraw, graph, train_mask, valid_mask, sf, eps = S._data(cuda, N, G, 1)
    model = _model(N, G, "fp32", 0.1, 1, graph, sf)        # CUDA-core GEMMs: each row's products do not depend on the chunk
    model.train(Xm, Xraw, graph, train_mask.view(torch.uint8), valid_mask.view(torch.uint8), eps_train=eps[0], eps_eval=eps[1],
                **S.COEF)
    results = {}
    for rows in (1000, 37, N, 10**6):
        monkeypatch.setattr(graphsci, "EVAL_CHUNK_ROWS", rows)
        loss, z, z_exp = model.evaluate(Xm, Xraw, graph, valid_mask, eps=eps[2], **S.COEF)
        results[rows] = (loss, z.clone(), z_exp.clone())
    loss0, z0, zexp0 = results[N]
    assert math.isfinite(loss0) and zexp0.shape == (N, G)
    for rows, (loss, z, z_exp) in results.items():
        assert abs(loss - loss0) <= 1e-6 * abs(loss0), (rows, loss, loss0)
        assert rel_err(z, z0) < 1e-6 and rel_err(z_exp, zexp0) < 1e-6, rows


def test_fit_keeps_the_callers_matrix(cuda, schedule):
    """fit() drops its own reference to the unmasked matrix; the caller's tensor stays alive and unchanged."""
    schedule("lean")
    N, G = 4099, 1001
    Xm, Xraw, graph, train_mask, valid_mask, sf, eps = S._data(cuda, N, G, 1)
    del graph.ndata["feat"]
    X = Xraw.clone()
    X_before = X.clone()
    model = _model(N, G, "tf32x3", 0.1, 1, graph, sf)
    model.fit(X, Xraw, graph, mask=train_mask.cpu().numpy(), n_epochs=2, eps_sequence=[eps[i] for i in range(4)], **S.COEF)
    torch.cuda.synchronize()
    assert torch.equal(X, X_before)
    assert math.isfinite(model.train_loss) and math.isfinite(model.valid_loss)


# ---- configuration 3 at full size -----------------------------------------------------------------------------------------
def _config3_data(cuda, N, G):
    """benchmarks/configs.py::config3's inputs: counts, log1p, the gene graph from a 20 k-cell sample, Xᵀ as the GNN's node
    features, an all-ones mask and the size factors."""
    from dance_b200 import ops, synth
    from dance_b200.data import AnnDataLite, Data
    from dance_b200.transforms import FeatureFeatureGraph
    Xraw = synth.expression_counts(N, G, seed=1, density=0.10, device=cuda)
    X = Xraw.clone()
    ops.normalize_total_log1p_(X, normalize=False, log1p=True)
    sample = Data(AnnDataLite(X[:20000].cpu().numpy()))
    FeatureFeatureGraph(threshold=0.05, normalize_edges=True)(sample)
    graph = sample.data.uns["FeatureFeatureGraph"]
    graph.ndata["feat"] = X.t().contiguous()
    n_counts = Xraw.sum(1)
    sf = (n_counts / torch.median(n_counts)).contiguous()
    return X, Xraw, graph, sf


def _zinb_column_ref(pre3, gamma, beta, y, sf, mask, le, ke_col):
    """float64 restatement of one gene column of the fused training kernel: training-mode BatchNorm of each head, the
    activations, le·mean_mask(nll) + ke_col·0.5·mean_mask(mse) and its gradients by autograd."""
    x = pre3.double().requires_grad_()
    g = gamma.double().requires_grad_()
    b = beta.double().requires_grad_()
    h = torch.stack([F.batch_norm(x[k][:, None], None, None, g[k:k + 1], b[k:k + 1], True, 0.0, 1e-5)[:, 0] for k in range(3)])
    pi = torch.sigmoid(h[0])
    disp = torch.clamp(F.softplus(h[1]), 1e-4, 1e4)
    mean = torch.clamp(torch.exp(h[2]), 1e-5, 1e6)
    y, sf, m = y.double(), sf.double(), mask.bool()
    mu = mean * sf
    e = 1e-10
    nb = (torch.lgamma(disp + e) + torch.lgamma(y + 1) - torch.lgamma(y + disp + e) + (disp + y) * torch.log(1.0 + mu / (disp + e))
          + y * (torch.log(disp + e) - torch.log(mu + e)))
    zero = -torch.log(pi + (1 - pi) * torch.pow(disp / (disp + mu + e), disp) + e)
    nll = torch.where(y < 1e-8, zero, nb)[m]
    mse = ((mu - y)**2)[m]
    loss = le * nll.mean() + ke_col * 0.5 * mse.mean()
    dx, dg, db = torch.autograd.grad(loss, (x, g, b))
    return dict(nll=float(nll.detach().sum()), mse=float(mse.detach().sum()), cnt=int(m.sum()), dpre=dx, dgamma=dg, dbeta=db,
                mean=x.detach().mean(1), var=x.detach().var(1, unbiased=False))


def test_config3_full_size(cuda, schedule, monkeypatch):
    from dance_b200 import graphsci_ops
    schedule("auto")
    N, G = 500_000, 3000
    X, Xraw, graph, sf = _config3_data(cuda, N, G)
    tm = torch.ones(N, G, dtype=torch.uint8, device=cuda)
    model = _model(N, G, "bf16", 0.1, 0, graph, sf)
    assert model.schedule() == "lean"
    coef = dict(le=1, la=1e-9, ke=1e2, ka=1)

    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    for _ in range(2):
        loss = model.train(X, Xraw, graph, tm, tm, **coef)
        assert math.isfinite(loss) and math.isfinite(model.valid_loss)
    torch.cuda.synchronize()
    peak_train = torch.cuda.max_memory_allocated()
    print(f"\n500000 x 3000 lean: peak {peak_train / 2**30:.2f} GiB over two train() steps")
    assert peak_train < FULL_SIZE_PEAK, peak_train

    # the fused training kernel, called directly on the heads' pre-BatchNorm buffers of a third step, one sampled gene at a time
    gen = torch.Generator().manual_seed(3)
    genes = torch.randperm(G, generator=gen)[:8].tolist()
    checked = []
    real = graphsci_ops.heads_train

    def heads_train(pre, gamma, beta, mean, invstd, Y, size_factors, mask, le, ke, **kw):
        for j in genes:
            cols = [t[:, j:j + 1] for t in pre]
            pre3 = torch.stack([c[:, 0] for c in cols])
            ref = _zinb_column_ref(pre3, gamma[:, j], beta[:, j], Y[:, j], size_factors, mask[:, j], le, ke / G)
            # the batch statistics the kernel is handed
            assert ((mean[:, j].double() - ref["mean"]).abs() / ref["var"].sqrt()).max() < 1e-5, j
            assert ((invstd[:, j].double() * (ref["var"] + 1e-5).sqrt() - 1).abs()).max() < 1e-5, j
            vec = [t[:, j:j + 1].contiguous() for t in (gamma, beta, mean, invstd)]
            acc, dg, db = real(cols, *vec, Y[:, j:j + 1], size_factors, mask[:, j:j + 1], le, ke / G)
            acc = acc.cpu()
            assert int(acc[2]) == ref["cnt"] == N, j
            assert abs(float(acc[0]) - ref["nll"]) < 1e-5 * abs(ref["nll"]), (j, float(acc[0]), ref["nll"])
            assert abs(float(acc[1]) - ref["mse"]) < 1e-5 * abs(ref["mse"]), (j, float(acc[1]), ref["mse"])
            for what, got, want in (("dgamma", dg[:, 0], ref["dgamma"]), ("dbeta", db[:, 0], ref["dbeta"])):
                assert ((got.double() - want).abs() <= 1e-4 * want.abs() + 1e-6 * want.abs().max()).all(), (j, what, got, want)
            rows = torch.randint(0, N, (64, ), generator=gen).to(cuda)
            got = torch.stack([c[rows, 0] for c in cols]).double()
            want = ref["dpre"][:, rows]
            scale = ref["dpre"].abs().amax(1, keepdim=True)
            err = float(((got - want).abs() / scale).max())
            assert err < 1e-4, (j, err)
            checked.append(j)
        return real(pre, gamma, beta, mean, invstd, Y, size_factors, mask, le, ke, **kw)

    monkeypatch.setattr(graphsci_ops, "heads_train", heads_train)
    model.train(X, Xraw, graph, tm, tm, **coef)
    monkeypatch.setattr(graphsci_ops, "heads_train", real)
    assert checked == genes               # 8 genes × 64 sampled rows: 512 dpre entries

    # fit() at full size: the GNN features come from fit's masked matrix
    del graph.ndata["feat"], tm
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    model.fit(X, Xraw, graph, n_epochs=2, **coef)
    torch.cuda.synchronize()
    peak_fit = torch.cuda.max_memory_allocated()
    print(f"500000 x 3000 lean: peak {peak_fit / 2**30:.2f} GiB over fit(n_epochs=2)")
    assert math.isfinite(model.train_loss) and math.isfinite(model.valid_loss)
    assert peak_fit < FULL_SIZE_PEAK, peak_fit
