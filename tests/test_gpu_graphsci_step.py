"""The GraphSCI training epoch (BASELINE configuration 3) against the float64 restatement in oracle/graphsci_step_ref.py, at
the configuration's gene count, with dropout and in every GEMM precision.

The fixture tests (tests/test_gpu_graphsci.py, 260 cells × 48 genes, dropout 0) never reach the paths the benchmarked epoch
runs: tensor-core GEMMs, split-K over the cell axis, the adjacency-loss row loop striding over more than 256 columns,
BatchNorm over many row chunks with a ragged last column tile (3 000 = 93·32 + 24), and, with dropout > 0, the unshared
backward of the two dec_mean calls (masks m2a / m2b) and the masking at each of the ten dropout sites.  Each case runs two
consecutive ``train()`` calls on synthetic data built as benchmarks/configs.py::config3 builds it, with real train / valid
masks, captures the keep-masks the module drew, and for each step restates that step in float64 from the module's own
weights and running statistics before it, so that errors do not compound.  Compared: the five losses, every gradient
(norm-wise, worst row and worst column), the running statistics, z_exp of the eval forward and, after both steps, the
weights against float64 Adam (weight decay 1e-5) applied to the module's own gradients.  bf16 is compared with the
restatement whose products round their operands to bf16 (tests/bf16_ref.py).

The loss weights make every term move the gradients it feeds (the benchmark's la = 1e-9 would leave the adjacency
cross-entropy invisible); the first step asserts each term's share from the restatement.
"""
import json
import os

import pytest
import torch

from bf16_ref import Bf16MatMul
from conftest import rel_err
from oracle import graphsci_step_ref as R

pytestmark = pytest.mark.gpu

COEF = dict(le=1.0, la=5e-7, ke=5e-3, ka=10.0)
LR, WD = 1e-3, 1e-5

# Upper bounds, 4-6x the largest error measured over seeds 0-2 of every case on an H100 80 GB HBM3 at a 700 W power limit
# (GRAPHSCI_STEP_REPORT below writes the measurements of a run).  "grad" are the weight gradients (norm-wise, "_row" / "_col"
# the worst row / column, see row_rel_err), "zero_grad" the biases in front of a BatchNorm (exact gradient 0) in units of the
# largest gradient of the step, "run" the BatchNorm running statistics, "zexp" the eval forward's reconstruction, "adam" the
# optimiser's move over both steps and "adam_max" its worst element in units of lr.
# Measured worst (fp32 / tf32x3 / bf16): loss 6.9e-7 / 2.3e-5 / 1.5e-2 (kl, a difference of near-equal terms); gradients
# 1.4e-3 / 4.5e-3 / 1.2e-1 norm-wise, worst row 1.1e-2 / 2.7e-1, worst column 5.6e-2 / 5.1e-1; zero gradients 8.5e-8 / 1.8e-7 /
# 7.8e-8; running statistics 2.0e-7 / 4.2e-5 / 8.2e-5; z_exp 6.8e-7 / 5.2e-5 / 7.8e-3, worst row 1.4e-6 / 6.6e-5 / 1.8e-2;
# Adam 9.7e-7 norm-wise and 1.2e-4 lr in the worst element in every precision.
# Yardstick: float32 torch autograd (cuBLAS, TF32 off) on the same inputs lands from float64 at most 8.3e-4 norm-wise, 5.4e-2 in
# the worst row and 4.8e-2 in the worst column of a gradient (3.4e-2 at 1 001 genes, in the same dec_mean weight column where
# fp32 measures 5.6e-2), 1.9e-6 on z_exp and 9.8e-6 on a loss.  Worst rows and columns are ill-conditioned at initialisation:
# signed sums over the cells that cancel.
# tf32x3 at 3 000 genes lands 10-40x further than float32 torch on z_exp, the first BatchNorm's statistics and the GNN
# gradients.  test_tf32x3_gemm_on_epoch_operands below traces this to the single products with K = 3 000 or 20 012: on the
# epoch's own operands the tensor-core tf32x3 GEMM is 7-11x further from float64 than the CUDA-core fp32 kernel (z·Wfᵀ 7.3e-6
# against 9.8e-7, X_d·zf 3.2e-6 against 2.8e-7, the split-K products 9.0e-6 against 8.3e-7).  The operand split accounts for
# little of that norm-wise: products of the split operands (hi = x & 0xFFFFE000, lo cut to tf32), summed in float64, land
# 2.0e-7 / 1.4e-7 from float64 on the same two products; the rest arises in the wgmma fp32 accumulation over K.  The split
# does bias every operand toward zero by up to 2^-21, and its worst gradient column (conv2, 5.1e-1) is where that shows most:
# a round-to-nearest split measured 9.8e-2 there, but it moves the kernel's results off what other tests pin and slows the
# scGNN step by about 3 %, so it is left for its own change.  At 1 001 genes those products run on the CUDA cores and tf32x3
# matches fp32.  The tf32x3 bounds below cover this measured GEMM error; the single-GEMM test bounds it directly.
TOL = {
    "fp32": dict(loss=3.5e-6, grad=7e-3, grad_row=5e-2, grad_col=2.5e-1, zero_grad=5e-7, run=1e-6, zexp=3.5e-6, zexp_row=7e-6,
                 adam=5e-6, adam_max=6e-4),
    # tf32x3 worst row / column: 0.9, below the 1.0 of a row or column that is entirely wrong or zero (3.4x / 1.8x the measured)
    "tf32x3": dict(loss=1.2e-4, grad=2.5e-2, grad_row=9e-1, grad_col=9e-1, zero_grad=1e-6, run=2e-4, zexp=2.5e-4, zexp_row=3.5e-4,
                   adam=5e-6, adam_max=6e-4),
    # bf16: gradients norm-wise only (a worst row / column of a bf16 gradient is off by more than its own size); "closer" bounds
    # the ratio of the distances to the rounded and to the unrounded restatement (measured at most 0.13)
    "bf16": dict(loss=8e-2, grad=6e-1, zero_grad=4e-7, run=4e-4, zexp=4e-2, zexp_row=9e-2, adam=5e-6, adam_max=6e-4, closer=0.5),
}
# a tf32x3 product on the epoch's operands, relative error against float64 norm-wise and in the worst row (measured at most
# 9.0e-6 and 1.1e-5)
GEMM_TOL = dict(norm=5e-5, row=6e-5)
SHARE = 5e-3        # each loss term carries at least this share of the gradient norm of a parameter it feeds

MEASURED = []       # (case, quantity, error): every comparison made, for setting the bounds above
# GRAPHSCI_STEP_REPORT=<file.json>: also measure float32 torch autograd against float64 on the same inputs (the yardstick
# quoted above) and write every entry of MEASURED to that file when the module's tests end.
REPORT = os.environ.get("GRAPHSCI_STEP_REPORT")


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if REPORT:
        with open(REPORT, "w") as f:
            json.dump(MEASURED, f)


def _check(case, what, err, tol):
    MEASURED.append((case, what, float(err)))
    assert err < tol, f"{case}: {what} error {err:.3g} exceeds {tol:.3g}"


def row_rel_err(a, ref):
    """Worst row of ‖a_i − ref_i‖ / ‖ref_i‖.  Rows whose reference norm is below 1e-3 of the RMS row norm are measured against
    that floor instead, so that a near-zero row does not turn rounding into a large ratio."""
    a = torch.as_tensor(a).double()
    ref = torch.as_tensor(ref).double().to(a.device)
    a, ref = a.reshape(a.shape[0], -1), ref.reshape(ref.shape[0], -1)
    den = ref.norm(dim=1)
    floor = 1e-3 * float(den.pow(2).mean().sqrt())
    return float(((a - ref).norm(dim=1) / den.clamp(min=max(floor, 1e-300))).max())


def _views(params, flat):
    """The named parameters of a FlatParams, as views into a copy `flat` of its flat buffer."""
    base = params.flat.storage_offset()
    return {k: flat[v.storage_offset() - base:v.storage_offset() - base + v.numel()].view(v.shape) for k, v in params.p.items()}


def _data(cuda, N, G, seed):
    """configs.py::config3's data at N × G: synthetic counts, log1p, the gene graph from a cell sample; then, as GraphSCI.fit
    does, a random 90 % entry mask, the first 90 % of the cells for training and the masked matrix as the GNN's features."""
    from dance_b200 import ops, synth
    from dance_b200.data import AnnDataLite, Data
    from dance_b200.transforms import FeatureFeatureGraph
    Xraw = synth.expression_counts(N, G, seed=seed + 1, density=0.10, device=cuda)
    X = Xraw.clone()
    ops.normalize_total_log1p_(X, normalize=False, log1p=True)
    sample = Data(AnnDataLite(X[:20000].cpu().numpy()))
    FeatureFeatureGraph(threshold=0.05, normalize_edges=True)(sample)
    graph = sample.data.uns["FeatureFeatureGraph"]
    gen = torch.Generator(device=cuda).manual_seed(seed)
    mask = torch.rand(N, G, device=cuda, generator=gen) < 0.9
    rows = (torch.arange(N, device=cuda) < int(0.9 * N))[:, None]
    train_mask, valid_mask = mask & rows, ~mask & rows
    Xm = (X * mask).contiguous()
    graph.ndata["feat"] = Xm.t().contiguous()
    n_counts = Xraw.sum(1)
    sf = (n_counts / torch.median(n_counts)).contiguous()
    eps = torch.randn(4, G, G, device=cuda, generator=gen)          # train / eval noise of two steps
    return Xm, Xraw, graph, train_mask, valid_mask, sf, eps


def _on_tensor_cores(A, B, M, N, K, precision):
    """The dispatch rule of b2_gemm_f32 (csrc/gemm.cu, gemm_tc.cu): tensor cores unless 'fp32' is asked for, K < 8,
    M·N·K < 2^18, or an operand's base / row pitch is not 16-byte aligned."""
    return (precision != "fp32" and K >= 8 and M * N * K >= (1 << 18) and A.stride(0) % 4 == 0 and B.stride(0) % 4 == 0
            and A.data_ptr() % 16 == 0 and B.data_ptr() % 16 == 0)


def _masks(gc, ac):
    """The keep-masks of one training forward, keyed by restatement site (None where nothing was dropped)."""
    m = {"feat": gc["m0"], "h1": gc["m1"], "h2_mean": gc["m2a"], "h2_log_std": None if gc["shared"] else gc["m2b"], "X": ac["mx"],
         "enc.1": ac["e1"]["m"], "enc.5": ac["e2"]["m"]}
    m.update({h: ac["heads"][h]["m"] for h in R.HEADS})
    return {k: v for k, v in m.items() if v is not None}


def _compare(case, name, got, ref, tol, kind, gmax=None):
    if gmax is not None and float(ref.abs().max()) < 1e-9 * gmax:
        # a bias in front of a BatchNorm: its exact gradient is zero, any evaluation holds rounding noise
        _check(case, name + " abs", float(got.abs().max()) / gmax, tol["zero_grad"])
        return
    _check(case, name, rel_err(got, ref), tol[kind])
    if got.dim() == 2 and kind + "_row" in tol:
        _check(case, name + " rows", row_rel_err(got, ref), tol[kind + "_row"])
        if kind == "grad":
            _check(case, name + " cols", row_rel_err(got.t(), ref.t()), tol[kind + "_col"])


def _compare_step(case, model, ref, grads, z_exp, tol):
    for k in ("loss_adj", "loss_exp", "kl", "train_loss", "valid_loss"):
        want = ref["losses"][k]
        _check(case, k, abs(getattr(model, k) - want) / abs(want), tol["loss"])
    gmax = max(float(v.abs().max()) for v in ref["grads"].values())
    for k in R.PARAMS:
        _compare(case, "d " + k, grads[k], ref["grads"][k], tol, "grad", gmax)
    for k, (rm, rv) in ref["running"].items():
        _check(case, f"running_mean {k}", rel_err(model.bn[k].running_mean, rm), tol["run"])
        _check(case, f"running_var {k}", rel_err(model.bn[k].running_var, rv), tol["run"])
    _compare(case, "z_exp", z_exp, ref["z_exp"], tol, "zexp")


def _bf16_outputs(model, z_exp, ref, plain):
    # loss_exp, train_loss and z_exp are left out: there the kernel sat as close to the unrounded restatement as to the rounded
    # one (ratios up to 2.7), the bf16 rounding moving them less than operands that land one bf16 ulp apart near a rounding
    # boundary (float64 activations in the restatement, float32 in the kernel)
    for k in ("loss_adj", "valid_loss"):
        yield k, getattr(model, k), ref["losses"][k], plain["losses"][k]
    for k in R.BN_KEYS:
        yield f"running_mean {k}", model.bn[k].running_mean, ref["running"][k][0], plain["running"][k][0]
        yield f"running_var {k}", model.bn[k].running_var, ref["running"][k][1], plain["running"][k][1]


def graphsci_case(cuda, N, G, precision, dropout, seed, monkeypatch, report_f32=False):
    from dance_b200 import ops
    from dance_b200.modules.graphsci import GraphSCI
    case = f"graphsci {N}x{G} {precision} dropout={dropout} seed={seed}"
    tol = TOL[precision]
    Xm, Xraw, graph, train_mask, valid_mask, sf, eps = _data(cuda, N, G, seed)
    assert G > 256 and G % 32 != 0            # adjacency-loss row loop strides; ragged BatchNorm column tile
    model = GraphSCI(num_cells=N, num_genes=G, dataset="synthetic", dropout=dropout, gpu=0, seed=seed, precision=precision)
    model._bind_graph(graph)
    model.size_factors = sf
    model.lr, model.weight_decay = LR, WD
    gene_graph = R.GeneGraph(*graph.edges(), G, cuda)

    cap = {}
    real_gnn, real_ae, real_eval = model._gnn_forward, model._ae_forward, model.evaluate

    def gnn_forward(feat, training, eps=None):
        out = real_gnn(feat, training, eps)
        if training:
            cap["gnn"] = out[3]
        return out

    def ae_forward(X, z, training):
        out = real_ae(X, z, training)
        if training:
            cap["ae"] = out[3]
        return out

    def evaluate(*a, **kw):
        out = real_eval(*a, **kw)
        cap["z_exp"] = out[2]
        return out

    model._gnn_forward, model._ae_forward, model.evaluate = gnn_forward, ae_forward, evaluate
    calls = []
    real_gemm = ops.gemm

    def recording_gemm(A, B, *, transA=False, transB=False, precision=None, **kw):
        M, K = (A.shape[1], A.shape[0]) if transA else A.shape
        n_out = B.shape[0] if transB else B.shape[1]
        calls.append((precision, M, n_out, K, int(transA), int(transB), _on_tensor_cores(A, B, M, n_out, K, precision)))
        return real_gemm(A, B, transA=transA, transB=transB, precision=precision, **kw)

    monkeypatch.setattr(ops, "gemm", recording_gemm)
    tm, vm = train_mask.view(torch.uint8), valid_mask.view(torch.uint8)
    flat_start = model.params.flat.clone()
    step_grads = []
    for step in range(2):
        at = f"{case} step {step + 1}"
        flat0 = model.params.flat.clone()
        run0 = {k: (b.running_mean.clone(), b.running_var.clone()) for k, b in model.bn.items()}
        calls.clear()
        model.train(Xm, Xraw, graph, tm, vm, eps_train=eps[2 * step], eps_eval=eps[2 * step + 1], **COEF)
        torch.cuda.synchronize()
        grads = _views(model.params, model.params.grad.clone())
        step_grads.append(model.params.grad.clone())
        gc, ac, z_exp = cap.pop("gnn"), cap.pop("ae"), cap.pop("z_exp")
        masks = _masks(gc, ac)
        # the branches this case exists for
        assert gc["shared"] is (dropout == 0.0)
        assert len(masks) == (10 if dropout > 0 else 0)
        assert calls and all(c[0] == precision for c in calls), sorted({c[0] for c in calls})
        on_tc = [c[6] for c in calls]
        if precision == "fp32":
            assert not any(on_tc)
        elif G % 4 == 0:
            assert all(on_tc), [c[1:4] for c in calls if not c[6]]
        else:
            assert any(on_tc) and not all(on_tc)          # G-pitched operands on the CUDA cores, the rest on the tensor cores
        if precision != "fp32":
            # the weight-gradient products over the cell axis with a narrow output split K
            long_k = [c for c in calls if c[3] == N and c[4] and c[6] and min(c[1], c[2]) <= 256]
            assert len(long_k) >= (5 if G % 4 == 0 else 1), long_k
            for c in long_k:
                assert ops.lib().b2_gemm_workspace_bytes(c[1], c[2], c[3], c[4], c[5], ops.PREC[precision]) > 0, c
        del gc, ac

        params0 = _views(model.params, flat0)
        args = (params0, run0, Xm, Xraw, sf, gene_graph, train_mask, valid_mask)
        kw = dict(eps_train=eps[2 * step], eps_eval=eps[2 * step + 1], masks=masks, **COEF)
        if precision == "bf16":
            ref = R.train_step(*args, mm=Bf16MatMul.apply, **kw)
            _compare_step(at, model, ref, grads, z_exp, tol)
            if step == 0:
                # a kernel that rounds its operands to bf16 sits clearly closer to the rounded restatement than to the unrounded
                # one on the well-conditioned outputs of the step (the kl loss is a difference of near-equal terms: left out)
                plain = R.train_step(*args, **kw)
                for what, got, near_ref, far_ref in _bf16_outputs(model, z_exp, ref, plain):
                    near, far = rel_err(got, near_ref), rel_err(got, far_ref)
                    MEASURED.append((at, f"bf16 {what} rounded / unrounded", near / far))
                    assert near < tol["closer"] * far, (what, near, far)
                del plain
        else:
            ref = R.train_step(*args, term_grads=(step == 0), **kw)
            _compare_step(at, model, ref, grads, z_exp, tol)
            if step == 0:
                # every loss term moves the gradients it feeds: the GNN's through z, the AE's through the ZINB and MSE terms
                for k, terms in (("gnnmodel.dec_mean.weight", ("exp", "adj", "kl_adj", "kl_exp")),
                                 ("aemodel.mul_layer.fc_layer.weight", ("exp", "kl_exp"))):
                    total = float(ref["grads"][k].norm())
                    for t in terms:
                        share = float(ref["term_grads"][t][k].norm()) / total
                        MEASURED.append((at, f"share {t} in d {k}", share))
                        assert share > SHARE, (k, t, share)
            if report_f32:
                f32 = R.train_step(*args, dtype=torch.float32, **kw)
                gmax = max(float(v.abs().max()) for v in ref["grads"].values())
                for k in R.PARAMS:
                    if float(ref["grads"][k].abs().max()) >= 1e-9 * gmax:
                        MEASURED.append((at, f"f32 torch d {k}", rel_err(f32["grads"][k], ref["grads"][k])))
                        if f32["grads"][k].dim() == 2:
                            MEASURED.append((at, f"f32 torch d {k} rows", row_rel_err(f32["grads"][k], ref["grads"][k])))
                            MEASURED.append((at, f"f32 torch d {k} cols", row_rel_err(f32["grads"][k].t(), ref["grads"][k].t())))
                MEASURED.append((at, "f32 torch z_exp", rel_err(f32["z_exp"], ref["z_exp"])))
                for k in ("loss_adj", "loss_exp", "kl", "train_loss", "valid_loss"):
                    MEASURED.append((at, f"f32 torch {k}", abs(f32["losses"][k] - ref["losses"][k]) / abs(ref["losses"][k])))
                del f32
        del ref, masks, grads, z_exp
    assert model.params.step == 2

    # Adam over both steps: float64 torch.optim.Adam with the module's weight decay, fed the module's own gradients
    p = flat_start.double().clone().requires_grad_()
    opt = torch.optim.Adam([p], lr=LR, weight_decay=WD)
    for g in step_grads:
        p.grad = g.double()
        opt.step()
    moved, want = model.params.flat.double() - flat_start.double(), p.detach() - flat_start.double()
    _check(case, "adam update", rel_err(moved, want), tol["adam"])
    _check(case, "adam update max/lr", float((moved - want).abs().max()) / LR, tol["adam_max"])


@pytest.mark.parametrize("precision,dropout", [("tf32x3", 0.0), ("tf32x3", 0.1), ("bf16", 0.0), ("bf16", 0.1)])
def test_graphsci_epoch_config3_genes(cuda, monkeypatch, precision, dropout):
    """20 012 cells × 3 000 genes (configuration 3's gene count): every GEMM on the tensor cores (the cell count is a multiple
    of 4, so the GNN's [G, N] features qualify as they do at the benchmark's 200 000 cells), split-K products over the cells,
    the adjacency row loop at 12 strides of 256, a ragged BatchNorm column tile."""
    graphsci_case(cuda, 20012, 3000, precision, dropout, seed=0, monkeypatch=monkeypatch, report_f32=bool(REPORT) and precision != "bf16")


@pytest.mark.parametrize("precision", ["fp32", "tf32x3"])
def test_graphsci_epoch_unaligned_genes(cuda, monkeypatch, precision):
    """4 099 cells × 1 001 genes: the products on G-pitched operands fall back to the CUDA cores (row pitch not a multiple of
    16 bytes) while the others stay on the tensor cores, so one epoch mixes both GEMM paths."""
    graphsci_case(cuda, 4099, 1001, precision, 0.1, seed=1, monkeypatch=monkeypatch, report_f32=bool(REPORT))


def test_tf32x3_gemm_on_epoch_operands(cuda):
    """The epoch's own tensor-core products, one GEMM at a time, against float64 and against the CUDA-core fp32 kernel:
    zf = z·Wfᵀ and X_d·zf (K = G = 3 000), and the split-K products over the 20 012 cells (the conv1 forward and a weight-
    gradient shaped Xᵀ·D).  These products carry the tf32x3 epoch's distance from float64 (see the bounds above): each is
    bounded against float64 directly, and the fp32 kernel's error on the same product is recorded beside it."""
    from dance_b200 import ops
    from dance_b200.modules.graphsci import GraphSCI
    N, G = 20012, 3000
    Xm, Xraw, graph, train_mask, valid_mask, sf, eps = _data(cuda, N, G, 0)
    model = GraphSCI(num_cells=N, num_genes=G, dataset="synthetic", dropout=0.1, gpu=0, seed=0, precision="tf32x3")
    model._bind_graph(graph)
    with torch.no_grad():
        z, _, _, gc = model._gnn_forward(model._graph_feat(graph), True, eps[0])
    P = model.params.p
    Wf, W1 = P["aemodel.mul_layer.fc_layer.weight"], P["gnnmodel.conv1.weight"]
    zf = ops.gemm(z, Wf, transB=True, precision="fp32")
    D = torch.randn(N, 256, device=cuda, generator=torch.Generator(device=cuda).manual_seed(1))
    cases = [("z·Wfᵀ", z, Wf, dict(transB=True), z.double() @ Wf.double().t()),
             ("X_d·zf", Xm, zf, {}, Xm.double() @ zf.double()),
             ("f_d·W1 (split-K)", gc["f_d"], W1, {}, gc["f_d"].double() @ W1.double()),
             ("Xᵀ·D (split-K)", Xm, D, dict(transA=True), Xm.double().t() @ D.double())]
    for name, A, B, kw, want in cases:
        M, K = (A.shape[1], A.shape[0]) if kw.get("transA") else A.shape
        n_out = B.shape[0] if kw.get("transB") else B.shape[1]
        assert _on_tensor_cores(A, B, M, n_out, K, "tf32x3"), name
        if K == N:
            assert ops.lib().b2_gemm_workspace_bytes(M, n_out, K, int(bool(kw.get("transA"))), int(bool(kw.get("transB"))),
                                                     ops.PREC["tf32x3"]) > 0, name
        tc = ops.gemm(A, B, precision="tf32x3", **kw)
        simt = ops.gemm(A, B, precision="fp32", **kw)
        for what, err in ((name, lambda x: rel_err(x, want)), (name + " rows", lambda x: row_rel_err(x, want))):
            e_tc, e_simt = err(tc), err(simt)
            MEASURED.append(("gemm tf32x3", what, e_tc))
            MEASURED.append(("gemm fp32", what, e_simt))
            assert e_tc < GEMM_TOL["row" if what.endswith(" rows") else "norm"], (what, e_tc, e_simt)
