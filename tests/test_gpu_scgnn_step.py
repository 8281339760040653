"""The scGNN training step that bench.py times, against the float64 restatement in oracle/scgnn_step_ref.py.

bench.py times one Feature-AE epoch (batch 12 800, LTMG loss with the all-zero TRS, Adam) and one Graph-AE GCN step (128-d input,
k = 15 kNN graph, EMB = 16).  At those sizes the engines take branches that the golden fixtures (160 × 32, 300 nodes) never
reach: split-K weight-gradient GEMMs, BN = 128 output tiles with a ragged last tile, the two-stage column sum of the bias
gradients, the tensor-core decoder fed mu / logvar as column slices of the packed [n, 2·EMB] buffer.  Each case below runs one
whole engine step on synthetic seeded data at such a size, asserts that the branch was taken, and compares the loss, the
activations, every gradient (norm-wise and as the worst row- or column-relative error, so that one wrong tile or split is not
averaged away) and the weights after the optimiser step.

The optimiser check applies float64 torch.optim.Adam to the GPU's OWN gradients: on its first step Adam moves every weight by
about lr·sign(g), so against the reference gradients every element whose |g| is near the gradient error could flip sign.
"""
import pytest
import torch

from conftest import rel_err
from oracle import scgnn_step_ref as R
from step_compare import adam_reference, param_views, row_rel_err

pytestmark = pytest.mark.gpu

PRECISIONS = ["fp32", "tf32x3"]
BATCH, K_NN, EMB = 12800, 15, 16        # bench.py

# Upper bounds, 4-6x the largest error measured over seeds 0-2 of every case on an H100 80 GB HBM3 at a 400 W power limit.
# "act" are activations, "dact" the gradients of the Graph-AE's z / mu / logvar, "grad" the weight gradients; "_row" / "_col" bound the
# worst row / column of a matrix (see row_rel_err); "adam_max" the worst element of the optimiser's move,
# in units of lr.  The Feature-AE gradient bounds are looser than 1e-4 because these gradients are ill-conditioned at
# initialisation (signed sums over 12 800 rows and 2 000 genes that cancel), not because of the kernels: float32 torch autograd
# (cuBLAS, TF32 off) on the same batches is off from the float64 reference by up to 6.0e-5 norm-wise, 1.2e-2 in the worst row and
# 3.1e-3 in the worst column of a weight gradient, against 1.0e-4, 2.1e-2 and 2.0e-3 for the engine in tf32x3 and 5.7e-5, 1.1e-2
# and 1.1e-3 in fp32.  Likewise the Graph-AE's worst gc1 gradient column (7.5e-5, tf32x3 with the CUDA-core decoder).
TOL = {
    ("fae", "fp32"): dict(loss=5e-6, act=2e-6, act_row=3e-6, grad=3e-4, grad_row=5e-2, grad_col=5e-3, adam=3e-6, adam_max=4e-5),
    ("fae", "tf32x3"): dict(loss=5e-6, act=2e-5, act_row=3e-5, grad=5e-4, grad_row=1e-1, grad_col=1e-2, adam=3e-6, adam_max=4e-5),
    ("gae", "fp32"): dict(loss=1e-6, act=3e-7, act_row=3e-6, dact=3e-6, dact_row=2e-5, dact_col=4e-6, grad=3e-5, grad_row=5e-5,
                          grad_col=5e-5, adam=2e-6, adam_max=1e-5),
    ("gae", "tf32x3"): dict(loss=3e-6, act=5e-6, act_row=2e-5, dact=2e-5, dact_row=1e-4, dact_col=3e-5, grad=5e-5, grad_row=1e-4,
                            grad_col=3e-4, adam=2e-6, adam_max=1e-5),
}

MEASURED = []        # (case, quantity, error): every comparison made, for setting the bounds above


def _check(case, what, err, tol):
    MEASURED.append((case, what, float(err)))
    assert err < tol, f"{case}: {what} error {err:.3g} exceeds {tol:.3g}"


def _compare(case, what, got, ref, tol, kind):
    """Norm-wise error; for a matrix also the worst row, and for a gradient matrix the worst column.  A 1-D bias gradient is
    compared norm-wise only: each element is one column sum over the batch, and for near-cancelling sums the per-element error
    of any float32 evaluation is of order 1e-2."""
    _check(case, what, rel_err(got, ref), tol[kind])
    if got.dim() == 2:
        _check(case, what + " rows", row_rel_err(got, ref), tol[kind + "_row"])
        if kind in ("grad", "dact"):
            _check(case, what + " cols", row_rel_err(got.t(), torch.as_tensor(ref).t()), tol[kind + "_col"])


def _check_adam(case, flat0, flat1, grads, lr, tol):
    """The optimiser's move of every weight, against float64 Adam on the same gradients: norm-wise, and worst element in units
    of lr (each step moves a weight by at most about lr)."""
    ref = adam_reference(flat0, grads, lr)
    moved, want = flat1.double() - flat0.double(), ref - flat0.double()
    _check(case, "adam update", rel_err(moved, want), tol["adam"])
    _check(case, "adam update max/lr", float((moved - want).abs().max()) / lr, tol["adam_max"])


def _gemm_ws(M, N, K, precision):
    from dance_b200 import ops
    return int(ops.lib().b2_gemm_workspace_bytes(M, N, K, 1, 0, ops.PREC[precision]))


def _assert_split_k(shapes, precision):
    """Weight-gradient GEMMs (transA, K = rows): split-K in tf32x3.  fp32 runs the CUDA-core kernel, which never splits."""
    for M, N, K in shapes:
        ws = _gemm_ws(M, N, K, precision)
        assert (ws > 0) if precision == "tf32x3" else (ws == 0), (M, N, K, precision, ws)


# ---------------------------------------------------------------------------------------------------------------- Feature-AE
def feature_ae_case(cuda, n_rows, genes, precision, seed):
    from dance_b200 import ops, synth
    from dance_b200.engine import FeatureAEEngine
    from dance_b200.parallel import batch_schedule
    case = f"fae n={n_rows} genes={genes} {precision} seed={seed}"
    tol = TOL[("fae", precision)]
    X = synth.expression_counts(n_rows, genes, seed=seed, density=0.10, device=cuda)
    ops.normalize_total_log1p_(X, target_sum=1e4, max_fraction=1.0)
    batches = batch_schedule(n_rows, BATCH)
    # the branches of the benchmarked step
    H, E = FeatureAEEngine.HID, FeatureAEEngine.EMB
    for b0, b1 in batches:
        B = b1 - b0
        tc_shapes = [(E, H, B), (H, E, B)]                               # fc2, fc3 weight gradients
        if genes % 4 == 0:
            tc_shapes += [(genes, H, B), (H, genes, B)]                   # fc4, fc1
        _assert_split_k(tc_shapes, precision)
        for N in (genes, H, E):
            assert ops.lib().b2_colsum_workspace_bytes(B, N) > 0, (B, N)    # two-stage bias-gradient column sum
    if genes % 4:
        assert X.stride(0) % 4 != 0          # row pitch not a multiple of 16 B: the GEMMs reading x / dr run on the CUDA cores

    eng = FeatureAEEngine(genes, device=cuda, lr=1e-3, precision=precision, seed=seed)
    steps = []                               # (weights before the step, gradients of the step)
    eng.grad_hook = lambda g: steps.append((eng.params.flat.clone(), g.clone()))
    z_all = torch.empty(n_rows, E, device=cuda)
    r_all = torch.empty_like(X)
    loss = eng.train_epoch(X, BATCH, "LTMG", 0.9, None, z_all, r_all).item()
    assert len(steps) == len(batches)
    ref_loss = 0.0
    for (b0, b1), (flat, grad) in zip(batches, steps):
        ref = R.feature_ae_step(X[b0:b1], param_views(eng.params, flat), "LTMG", 0.9, None)
        ref_loss += ref["loss"].item()
        at = f"{case} rows {b0}:{b1}"
        _compare(at, "z", z_all[b0:b1], ref["z"], tol, "act")
        _compare(at, "recon", r_all[b0:b1], ref["recon"], tol, "act")
        g = param_views(eng.params, grad)
        for k in R.FEATURE_AE_PARAMS:
            _compare(at, f"d {k}", g[k], ref["grads"][k], tol, "grad")
    for k, v in param_views(eng.params, steps[-1][1]).items():
        assert torch.equal(eng.params.g[k], v), k          # params.g still holds the last batch's gradients after Adam
    _check(case, "loss", abs(loss - ref_loss) / abs(ref_loss), tol["loss"])
    _check_adam(case, steps[0][0], eng.params.flat, [g for _, g in steps], eng.lr, tol)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_feature_ae_full_batch(cuda, precision):
    """One full 12 800 × 2 000 batch: split-K weight gradients, BN = 128 output tiles (2 000 = 15·128 + 80), split column sums."""
    feature_ae_case(cuda, BATCH, 2000, precision, seed=0)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_feature_ae_epoch_with_ragged_batch(cuda, precision):
    """train_epoch over 15 801 rows: a full batch, then a ragged 3 001-row batch with its own buffers and split plans."""
    feature_ae_case(cuda, 15801, 2000, precision, seed=1)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_feature_ae_unaligned_gene_count(cuda, precision):
    """1 999 genes: the GEMMs reading x, dr or the recon gradient fall back to the CUDA-core kernel (row pitch not a multiple
    of 16 bytes), the others stay on the tensor cores; the mixed step must be just as exact."""
    feature_ae_case(cuda, BATCH, 1999, precision, seed=2)


# ---------------------------------------------------------------------------------------------------------------- Graph-AE
def graph_ae_case(cuda, n, precision, seed, eps_zero=False, path="auto"):
    from dance_b200 import ops
    from dance_b200.engine import GraphAEEngine
    case = f"gae n={n} {precision} path={path}{' eps=0' if eps_zero else ''} seed={seed}"
    tol = TOL[("gae", precision)]
    gen = torch.Generator(device=cuda).manual_seed(seed)
    centres = torch.randn(10, 128, device=cuda, generator=gen) * 3
    lab = torch.randint(0, 10, (n, ), device=cuda, generator=gen)
    # a clustered, non-negative (ReLU-like) embedding, scaled so that the logits and logvar stay out of saturation
    x = ((torch.randn(n, 128, device=cuda, generator=gen) + centres[lab]).abs() * 0.1).contiguous()
    idx, _ = ops.knn(x, K_NN, return_dist=False)
    A = ops.knn_graph_build(idx)
    labels = ops.CSR(A.rowptr, A.colidx, None, A.shape)
    adj_sum = A.nnz - n                                   # bench.py
    pos_weight = float(n * n - adj_sum) / adj_sum
    norm = n * n / float((n * n - adj_sum) * 2)
    eps = torch.zeros(n, EMB, device=cuda) if eps_zero else torch.randn(n, EMB, device=cuda, generator=gen)

    H = GraphAEEngine.HID
    _assert_split_k([(H, 2 * EMB, n), (128, H, n)], precision)      # gc23, gc1 weight gradients (K = n)
    eng = GraphAEEngine(128, EMB, device=cuda, lr=1e-2, precision=precision, seed=seed)
    w0, flat0 = eng.state_dict(), eng.params.flat.clone()
    ops.set_path("gae", path)
    try:
        if path == "auto":
            assert ops.get_path("gae") == "auto" and n * n >= (1 << 22)    # the tensor-core decoder
        z, mu, logvar = eng.train_step(x, A, labels, norm, pos_weight, eps)
    finally:
        ops.set_path("gae", "auto")
    ref = R.graph_ae_step(x, A.rowptr, A.colidx, A.vals, A.rowptr, A.colidx, norm, pos_weight, w0, eps)

    _check(case, "loss", abs(eng.loss.item() - ref["loss"]) / abs(ref["loss"]), tol["loss"])
    for name, got in (("z", z), ("mu", mu), ("logvar", logvar)):
        _compare(case, name, got, ref[name], tol, "act")
    b = eng._buffers(n)
    _compare(case, "dz", b["dz"], ref["dz"], tol, "dact")
    _compare(case, "dmu", b["dml"][:, :EMB], ref["dmu"], tol, "dact")
    _compare(case, "dlogvar", b["dml"][:, EMB:], ref["dlogvar"], tol, "dact")
    for k, g in eng.grads().items():
        _compare(case, f"d {k}", g, ref["grads"][k], tol, "grad")
    _check_adam(case, flat0, eng.params.flat, [eng.params.grad], eng.lr, tol)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("n,eps_zero", [(2049, False), (2049, True), (20011, False), (131_001, False)])
def test_graph_ae_step(cuda, n, eps_zero, precision):
    """n = 2 049: just above the tensor-core decoder threshold, a ragged last 128-row block; with eps = 0, z = mu and the logvar
    gradient is the KLD term alone, the one case where that term is checked at full relative precision.  n = 20 011 and
    131 001: long-K split weight gradients."""
    graph_ae_case(cuda, n, precision, seed=0, eps_zero=eps_zero)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_graph_ae_step_cuda_core_decoder(cuda, precision):
    """The same step with the CUDA-core decoder selected, so the engine is checked with both decoders."""
    graph_ae_case(cuda, 20011, precision, seed=1, path="cuda")
