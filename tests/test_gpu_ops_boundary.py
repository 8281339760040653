"""Every ops wrapper refuses a malformed tensor before it launches anything.

One table case per wrapper: a valid small call, then, for each tensor the caller supplies, a copy of the same arguments with that
tensor replaced by a bad variant: the wrong dtype, one row (or element) short, and a non-unit inner stride.  Operands whose
extent defines the problem size get no short variant, since a shorter one is a smaller valid problem.  Every bad call must raise
B2Error, launch no kernel and leave every tensor of the call, the caller's sentinel-filled outputs included, as it was."""
import pytest
import torch

from dance_b200 import ops
from dance_b200._lib import B2Error

SENTINEL = 7.0
_WRONG = {torch.float32: torch.float64, torch.float64: torch.float32, torch.int32: torch.int64, torch.int64: torch.int32,
          torch.uint8: torch.int32, torch.bfloat16: torch.float16}


def _graph(dev, n=6, vals=True):
    """A ring with self loops: row i holds columns i and i + 1 (mod n)."""
    cols = torch.tensor([[i, (i + 1) % n] for i in range(n)], dtype=torch.int32).sort(1).values.reshape(-1)
    return ops.CSR(torch.arange(0, 2 * n + 1, 2, dtype=torch.int32, device=dev), cols.to(dev),
                   torch.rand(2 * n, device=dev) if vals else None, (n, n))


def _cases():
    """{label: (wrapper, builder)}; builder(dev) → (kwargs, fixed, free): ``fixed`` tensors have an extent implied by the other
    arguments, ``free`` ones define it.  Tensors named in neither are outputs the wrapper allocates or CSR parts."""
    def r(*s, dev, dtype=torch.float32):
        return torch.rand(*s, device=dev).to(dtype)

    def o(*s, dev, dtype=torch.float32):                   # a caller-supplied output, filled with the sentinel
        return torch.full(s, SENTINEL, device=dev).to(dtype)

    def knn_idx(n, k, dev, self_first=False):
        idx = torch.tensor([[(i + j + (0 if self_first else 1)) % n for j in range(k)] for i in range(n)], dtype=torch.int32)
        return idx.to(dev)

    C = {}

    def case(label, fn=None):
        def deco(builder):
            C[label] = (fn or label, builder)
            return builder
        return deco

    @case("to_x16")
    def _(d): return dict(X=r(5, 8, dev=d), out=o(5, 8, dev=d, dtype=torch.bfloat16)), ["out"], ["X"]

    @case("spmm")
    def _(d): return dict(A=_graph(d), X=r(6, 8, dev=d), out=o(6, 8, dev=d), bias=r(8, dev=d)), ["X", "out", "bias"], []

    @case("spmm_bf16", "spmm")
    def _(d): return (dict(A=_graph(d), X=r(6, 8, dev=d, dtype=torch.bfloat16), out=o(6, 8, dev=d),
                           out16=o(6, 8, dev=d, dtype=torch.bfloat16)), ["X", "out", "out16"], [])

    @case("csr_transpose")
    def _(d): return dict(A=_graph(d)), [], []

    @case("gemm")
    def _(d): return (dict(A=r(8, 4, dev=d), B=r(4, 8, dev=d), out=o(8, 8, dev=d), bias=r(8, dev=d), mask=r(8, 8, dev=d)),
                      ["B", "out", "bias", "mask"], ["A"])

    @case("colsum")
    def _(d): return dict(X=r(8, 4, dev=d), out=o(4, dev=d)), ["out"], ["X"]

    @case("mse_sum_loss_grad")
    def _(d): return (dict(recon=r(4, 4, dev=d), target=r(4, 4, dev=d), ltmg_regu=r(4, 4, dev=d), grad=o(4, 4, dev=d),
                           loss_out=o(1, dev=d)), ["target", "ltmg_regu", "grad", "loss_out"], ["recon"])

    def gae(d, sym):
        kw = dict(z=r(6, 8, dev=d), labels=_graph(d, vals=False), norm=1.0, pos_weight=2.0, mu=r(6, 8, dev=d), logvar=r(6, 8, dev=d),
                  dmu=o(6, 8, dev=d), dlogvar=o(6, 8, dev=d), loss=o(1, dev=d))
        kw.update(dict(sb_begin=0, sb_end=1, dz_full=o(6, 8, dev=d)) if sym else dict(dz=o(6, 8, dev=d)))
        return kw, ["mu", "logvar", "dmu", "dlogvar", "loss", "dz_full" if sym else "dz"], ["z"]

    case("gae_loss_grad")(lambda d: gae(d, False))
    case("gae_loss_grad_sym")(lambda d: gae(d, True))

    @case("adam_step")
    def _(d): return (dict(param=r(10, dev=d), grad=r(10, dev=d), exp_avg=r(10, dev=d), exp_avg_sq=r(10, dev=d), step=1),
                      ["grad", "exp_avg", "exp_avg_sq"], ["param"])

    @case("reparam_fwd")
    def _(d): return (dict(mu=r(6, 8, dev=d), logvar=r(6, 8, dev=d), eps=r(6, 8, dev=d), out=o(6, 8, dev=d)),
                      ["logvar", "eps", "out"], ["mu"])

    @case("reparam_bwd")
    def _(d): return (dict(dz=r(6, 8, dev=d), logvar=r(6, 8, dev=d), eps=r(6, 8, dev=d), dmu=o(6, 8, dev=d), dlogvar=o(6, 8, dev=d)),
                      ["logvar", "eps", "dmu", "dlogvar"], ["dz"])

    @case("knn")
    def _(d): return dict(X=r(8, 4, dev=d), k=2), [], ["X"]

    @case("pairwise_l2_dense")
    def _(d): return dict(X=r(8, 4, dev=d)), [], ["X"]

    @case("knn_graph_build")
    def _(d): return dict(knn_idx=knn_idx(6, 2, d)), [], ["knn_idx"]

    @case("knn_graph_weighted_build")
    def _(d): return dict(knn_idx=knn_idx(6, 2, d), knn_dist=r(6, 2, dev=d, dtype=torch.float64)), ["knn_dist"], ["knn_idx"]

    @case("normalize_total_log1p_")
    def _(d): return dict(X=r(5, 4, dev=d), target_sum=10.0), [], ["X"]

    @case("dropout")
    def _(d): return dict(x=r(5, 4, dev=d), p=0.5, seed=1, key=2, out=o(5, 4, dev=d)), ["out"], ["x"]

    @case("gat_scores")
    def _(d): return dict(H=r(6, 8, dev=d), a_src=r(8, dev=d), a_trg=r(8, dev=d), nheads=2), ["a_src", "a_trg"], ["H"]

    @case("gat_aggregate_fwd")
    def _(d): return (dict(T=_graph(d, vals=False), H=r(6, 8, dev=d), s_src=r(6, 2, dev=d), s_trg=r(6, 2, dev=d), nheads=2,
                           out=o(6, 8, dev=d)), ["H", "s_src", "s_trg", "out"], [])

    @case("gat_aggregate_bwd")
    def _(d):
        T = _graph(d, vals=False)
        Tt, perm = ops.csr_transpose(T)
        H, a = r(6, 8, dev=d), r(8, dev=d)
        s, t = ops.gat_scores(H, a, a, 2)
        _, alpha, gmax = ops.gat_aggregate_fwd(T, H, s, t, 2)
        return (dict(T=T, Tt=Tt, t_perm=perm, H=H, a_src=a, a_trg=a.clone(), s_src=s, s_trg=t, alpha=alpha, dOut=r(6, 8, dev=d), nheads=2,
                     gmax=gmax), ["t_perm", "H", "a_src", "a_trg", "s_src", "s_trg", "alpha", "dOut", "gmax"], [])

    @case("gat_combine_fwd")
    def _(d): return dict(agg=r(6, 8, dev=d), skip=r(6, 8, dev=d), bias=r(8, dev=d), nheads=2, concat=True), ["skip", "bias"], ["agg"]

    @case("gat_combine_bwd")
    def _(d): return (dict(dout=r(6, 8, dev=d), out=r(6, 8, dev=d), nheads=2, F=4, concat=True, dpre=o(6, 8, dev=d)),
                      ["out", "dpre"], ["dout"])

    @case("cellgene_graph")
    def _(d): return dict(X=r(5, 4, dev=d)), [], ["X"]

    @case("sage_edge_values")
    def _(d): return dict(T=_graph(d), w=r(12, dev=d), alpha=r(4, dev=d), n_genes=2), ["w", "alpha"], []

    @case("softmax_ce_sum")
    def _(d): return (dict(logits=r(5, 3, dev=d), labels=torch.tensor([0, 1, 2, 1, 0], device=d), dlogits=o(5, 3, dev=d),
                           loss_out=o(1, dev=d)), ["labels", "dlogits", "loss_out"], ["logits"])

    @case("sym_eig")
    def _(d):
        x = r(4, 4, dev=d)
        return dict(Cm=x + x.t()), [], ["Cm"]

    @case("pca")
    def _(d): return dict(X=r(8, 4, dev=d), n_components=2), [], ["X"]

    @case("dec_q")
    def _(d): return dict(z=r(6, 4, dev=d), mu=r(3, 4, dev=d)), [], ["z", "mu"]

    @case("dec_target")
    def _(d): return dict(q=r(6, 3, dev=d)), [], ["q"]

    @case("dec_kl_grad")
    def _(d): return (dict(z=r(6, 4, dev=d), mu=r(3, 4, dev=d), p=r(6, 3, dev=d), dz=o(6, 4, dev=d), dmu=o(3, 4, dev=d), loss=o(1, dev=d),
                           q_out=o(6, 3, dev=d), labels_out=o(6, dev=d, dtype=torch.int32)),
                      ["p", "dz", "dmu", "loss", "q_out", "labels_out"], ["z", "mu"])

    @case("sgd_momentum_step")
    def _(d): return dict(param=r(10, dev=d), grad=r(10, dev=d), buf=r(10, dev=d), step=1, lr=0.1), ["grad", "buf"], ["param"]

    @case("exp_adj")
    def _(d): return dict(D=r(4, 4, dev=d), l=1.0, want_sum=True), [], ["D"]

    @case("clip_grad_norm_")
    def _(d): return dict(grad=r(10, dev=d), max_norm=1.0, norm_out=o(1, dev=d)), ["norm_out"], ["grad"]

    @case("radius_graph")
    def _(d): return dict(X=r(6, 2, dev=d, dtype=torch.float64), radius=0.5), [], ["X"]

    @case("matrix_normalize")
    def _(d): return dict(X=r(5, 4, dev=d), out=o(5, 4, dev=d)), ["out"], ["X"]

    @case("pearson_corr")
    def _(d): return dict(X=r(6, 4, dev=d)), [], ["X"]

    @case("threshold_graph")
    def _(d): return dict(adj=r(4, 4, dev=d), threshold=0.5), [], ["adj"]

    @case("umap_connectivities")
    def _(d):
        dist = torch.sort(r(6, 3, dev=d), 1).values
        dist[:, 0] = 0
        return dict(knn_idx=knn_idx(6, 3, d, self_first=True), knn_dist=dist), ["knn_dist"], ["knn_idx"]

    @case("batchnorm_fwd")
    def _(d): return (dict(X=r(6, 4, dev=d), gamma=r(4, dev=d), beta=r(4, dev=d), running_mean=r(4, dev=d), running_var=r(4, dev=d),
                           training=True), ["gamma", "beta", "running_mean", "running_var"], ["X"])

    @case("batchnorm_bwd")
    def _(d): return (dict(dY=r(6, 4, dev=d), Y=r(6, 4, dev=d), X=r(6, 4, dev=d), gamma=r(4, dev=d), save_mean=r(4, dev=d),
                           save_invstd=r(4, dev=d), act="relu", dgamma=o(4, dev=d), dbeta=o(4, dev=d)),
                      ["dY", "Y", "gamma", "save_mean", "save_invstd", "dgamma", "dbeta"], ["X"])

    @case("zinb_loss_grad")
    def _(d): return (dict(a_pi=r(4, 5, dev=d), b_disp=r(4, 5, dev=d), c_mean=r(4, 5, dev=d), Y=r(4, 5, dev=d), size_factors=r(4, dev=d),
                           mask=torch.ones(4, 5, dtype=torch.uint8, device=d)), ["b_disp", "c_mean", "Y", "size_factors", "mask"], ["a_pi"])

    @case("adj_sample")
    def _(d): return dict(mu=r(16, dev=d), log_std=r(16, dev=d), eps=r(16, dev=d)), ["log_std", "eps"], ["mu"]

    @case("adj_loss_grad")
    def _(d): return (dict(z=r(4, 4, dev=d), mu=r(4, 4, dev=d), log_std=r(4, 4, dev=d), target=r(4, 4, dev=d), class_weight=r(4, dev=d)),
                      ["mu", "log_std", "target", "class_weight"], ["z"])

    @case("adj_reparam_bwd")
    def _(d): return (dict(dz=r(16, dev=d), mu=r(16, dev=d), log_std=r(16, dev=d), eps=r(16, dev=d), coef_kl=1.0),
                      ["dz", "log_std", "eps"], ["mu"])

    @case("kmeans")
    def _(d): return dict(X=r(8, 4, dev=d), centers=r(2, 4, dev=d), max_iter=2), [], ["X", "centers"]

    @case("graph_regu_weights")
    def _(d): return dict(A=_graph(d), labels=torch.tensor([0, 1] * 3, dtype=torch.int32, device=d), n_clusters=2), ["labels"], []

    @case("graph_regu_weights_weighted")
    def _(d):
        A = _graph(d)
        return (dict(rowptr=A.rowptr, colidx=A.colidx, vals=A.vals.double(), labels=torch.tensor([0, 1] * 3, dtype=torch.int32, device=d),
                     n_clusters=2), ["vals", "labels"], ["rowptr", "colidx"])

    @case("celltype_loss_grad")
    def _(d): return (dict(recon=r(5, 4, dev=d), target=r(5, 4, dev=d), x_dropout=r(5, 4, dev=d), row_weight=r(5, dev=d),
                           grad=o(5, 4, dev=d), loss_out=o(1, dev=d)), ["target", "x_dropout", "row_weight", "grad", "loss_out"], ["recon"])

    @case("l1_grad_add")
    def _(d): return dict(param=r(10, dev=d), grad=r(10, dev=d), l1_out=o(1, dev=d)), ["grad", "l1_out"], ["param"]

    @case("gene_stats")
    def _(d): return dict(X=r(5, 4, dev=d)), [], ["X"]

    @case("cell_stats")
    def _(d): return dict(X=r(5, 4, dev=d)), [], ["X"]

    @case("subset")
    def _(d): return (dict(X=r(5, 4, dev=d), rows=torch.tensor([4, 0, 2], device=d), cols=torch.tensor([3, 1], dtype=torch.int32, device=d)),
                      [], ["X", "rows", "cols"])

    @case("cellwise_mask")
    def _(d): return dict(X=r(5, 8, dev=d), min_gene_counts=1), [], ["X"]

    @case("locality_order")
    def _(d): return dict(X=r(8, 4, dev=d), n_anchors=2), [], ["X"]

    @case("quantiles")
    def _(d): return dict(base=r(5, 4, dev=d), qs=(0.1, 0.9)), [], ["base"]

    @case("col_minmax")
    def _(d): return dict(x=r(5, 4, dev=d), nonfinite=o(1, dev=d, dtype=torch.float64)), ["nonfinite"], ["x"]

    @case("concat_normalized")
    def _(d): return dict(left=r(5, 4, dev=d), right=r(5, 3, dev=d)), ["right"], ["left"]

    @case("act")
    def _(d): return dict(x=r(5, 4, dev=d), act="gelu", out=o(5, 4, dev=d)), ["out"], ["x"]

    @case("act_bwd")
    def _(d): return dict(dy=r(5, 4, dev=d), act="relu", y=r(5, 4, dev=d), out=o(5, 4, dev=d)), ["y", "out"], ["dy"]

    @case("graphsc_block_degrees")
    def _(d): return (dict(A=_graph(d), dst=torch.tensor([1, 4, -1], dtype=torch.int32, device=d), outdeg=o(6, dev=d, dtype=torch.int32)),
                      ["outdeg"], ["dst"])

    def block(d, transposed):
        A, dst = _graph(d), torch.tensor([1, 4, -1], dtype=torch.int32, device=d)
        deg = ops.graphsc_block_degrees(A, dst)
        x, out = (r(3, 4, dev=d), o(6, 4, dev=d)) if transposed else (r(6, 4, dev=d), o(3, 4, dev=d))
        return dict(A=A, dst=dst, outdeg=deg, x=x, transposed=transposed, out=out), ["outdeg", "x", "out"], ["dst"]

    case("graphsc_block_aggregate")(lambda d: block(d, False))
    case("graphsc_block_aggregate_transposed", "graphsc_block_aggregate")(lambda d: block(d, True))

    @case("graphsc_batch_decoder")
    def _(d): return dict(z=r(4, 4, dev=d), dz=o(4, 4, dev=d), loss=o(1, dev=d)), ["dz", "loss"], ["z"]

    @case("graphsc_scatter_rows")
    def _(d): return (dict(x=r(3, 4, dev=d), idx=torch.tensor([5, 0, 2], dtype=torch.int32, device=d), out=o(6, 4, dev=d)),
                      ["idx"], ["x", "out"])
    return C


CASES = _cases()


def bad_variants(kw, fixed, free):
    """(label, kwargs) for every bad variant of every caller-supplied tensor."""
    for name in fixed + free:
        t = kw[name]
        vs = [("dtype", t.to(_WRONG[t.dtype]))]
        if name in fixed:
            vs.append(("short", t[:-1]))
        if t.numel() > 1:
            wide = torch.zeros(*t.shape[:-1], 2 * t.shape[-1], dtype=t.dtype, device=t.device)
            wide[..., ::2] = t
            vs.append(("stride", wide[..., ::2]))
        for label, v in vs:
            yield f"{name}:{label}", {**kw, name: v}


def test_every_wrapper_has_a_case():
    from test_ops_boundary import CASES as CPU_CASES
    assert {fn for fn, _ in CASES.values()} == set(CPU_CASES)


@pytest.mark.gpu
@pytest.mark.parametrize("label", sorted(CASES))
def test_wrapper_refuses_bad_tensors_before_launching(cuda, label):
    fn, builder = CASES[label]
    kw, _, _ = builder(cuda)
    getattr(ops, fn)(**kw)                                  # the valid call runs
    torch.cuda.synchronize()
    n_bad = 0
    for what, bad in bad_variants(*builder(cuda)):
        tensors = {k: v.clone() for k, v in bad.items() if isinstance(v, torch.Tensor)}
        before = ops.counters()["launches"]
        with pytest.raises(B2Error):
            getattr(ops, fn)(**bad)
        assert ops.counters()["launches"] == before, what
        torch.cuda.synchronize()
        for k, v in tensors.items():
            assert torch.equal(bad[k], v), f"{what}: {k} was written"
        n_bad += 1
    kw, fixed, free = builder(cuda)
    assert n_bad == sum(2 + (k in fixed) - (kw[k].numel() <= 1) for k in fixed + free)


@pytest.mark.gpu
def test_csr_checks_its_extents(cuda):
    rp, ci = torch.tensor([0, 1, 2], dtype=torch.int32, device=cuda), torch.tensor([0, 1], dtype=torch.int32, device=cuda)
    ops.CSR(rp, ci, torch.ones(2, device=cuda), (2, 2))
    with pytest.raises(B2Error, match="rowptr"):
        ops.CSR(rp, ci, None, (3, 3))
    with pytest.raises(B2Error, match="vals"):
        ops.CSR(rp, ci, torch.ones(3, device=cuda), (2, 2))
    with pytest.raises(B2Error, match="colidx"):
        ops.CSR(rp, ci.long(), None, (2, 2))
