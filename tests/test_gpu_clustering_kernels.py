"""The clustering kernels element by element against the float64 restatements of tests/clustering_ref.py: SpaGCN's DEC head
(csrc/dec.cu) and scGNN's k-means step, regulariser weights, Cell-type loss and L1 term (csrc/em.cu).

Sizes that must cross a grid-stride cap ("past one wave") are derived from the device's SM count, so each case crosses its cap
on any H100.  Bounds are per element, in units of an error scale of the same element; each case prints its worst ratio to the
bound (≤ 1 passes)."""
import math

import numpy as np
import pytest
import torch

import clustering_ref as ref

pytestmark = pytest.mark.gpu

U = 2.0**-24                     # float32 unit roundoff


def _sms():
    from dance_b200 import ops
    return ops.device_info()[0]


def _ratio(err, bound):
    """max(err / bound) over the elements, with 0/0 = 0 and NaN kept."""
    err, bound = err.double(), torch.as_tensor(bound, dtype=torch.float64, device=err.device)
    return float(torch.where(err == 0, torch.zeros_like(err), err / bound).max())


def _report(name, ratios):
    print(f"\n{name}: " + ", ".join(f"{k} {v:.3g}" for k, v in ratios.items()))
    bad = {k: v for k, v in ratios.items() if not v <= 1.0}
    assert not bad, f"{name}: over the bound {bad}"


def _ulp(x):
    """The float32 spacing at |x|."""
    a = x.abs()
    return torch.nextafter(a, torch.full_like(a, float("inf"))) - a


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


# ---- DEC head -----------------------------------------------------------------------------------------------------------------
# dec_kl_grad runs at most 4·SMs blocks of 8 warps (16·SMs with the global-atomic dμ), dec_q / dec_target 16·SMs blocks; a warp
# takes one spot per turn.
N_DEC = {"1": lambda sm: 1, "31": lambda sm: 31, "wave+1": lambda sm: 4 * sm * 8 + 1, "big": lambda sm: max(50_000, 3 * 16 * sm * 8),
         "200k": lambda sm: 200_000}
KS, HS = (1, 2, 31, 32, 33, 64), (1, 31, 32, 50, 193, 256)
# K·h = 12 288 floats (48 KB) is the last shape with per-block shared-memory dμ partials; (64, 193) the first one without
DEC_SHAPES = ([(K, h, s) for s in ("1", "31", "wave+1", "big") for K in KS for h in HS]
              + [(K, h, s) for s in ("wave+1", "big") for K, h in ((64, 192), (64, 193), (48, 256), (33, 400))]
              + [(10, 50, "200k")])                                     # the configuration-5 size

P_TOL = 16 * U
LOSS_TOL = 1e-5


def _dec_tols(h, alpha):
    """(q, dz, dμ) bounds.  q's float32 error grows like (α + 1)·√h: d² sums h squared differences with one rounding each, and
    q = t^(α+1)/2 raises its error to the power α + 1.  A float32 emulation of dec_row_q at 50 688 spots and K = 64 reaches
    43·2⁻²⁴ at h = 256, α = 1 and 12.5·2⁻²⁴ at h = 50, α = 0.2, so 16·2⁻²⁴ holds only at small h; the bound is 16·2⁻²⁴ or
    4·(α + 1)·√(h + 2)·2⁻²⁴, whichever is larger (about 3× the emulated maximum)."""
    return max(16.0, 4 * (alpha + 1) * math.sqrt(h + 2)) * U, 2.0**-16, 2.0**-14


GAP = 1e-5


def _dec_data(n, K, h, seed):
    g = _gen(seed)
    mu = torch.randn((K, h), generator=g, device="cuda")
    lab = torch.randint(0, K, (n, ), generator=g, device="cuda")
    z = mu[lab] + 0.6 * torch.randn((n, h), generator=g, device="cuda")
    return z, mu


def _check_labels(labels, q64, gap):
    """The kernel's argmax of q: the float64 argmax wherever the top two float64 q differ by more than ``gap`` relative; inside
    that gap, a q within it."""
    top = q64.max(1).values
    chosen = q64.gather(1, labels.long().clamp(0, q64.shape[1] - 1)[:, None])[:, 0]
    assert bool(((labels >= 0) & (labels < q64.shape[1])).all())
    return _ratio(top - chosen, gap * top)


def _dec_check(name, r, h, alpha, q, p, q_out, dz, dmu, loss, labels):
    """Every DEC output against the float64 restatement ``r``; p against the target distribution of the kernel's own q and
    column sums (the operands b2_dec_target_f32 is given)."""
    from dance_b200 import ops
    assert torch.isfinite(dz).all() and torch.isfinite(dmu).all()
    assert torch.equal(q_out, q)
    p64 = q.double()**2 / ops.colsum(q).double()
    p64 /= p64.sum(1, keepdim=True)
    q_tol, dz_tol, dmu_tol = _dec_tols(h, alpha)
    # the warps' partial losses meet in float32 atomic adds, whose roundings add up like a random walk over the warps
    _report(name, {
        "q": _ratio((q.double() - r["q"]).abs(), q_tol * r["q"]),
        "p": _ratio((p.double() - p64).abs(), P_TOL * p64),
        "dz": _ratio((dz.double() - r["dz"]).abs(), dz_tol * r["scale_dz"]),
        "dmu": _ratio((dmu.double() - r["dmu"]).abs(), dmu_tol * r["scale_dmu"]),
        # plus 8·2⁻²⁴ absolute: log(p / (q + 1e-6)) of a ratio near 1 has an absolute error of a few ulp, which the |p·log|
        # terms (~1e-6 per row at K = 1, where p = q = 1) do not bound
        "loss": abs(float(loss) - r["loss"]) / (LOSS_TOL * r["loss_abs"] + 8 * U),
        "labels": _check_labels(labels, r["q"], GAP),
    })


@pytest.mark.parametrize("alpha", [0.2, 1.0])
@pytest.mark.parametrize("K,h,size", DEC_SHAPES, ids=[f"K{K}-h{h}-n{s}" for K, h, s in DEC_SHAPES])
def test_dec_head_against_float64(cuda, K, h, size, alpha):
    """q, p, loss, dz, dμ and the labels of dec_q / dec_target / dec_kl_grad.  Bounds (see _dec_tols): q relative, p 16·2⁻²⁴
    relative; dz and dμ in units of Σ c̄_ij |z_ic − μ_jc|, where c̄ is ∂L/∂d² with its one subtraction taken by magnitude —
    ∂L/∂u_j = (g_j − Σ g q)/S cancels where p ≈ q, and the float32 rounding of q enters g_j before that cancellation."""
    from dance_b200 import ops
    n = N_DEC[size](_sms())
    z, mu = _dec_data(n, K, h, seed=K * 1000 + h)
    q = ops.dec_q(z, mu, alpha)
    p = ops.dec_target(q)
    q_out = torch.full_like(q, float("nan"))
    dz = torch.full_like(z, float("nan"))
    labels = torch.full((n, ), -7, dtype=torch.int32, device=cuda)
    loss, dz, dmu = ops.dec_kl_grad(z, mu, p, alpha, dz=dz, q_out=q_out, labels_out=labels)
    r = ref.dec_reference(z, mu, p, alpha)
    _dec_check(f"dec n={n} K={K} h={h} alpha={alpha}", r, h, alpha, q, p, q_out, dz, dmu, loss, labels)


def _dec_pad(n, w, ld, like=None):
    """A [n, w] view of an [n, ld] NaN-filled buffer (holding ``like`` when given), and the buffer."""
    buf = torch.full((n, ld), float("nan"), device="cuda")
    if like is not None:
        buf[:, :w] = like
    return buf[:, :w], buf


@pytest.mark.parametrize("K,h,size", [(1, 1, "wave+1"), (33, 50, "big"), (64, 193, "big"), (31, 256, "wave+1")])
def test_dec_head_padded_operands(cuda, K, h, size):
    """Leading dimensions h + 3 for z, K + 5 for q, p and q_out, h + 7 for dz: the guard columns stay NaN, q and dz equal the
    contiguous call's bit for bit, and everything holds against float64."""
    from dance_b200 import ops
    n, alpha = N_DEC[size](_sms()), 0.2
    z0, mu = _dec_data(n, K, h, seed=7 + K + h)
    z, zb = _dec_pad(n, h, h + 3, z0)
    q, qb = _dec_pad(n, K, K + 5)
    p, pb = _dec_pad(n, K, K + 5)
    q_out, ob = _dec_pad(n, K, K + 5)
    dz, db = _dec_pad(n, h, h + 7)
    st = torch.cuda.current_stream().cuda_stream
    ops._call("b2_dec_q_f32", z.data_ptr(), h + 3, mu.data_ptr(), n, K, h, alpha, q.data_ptr(), K + 5, st)
    cs = ops.colsum(q)
    ops._call("b2_dec_target_f32", q.data_ptr(), K + 5, cs.data_ptr(), n, K, p.data_ptr(), K + 5, st)
    labels = torch.full((n, ), -7, dtype=torch.int32, device=cuda)
    loss, _, dmu = ops.dec_kl_grad(z, mu, p, alpha, dz=dz, q_out=q_out, labels_out=labels)
    for name, buf, w in (("z", zb, h), ("q", qb, K), ("p", pb, K), ("q_out", ob, K), ("dz", db, h)):
        assert bool(buf[:, w:].isnan().all()), f"{name}: a guard column was written"
    assert torch.equal(q, ops.dec_q(z0, mu, alpha))
    _, dz_c, _ = ops.dec_kl_grad(z0, mu, p.contiguous(), alpha)
    assert torch.equal(dz, dz_c)
    r = ref.dec_reference(z0, mu, p, alpha)
    _dec_check(f"dec padded n={n} K={K} h={h}", r, h, alpha, q, p, q_out, dz, dmu, loss, labels)


@pytest.mark.parametrize("K,pairs", [(31, [(3, 4), (29, 30)]), (33, [(3, 4), (0, 32)]), (64, [(3, 4), (5, 37), (6, 45), (62, 63)])],
                         ids=["K31", "K33", "K64"])
def test_dec_labels_exact_ties_take_the_lower_index(cuda, K, pairs):
    """μ_b = μ_a for each pair (a < b): every spot is drawn near μ_a, so its two largest q are bit-equal and the label must be a.
    The pairs put a and b on neighbouring lanes (j, j + 1), in one lane's two slots (j, j + 32) and on different lanes across
    the slots (j < 32, j' ≥ 32)."""
    from dance_b200 import ops
    n, h = N_DEC["big"](_sms()), 50
    g = _gen(K)
    mu = torch.randn((K, h), generator=g, device="cuda")
    for a, b in pairs:
        mu[b] = mu[a]
    lo = torch.tensor([a for a, _ in pairs], device="cuda")
    want = lo[torch.randint(0, len(pairs), (n, ), generator=g, device="cuda")]
    z = mu[want] + 0.3 * torch.randn((n, h), generator=g, device="cuda")
    p = ops.dec_target(ops.dec_q(z, mu, 0.2))
    labels = torch.full((n, ), -7, dtype=torch.int32, device=cuda)
    ops.dec_kl_grad(z, mu, p, 0.2, labels_out=labels)
    wrong = int((labels.long() != want).sum())
    print(f"\ndec ties n={n} K={K} pairs={pairs}: {wrong} labels not the lower index")
    assert wrong == 0


# ---- k-means, one Lloyd step --------------------------------------------------------------------------------------------------
# The assign kernel runs at most 16·SMs blocks of 256 threads, one point per thread per turn; k·d floats of centroids are staged
# in dynamic shared memory (above 48 KB through the per-device opt-in, up to 96 KB).
KM_CASES = {"1-1-1": lambda sm: (1, 1, 1), "100-3-7": lambda sm: (100, 3, 7),
            "wave": lambda sm: (max(600_000, 16 * sm * 256 * 10 // 9), 16, 64),
            "1M-16-64": lambda sm: (1_000_000, 16, 64),          # locality_order's shape in the benchmark
            "5000-200-64": lambda sm: (5000, 200, 64),           # 51 200 B of centroids: the opt-in path
            "3000-256-96": lambda sm: (3000, 256, 96)}           # exactly 96 KB


def _n_ties(n):
    return min(n // 10, 4000)


def _kmeans_data(n, d, k, pad, seed):
    """Integer centres C0 and points drawn around them, with ties: C0[k−1] = C0[1] (so cluster k−1 stays empty), C0[2] far from
    every point (empty too), C0[3] = C0[0] + 8·e0; some rows, the last one included, are integer points equidistant from 0 and 3
    (the midpoint) or from 1 and k−1."""
    g = _gen(seed)
    C0 = torch.randint(-16, 16, (k, d), generator=g, device="cuda").float()
    lab = torch.randint(0, k, (n, ), generator=g, device="cuda")
    if k >= 4:
        C0[k - 1] = C0[1]
        C0[2] = 1000.0
        C0[3] = C0[0]
        C0[3, 0] += 8.0
        lab[lab == 2] = 0
        lab[lab == k - 1] = 1
    X = C0[lab] + 0.7 * torch.randn((n, d), generator=g, device="cuda")
    if k >= 4:
        m = _n_ties(n)
        rows = torch.cat([torch.randperm(n, generator=g, device="cuda")[:m - 1], torch.tensor([n - 1], device="cuda")])
        mid = C0[0].clone()
        mid[0] += 4.0
        off = torch.randint(-1, 2, (m, d), generator=g, device="cuda").float()
        X[rows] = torch.where(torch.arange(m, device="cuda")[:, None] % 2 == 0, mid.expand(m, d), C0[1] + off)
    buf = torch.full((n, d + pad), float("nan"), device="cuda")
    buf[:, :d] = X
    return buf[:, :d], C0


def _kmeans_step(X, C, labels, stats, update):
    from dance_b200 import ops
    n, d = X.shape
    k = C.shape[0]
    ws = torch.empty(ops.lib().b2_kmeans_workspace_bytes(k, d), dtype=torch.uint8, device="cuda")
    ops._call("b2_kmeans_step_f32", X.data_ptr(), X.stride(0), n, d, C.data_ptr(), k, labels.data_ptr(), int(update), stats.data_ptr(),
              ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("pad", [0, 5], ids=["ldx=d", "ldx=d+5"])
@pytest.mark.parametrize("case", list(KM_CASES))
def test_kmeans_step_against_float64(cuda, case, pad):
    """One b2_kmeans_step_f32: labels by the near-tie rule, exact ties to the lowest index, each new centre within 1 ulp of the
    float32 of the float64 mean of the points the kernel assigned to it, empty clusters and update = 0 leaving centres bit for
    bit, inertia and ‖ΔC‖² within 1e-6, and the changed count exact."""
    n, d, k = KM_CASES[case](_sms())
    X, C0 = _kmeans_data(n, d, k, pad, seed=n + d + k)
    g = _gen(1)
    prev = torch.randint(0, k, (n, ), generator=g, device="cuda", dtype=torch.int32)
    labels, C = prev.clone(), C0.clone()
    stats = torch.full((3, ), float("nan"), dtype=torch.float64, device="cuda")
    _kmeans_step(X, C, labels, stats, update=True)
    D = ref.sq_dist(X, C0)
    best, second, first = ref.nearest_two(D)
    lab = labels.long()
    assert bool(((lab >= 0) & (lab < k)).all())
    tie = second == best
    if k >= 4:
        assert int(tie.sum()) >= _n_ties(n) // 2, "the constructed ties are missing"
    tie_wrong = int((lab[tie] != first[tie]).sum())
    new64, counts = ref.lloyd_update(X, C0, lab)
    empty = counts == 0
    if k >= 4:
        assert bool(empty[2]) and bool(empty[k - 1])
    assert torch.equal(C[empty].view(torch.int32), C0[empty].view(torch.int32)), "an empty cluster's centre moved"
    want = torch.where(empty[:, None], C0, new64.float())
    inertia, shift2, changed = ref.lloyd_stats(D, lab, prev, C0, C)       # ‖ΔC‖² of the centres the kernel wrote
    chosen = D.gather(1, lab[:, None])[:, 0]
    gap = GAP
    ratios = {"labels": _ratio(chosen - best, gap * best), "centres (ulp)": _ratio((C - want).abs(), _ulp(want)),
              "inertia": abs(stats[0].item() - inertia) / (1e-6 * inertia) if inertia else abs(stats[0].item()),
              "shift": abs(stats[1].item() - shift2) / (1e-6 * shift2) if shift2 else abs(stats[1].item())}
    print(f"\nkmeans n={n} d={d} k={k} ldx={X.stride(0)}: {int(tie.sum())} exact ties, {tie_wrong} not to the lowest index, "
          f"{int(((second - best) <= gap * best).sum())} near ties")
    assert tie_wrong == 0
    assert stats[2].item() == changed
    _report(f"kmeans n={n} d={d} k={k} ldx={X.stride(0)}", ratios)
    # update = 0: labels only, the centres untouched bit for bit
    C1 = C.clone()
    prev1 = labels.clone()
    _kmeans_step(X, C, labels, stats, update=False)
    assert torch.equal(C.view(torch.int32), C1.view(torch.int32))
    assert stats[1].item() == 0.0 and stats[2].item() == int((labels != prev1).sum())


def test_kmeans_loop_matches_float64_lloyd(cuda):
    """ops.kmeans with tol = 0 against a float64 Lloyd loop from the same C0: the same iteration count and the same labels.  The
    data are chosen so that no point of any iteration comes within 1e-4 (relative) of a second centre in float64."""
    from dance_b200 import ops
    rng = np.random.default_rng(14)
    n, d, k = 5000, 8, 16
    cen = rng.normal(scale=3.0, size=(k, d))
    X = (cen[rng.integers(0, k, n)] + rng.normal(size=(n, d))).astype(np.float32)
    C0 = X[rng.permutation(n)[:k]].copy()
    want, it_ref, min_gap = ref.lloyd_loop(torch.from_numpy(X).cuda(), torch.from_numpy(C0).cuda())
    assert min_gap > 1e-4 and it_ref > 3
    labels, inertia, it = ops.kmeans(torch.from_numpy(X).cuda(), torch.from_numpy(C0).cuda(), max_iter=300, tol=0.0)
    print(f"\nkmeans loop: {it} iterations (float64: {it_ref}), smallest float64 gap {min_gap:.3g}")
    assert it == it_ref
    assert torch.equal(labels.long(), want)



# ---- scGNN regulariser weights, Cell-type loss, L1 ----------------------------------------------------------------------------
def _n_regu():
    return max(600_000, 16 * _sms() * 256 * 10 // 9)          # past 16·SMs blocks of 256 threads


def _regu_graph(n, n_clusters, weighted, seed):
    """Random CSR rows of 0..8 entries: zero-degree rows, rows holding only their self-loop, self-loops in some rows only, rows
    of weight 0 (weighted), and labels of −1 and n_clusters besides the clusters."""
    rng = np.random.default_rng(seed)
    deg = rng.integers(0, 9, n)
    deg[rng.random(n) < 0.05] = 0
    rowptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(deg, out=rowptr[1:])
    rows = np.repeat(np.arange(n), deg)
    colidx = rng.integers(0, n, rowptr[-1])
    first = rowptr[:-1][deg > 0]
    loop = first[rng.random(len(first)) < 0.3]
    colidx[loop] = rows[loop]                                  # self-loops in some rows; a 1-entry row of them has degree 0
    vals = rng.uniform(0.1, 2.0, rowptr[-1])
    vals[np.isin(rows, np.nonzero(rng.random(n) < 0.03)[0])] = 0.0
    labels = rng.integers(-1, n_clusters + 1, n)
    return rowptr.astype(np.int32), colidx.astype(np.int32), vals, labels.astype(np.int32)


@pytest.mark.parametrize("weighted", [False, True], ids=["degree", "weighted"])
def test_regulariser_weights_against_float64(cuda, weighted):
    from dance_b200 import ops
    n, n_clusters = _n_regu(), 12
    rowptr, colidx, vals, labels = _regu_graph(n, n_clusters, weighted, seed=5 + weighted)
    t = lambda a: torch.from_numpy(a).cuda()
    if weighted:
        w = ops.graph_regu_weights_weighted(t(rowptr), t(colidx), t(vals), t(labels), n_clusters)
        w64 = ref.regu_weights_weighted(rowptr, colidx, vals, labels, n_clusters)
    else:
        w = ops.graph_regu_weights(ops.CSR(t(rowptr), t(colidx), None, (n, n)), t(labels), n_clusters)
        w64 = ref.regu_weights(rowptr, colidx, labels, n_clusters)
    want = torch.from_numpy(w64).cuda().float()
    zero = want == 0
    assert int(zero.sum()) > 0.05 * n and int((~zero).sum()) > 0.5 * n
    assert bool((w[zero] == 0).all())
    _report(f"regulariser weights n={n} {'weighted' if weighted else 'degree'}", {"w (ulp)": _ratio((w - want).abs(), _ulp(want))})


@pytest.mark.parametrize("relu_mask", [True, False], ids=["relu", "no-relu"])
@pytest.mark.parametrize("zero_dropout", [False, True], ids=["dropout", "zero-dropout"])
def test_celltype_loss_grad_against_float64(cuda, relu_mask, zero_dropout):
    """2 000 × 2 001 with cols_orig = 1 990 (past one wave of the grid-stride loop); an all-zero x_dropout makes the norm 0."""
    from dance_b200 import ops
    rows, cols, co = 2000, 2001, 1990
    g = _gen(3)
    recon = torch.relu(torch.randn((rows, cols), generator=g, device="cuda"))
    recon[:, ::7] = -torch.rand((rows, (cols + 6) // 7), generator=g, device="cuda")   # negatives for the mask
    target = torch.randn((rows, cols), generator=g, device="cuda")
    xd = torch.randn((rows, co), generator=g, device="cuda") * (torch.rand((rows, co), generator=g, device="cuda") < 0.4)
    if zero_dropout:
        xd.zero_()
    roww = torch.rand(rows, generator=g, device="cuda") + 0.1
    loss64, grad64, scale = ref.celltype_loss_grad(recon, target, xd, roww, relu_mask)
    v0 = float(np.float32(loss64 / 4))                          # what loss_out holds before: losing it is far outside the bound
    loss_out = torch.full((1, ), v0, device="cuda")
    loss, grad = ops.celltype_loss_grad(recon, target, xd, roww, relu_mask=relu_mask, loss_out=loss_out)
    assert torch.isfinite(grad).all()
    if relu_mask:
        assert bool((grad[recon <= 0] == 0).all())
    _report(f"celltype relu={relu_mask} zero_dropout={zero_dropout}",
            {"grad": _ratio((grad.double() - grad64).abs(), 8 * U * scale),
             "loss": abs(loss.item() - v0 - loss64) / (1e-6 * (v0 + loss64))})


def test_l1_grad_add_against_float32(cuda):
    """grad + coef·sign(p) bit for bit, sign 0 at +0 and −0; l1_out accumulates coef·Σ|p| onto what it holds."""
    from dance_b200 import ops
    n = 5 * 16 * _sms() * 256 + 1
    g = _gen(4)
    p = torch.randn(n, generator=g, device="cuda")
    p[::5] = 0.0
    p[1::5] = -0.0
    grad = torch.randn(n, generator=g, device="cuda")
    grad[::11] = -0.0
    want, l1 = ref.l1_grad_add(p, grad.clone(), 0.37)
    v0 = float(np.float32(l1 / 4))                             # what l1_out holds before: losing it is far outside the bound
    l1_out = torch.full((1, ), v0, device="cuda")
    ops.l1_grad_add(p, grad, 0.37, l1_out)
    assert torch.equal(grad.view(torch.int32), want.view(torch.int32))
    first = l1_out.item()
    ops.l1_grad_add(p, grad, 0.37, l1_out)
    # one float32 atomic add per warp partial: the sum's rounding error is at most (number of warps)·2⁻²⁴ of the total
    # one float32 atomic add per warp partial, 16·SMs·8 of them: their roundings walk like √(warps)·2⁻²⁴ of the total; 4× that
    # still fails on one lost partial (1/(16·SMs·8) of the sum)
    tol = 4 * math.sqrt(16 * _sms() * 8) * U
    _report(f"l1 n={n}", {"l1": abs(first - v0 - l1) / (tol * (v0 + l1)), "l1 twice": abs(l1_out.item() - v0 - 2 * l1) / (tol * (v0 + 2 * l1))})
