"""The GAT kernels (dance_b200/csrc/gat.cu) called directly through ``ops.gat_*`` against the fp64 restatement in
oracle/gat_ref.py: scores, the fused edge softmax + aggregate (wide- and narrow-head paths, global / per-target shift,
LeakyReLU / sigmoid scores), the plain and tied backward, and the combine kernels.

Errors are measured per row as well as globally: a Frobenius norm over 40 000 rows does not see one wrong hub row or one
wrong empty row.  ``row_err`` = max over rows of ‖Δrow‖ / max(‖ref row‖, floor · rms row norm of ref).

Tolerances are about 10x the largest error measured on an H100 80 GB HBM3 (400 W limit): forward 1.1e-7 global / 7.8e-6 per
row, gradients 5.3e-7 global, combine 2.8e-7 per row.  Gradient rows use a 1e-2 floor: a source without out-edges has the
row ds_trg · a_trg, and for a LeakyReLU target whose scores share a sign ds_trg = Σ α(dα - t)·act' = t(1 - Σα)·act' cancels
to ~0 exactly, leaving fp32 rounding of its terms (measured up to 6e-7 · rms)."""
import functools

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu

# (nheads, F): the first four take the wide-head path (F % 32 == 0), the rest the narrow one; W reaches 512, nheads 32, F 1
HEADS = [(1, 512), (2, 64), (4, 128), (16, 32), (2, 16), (3, 100), (5, 24), (32, 16), (7, 1)]
MODES = [("leakyrelu", "global"), ("leakyrelu", "segment"), ("sigmoid", "global"), ("sigmoid", "segment")]
SPECIAL_DEGREES = (1, 31, 32, 33, 64)    # lanes start striding over the in-edges above 32
HUB_DEGREE = 2100


FWD_REL, FWD_ROW = 2e-6, 5e-5
GRAD_REL, GRAD_ROW, GRAD_FLOOR = 5e-6, 2e-4, 1e-2


def row_err(got, ref, floor=1e-3):
    got, ref = got.double().reshape(ref.shape[0], -1), ref.double().reshape(ref.shape[0], -1)
    rn = ref.norm(dim=1)
    floor = max(floor * rn.pow(2).mean().sqrt().item(), 1e-30)
    return ((got - ref).norm(dim=1) / rn.clamp(min=floor)).max().item()


@functools.lru_cache(maxsize=None)
def _graph(n, seed=0):
    """Target-indexed CSR with: empty first / last rows and more empty targets, targets of in-degree exactly 1, 31, 32, 33 and
    64, one hub with HUB_DEGREE in-edges, random in-degrees 0-8 elsewhere, and sources that send nothing (every id ≡ 3 mod 7)."""
    from dance_b200 import ops
    rng = np.random.default_rng(seed)
    pool = np.flatnonzero(np.arange(n) % 7 != 3)
    deg = rng.integers(0, 9, n)
    deg[[0, n - 1]] = 0
    deg[5:5 + len(SPECIAL_DEGREES)] = SPECIAL_DEGREES
    deg[n // 2] = HUB_DEGREE
    trg = np.repeat(np.arange(n), deg)
    src = np.concatenate([rng.choice(pool, d, replace=False) for d in deg])
    T = sp.csr_matrix((np.ones(len(src), np.float32), (trg, src)), shape=(n, n))
    T.sort_indices()
    assert T.nnz == len(src)
    Tc = ops.CSR.from_scipy(T, "cuda", with_values=False)
    Tt, perm = ops.csr_transpose(Tc)
    return Tc, Tt, perm, torch.from_numpy(T.indices.astype(np.int64)).cuda(), torch.from_numpy(T.tocoo().row.astype(np.int64)).cuda()


def _indeg(T):
    return (T.rowptr[1:] - T.rowptr[:-1]).long()


def _params(n, nh, F, seed, spread=1.0):
    """H as the engine passes it (the first W columns of an [n, 2W] buffer) and attention vectors giving O(spread) scores."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    W = nh * F
    hs = torch.randn(n, 2 * W, device="cuda", generator=gen)
    a_src = torch.randn(W, device="cuda", generator=gen) * (spread / F**0.5)
    a_trg = torch.randn(W, device="cuda", generator=gen) * (spread / F**0.5)
    return hs, hs[:, :W], a_src, a_trg


def _reference(H, a_src, a_trg, src, trg, nh, act, shift, dOut=None, H2=None, dOut2=None, detach_max=False):
    """fp64 forward (out, α) and, given dOut, autograd gradients (dH, da_src, da_trg[, dH2])."""
    from oracle import gat_ref
    leaves = [t.detach().double().requires_grad_() for t in (H, a_src, a_trg)]
    if H2 is not None:
        leaves.append(H2.detach().double().requires_grad_())
    s_src, s_trg = gat_ref.scores(leaves[0], leaves[1], leaves[2], nh)
    res = gat_ref.aggregate(leaves[0], s_src, s_trg, src, trg, nh, act, 0.2, shift, detach_max=detach_max,
                            H2=leaves[3] if H2 is not None else None)
    out, alpha = res[0], res[1]
    if dOut is None:
        return out.detach(), alpha.detach()
    loss = (out * dOut.double()).sum()
    if H2 is not None:
        loss = loss + (res[2] * dOut2.double()).sum()
    return out.detach(), alpha.detach(), torch.autograd.grad(loss, leaves)


# ---------------------------------------------------------------------------------------------------------- scores / forward
@pytest.mark.parametrize("nh,F", HEADS)
def test_gat_scores_match_fp64(cuda, nh, F):
    from dance_b200 import ops
    from oracle import gat_ref
    n = 3000
    _, H, a_src, a_trg = _params(n, nh, F, seed=nh * 1000 + F)
    s_src, s_trg = ops.gat_scores(H, a_src, a_trg, nh)
    r_src, r_trg = gat_ref.scores(H.double(), a_src.double(), a_trg.double(), nh)
    scale = (H.double().abs().reshape(n, nh, F) * a_src.double().abs().reshape(nh, F)).sum(-1)   # Σ|h·a|: the dot's rounding scale
    assert ((s_src.double() - r_src).abs() <= 2e-6 * scale + 1e-30).all()
    scale = (H.double().abs().reshape(n, nh, F) * a_trg.double().abs().reshape(nh, F)).sum(-1)
    assert ((s_trg.double() - r_trg).abs() <= 2e-6 * scale + 1e-30).all()


@pytest.mark.parametrize("act,shift", MODES)
@pytest.mark.parametrize("nh,F", HEADS)
def test_gat_aggregate_fwd_matches_fp64(cuda, nh, F, act, shift):
    from dance_b200 import ops
    n = 3000
    T, _, _, src, trg = _graph(n)
    _, H, a_src, a_trg = _params(n, nh, F, seed=nh * 1000 + F)
    W = nh * F
    s_src, s_trg = ops.gat_scores(H, a_src, a_trg, nh)
    out, alpha, gmax = ops.gat_aggregate_fwd(T, H, s_src, s_trg, nh, act, 0.2, shift)
    ref_out, ref_alpha = _reference(H, a_src, a_trg, src, trg, nh, act, shift)
    assert rel_err(out, ref_out.cpu()) < FWD_REL and row_err(out, ref_out) < FWD_ROW
    assert rel_err(alpha, ref_alpha.cpu()) < FWD_REL and row_err(alpha, ref_alpha) < FWD_ROW
    # the output without α is the same arithmetic; a padded output buffer gets the same rows and keeps its padding
    out2, none, _ = ops.gat_aggregate_fwd(T, H, s_src, s_trg, nh, act, 0.2, shift, keep_alpha=False)
    assert none is None and torch.equal(out2, out)
    buf = torch.full((n, W + 7), float("nan"), device="cuda")
    ops.gat_aggregate_fwd(T, H, s_src, s_trg, nh, act, 0.2, shift, out=buf[:, :W])
    assert torch.equal(buf[:, :W], out) and buf[:, W:].isnan().all()
    deg = _indeg(T)
    assert (out[deg == 0] == 0).all()
    # Σα over each target's in-edges is 1 up to fp32 rounding of α and of the denominator (deg terms)
    asum = torch.zeros(n, nh, dtype=torch.float64, device="cuda").index_add_(0, trg, alpha.double())
    tol = 4e-7 * deg.clamp(min=8).double().unsqueeze(1)
    assert ((asum - 1).abs()[deg > 0] <= tol.expand(-1, nh)[deg > 0]).all()
    if shift == "global" and act == "leakyrelu":
        e = torch.nn.functional.leaky_relu(s_src[src] + s_trg[trg], 0.2)
        assert torch.equal(gmax, e.max().reshape(1))          # the max is order-independent: bit-equal


def test_gat_edge_max_all_negative_scores_is_exact(cuda):
    """Every LeakyReLU score negative: the global max goes through the unsigned-min branch of the float atomic max and is exact.
    The same negative pre-activations under sigmoid give scores in (0, 0.5), whose max agrees with fp64 within rounding."""
    from dance_b200 import ops
    n, nh = 3000, 3
    T, _, _, src, trg = _graph(n)
    gen = torch.Generator(device="cuda").manual_seed(11)
    s_src = -torch.rand(n, nh, device="cuda", generator=gen) - 0.5
    s_trg = -torch.rand(n, nh, device="cuda", generator=gen)
    H = torch.randn(n, nh * 8, device="cuda", generator=gen)
    for act in ("leakyrelu", "sigmoid"):
        _, _, gmax = ops.gat_aggregate_fwd(T, H, s_src, s_trg, nh, act, 0.2, "global")
        if act == "leakyrelu":
            want = torch.nn.functional.leaky_relu(s_src[src] + s_trg[trg], 0.2).max()
            assert gmax.item() < 0 and torch.equal(gmax, want.reshape(1))
        else:
            want = torch.sigmoid((s_src[src] + s_trg[trg]).double()).max()
            assert abs(gmax.item() - want.item()) <= 2e-7


# ---------------------------------------------------------------------------------------------------------- backward
@pytest.mark.parametrize("act,shift", MODES)
@pytest.mark.parametrize("nh,F", HEADS)
def test_gat_aggregate_bwd_matches_autograd(cuda, nh, F, act, shift):
    from dance_b200 import ops
    n = 3000
    T, Tt, perm, src, trg = _graph(n)
    _, H, a_src, a_trg = _params(n, nh, F, seed=nh * 1000 + F + 1)
    dOut = torch.randn(n, nh * F, device="cuda", generator=torch.Generator(device="cuda").manual_seed(F))
    s_src, s_trg = ops.gat_scores(H, a_src, a_trg, nh)
    _, alpha, gmax = ops.gat_aggregate_fwd(T, H, s_src, s_trg, nh, act, 0.2, shift)
    dH, da_src, da_trg = ops.gat_aggregate_bwd(T, Tt, perm, H, a_src, a_trg, s_src, s_trg, alpha, dOut, nh, act, 0.2,
                                               gmax=gmax if shift == "global" else None)
    _, _, (g_H, g_as, g_at) = _reference(H, a_src, a_trg, src, trg, nh, act, shift, dOut)
    assert rel_err(dH, g_H.cpu()) < GRAD_REL and row_err(dH, g_H, GRAD_FLOOR) < GRAD_ROW
    assert rel_err(da_src, g_as.cpu()) < GRAD_REL and rel_err(da_trg, g_at.cpu()) < GRAD_REL


@pytest.mark.parametrize("nh,F,act,shift", [(1, 512, "sigmoid", "segment"), (2, 16, "leakyrelu", "global"), (3, 100, "sigmoid", "global")])
def test_gat_aggregate_bwd_tied_matches_autograd(cuda, nh, F, act, shift):
    """STAGATE's tied attention: one α weights H and H2, dα sums both layers' dots; dH2 is the message path only."""
    from dance_b200 import ops
    n = 3000
    T, Tt, perm, src, trg = _graph(n)
    hs, H, a_src, a_trg = _params(n, nh, F, seed=7 * F + nh)
    W = nh * F
    gen = torch.Generator(device="cuda").manual_seed(3)
    H2 = hs[:, W:]
    dOut = torch.randn(n, W, device="cuda", generator=gen)
    dOut2 = torch.randn(n, W + 5, device="cuda", generator=gen)[:, :W]
    s_src, s_trg = ops.gat_scores(H, a_src, a_trg, nh)
    _, alpha, gmax = ops.gat_aggregate_fwd(T, H, s_src, s_trg, nh, act, 0.2, shift)
    gm = gmax if shift == "global" else None
    _, _, (g_H, g_as, g_at, g_H2) = _reference(H, a_src, a_trg, src, trg, nh, act, shift, dOut, H2=H2, dOut2=dOut2)
    for want_dH2 in (True, False):
        dH, da_src, da_trg, dH2 = ops.gat_aggregate_bwd(T, Tt, perm, H, a_src, a_trg, s_src, s_trg, alpha, dOut, nh, act, 0.2, H2=H2,
                                                        dOut2=dOut2, want_dH2=want_dH2, gmax=gm)
        assert rel_err(dH, g_H.cpu()) < GRAD_REL and row_err(dH, g_H, GRAD_FLOOR) < GRAD_ROW
        assert rel_err(da_src, g_as.cpu()) < GRAD_REL and rel_err(da_trg, g_at.cpu()) < GRAD_REL
        if want_dH2:
            assert rel_err(dH2, g_H2.cpu()) < GRAD_REL and row_err(dH2, g_H2, GRAD_FLOOR) < GRAD_ROW
        else:
            assert dH2 is None


@pytest.mark.parametrize("act,shift", MODES)
@pytest.mark.parametrize("nh,F", [(1, 32), (4, 8)])
def test_gat_large_graph_fwd_bwd(cuda, nh, F, act, shift):
    """n = 40 000: the warps' grid-stride loops wrap (more rows than SMs·16·8) and the score-gradient reduction runs with
    many row splits."""
    from dance_b200 import ops
    n = 40_000
    T, Tt, perm, src, trg = _graph(n, seed=1)
    _, H, a_src, a_trg = _params(n, nh, F, seed=F)
    dOut = torch.randn(n, nh * F, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    s_src, s_trg = ops.gat_scores(H, a_src, a_trg, nh)
    out, alpha, gmax = ops.gat_aggregate_fwd(T, H, s_src, s_trg, nh, act, 0.2, shift)
    dH, da_src, da_trg = ops.gat_aggregate_bwd(T, Tt, perm, H, a_src, a_trg, s_src, s_trg, alpha, dOut, nh, act, 0.2,
                                               gmax=gmax if shift == "global" else None)
    ref_out, ref_alpha, (g_H, g_as, g_at) = _reference(H, a_src, a_trg, src, trg, nh, act, shift, dOut)
    assert rel_err(out, ref_out.cpu()) < FWD_REL and row_err(out, ref_out) < FWD_ROW
    assert row_err(alpha, ref_alpha) < FWD_ROW
    assert (out[_indeg(T) == 0] == 0).all()
    assert rel_err(dH, g_H.cpu()) < GRAD_REL and row_err(dH, g_H, GRAD_FLOOR) < GRAD_ROW
    assert rel_err(da_src, g_as.cpu()) < GRAD_REL and rel_err(da_trg, g_at.cpu()) < GRAD_REL


@pytest.mark.parametrize("shift", ["global", "segment"])
@pytest.mark.parametrize("nh,F", [(2, 16), (1, 32)])
def test_gat_wide_score_spread(cuda, nh, F, shift):
    """A group of targets whose scores all lie 38-48 below every other score.  Global shift: Σ exp(score - max) of those targets is
    comparable to the 1e-16 of the denominator, their α sum to well below 1, and the gradient through the (non-detached) global max
    is O(1) — the backward with the forward's gmax matches the literal autograd, which this case makes differ from the detached one
    by far more than the tolerance.  Per-target shift: the shift alone keeps those targets' softmax normal."""
    from dance_b200 import ops
    n = 3000
    W = nh * F
    T, Tt, perm, src, trg = _graph(n)
    gen = torch.Generator(device="cuda").manual_seed(21)
    H = torch.randn(n, W, device="cuda", generator=gen)
    a_src = torch.randn(nh, F, device="cuda", generator=gen) / F**0.5
    a_trg = torch.randn(nh, F, device="cuda", generator=gen) * 0.05
    a_src[:, 0], a_trg[:, 0] = 0.0, 1.0
    # the low group: targets that send no messages (ids ≡ 3 mod 7), so their large column 0 only moves their own s_trg
    low = torch.arange(n, device="cuda") % 7 == 3
    offs = -5.0 * (38.0 + 10.0 * torch.rand(n, nh, device="cuda", generator=gen))     # LeakyReLU(0.2) · offs ∈ [-48, -38]
    H.view(n, nh, F)[:, :, 0] = torch.where(low.unsqueeze(1), offs, H.view(n, nh, F)[:, :, 0])
    a_src, a_trg = a_src.reshape(-1).contiguous(), a_trg.reshape(-1).contiguous()
    dOut = torch.randn(n, W, device="cuda", generator=gen)
    s_src, s_trg = ops.gat_scores(H, a_src, a_trg, nh)
    out, alpha, gmax = ops.gat_aggregate_fwd(T, H, s_src, s_trg, nh, "leakyrelu", 0.2, shift)
    ref_out, ref_alpha, (g_H, g_as, g_at) = _reference(H, a_src, a_trg, src, trg, nh, "leakyrelu", shift, dOut)
    asum = torch.zeros(n, nh, dtype=torch.float64, device="cuda").index_add_(0, trg, ref_alpha)
    deg = _indeg(T)
    assert asum[~low & (deg > 0)].min() > 1 - 1e-9
    assert rel_err(out, ref_out.cpu()) < FWD_REL and row_err(out, ref_out) < FWD_ROW and row_err(alpha, ref_alpha) < FWD_ROW
    if shift == "global":
        assert asum[low & (deg > 0)].max() < 0.9
        _, _, (d_H, _, _) = _reference(H, a_src, a_trg, src, trg, nh, "leakyrelu", "global", dOut, detach_max=True)
        assert row_err(d_H, g_H) > 10 * GRAD_ROW                          # the shift's gradient is visible at this spread
    dH, da_src, da_trg = ops.gat_aggregate_bwd(T, Tt, perm, H, a_src, a_trg, s_src, s_trg, alpha, dOut, nh, "leakyrelu", 0.2,
                                               gmax=gmax if shift == "global" else None)
    assert rel_err(dH, g_H.cpu()) < GRAD_REL and row_err(dH, g_H, GRAD_FLOOR) < GRAD_ROW
    assert rel_err(da_src, g_as.cpu()) < GRAD_REL and rel_err(da_trg, g_at.cpu()) < GRAD_REL


# ---------------------------------------------------------------------------------------------------------- known answers
@pytest.mark.parametrize("act,shift", MODES)
@pytest.mark.parametrize("nh,F", [(2, 64), (5, 24)])
def test_gat_zero_attention_is_neighbour_mean(cuda, nh, F, act, shift):
    from dance_b200 import ops
    n = 3000
    T, _, _, src, trg = _graph(n)
    _, H, _, _ = _params(n, nh, F, seed=2)
    zero = torch.zeros(nh * F, device="cuda")
    s_src, s_trg = ops.gat_scores(H, zero, zero, nh)
    out, _, _ = ops.gat_aggregate_fwd(T, H, s_src, s_trg, nh, act, 0.2, shift)
    deg = _indeg(T).double().clamp(min=1).unsqueeze(1)
    mean = torch.zeros(n, nh * F, dtype=torch.float64, device="cuda").index_add_(0, trg, H.double()[src]) / deg
    assert row_err(out, mean) < 1e-5


@pytest.mark.parametrize("act", ["leakyrelu", "sigmoid"])
@pytest.mark.parametrize("nh,F", [(2, 64), (5, 24)])
def test_gat_single_in_edge_copies_the_source(cuda, nh, F, act):
    """Every target has exactly one in-edge: out = H[src].  Per-target shift: p = exp(0) = 1 and α = 1/(1 + 1e-16f) = 1 exactly."""
    from dance_b200 import ops
    n = 3000
    src = torch.from_numpy(np.random.default_rng(4).permutation(n).astype(np.int32)).cuda()
    T = ops.CSR(torch.arange(n + 1, dtype=torch.int32, device="cuda"), src, None, (n, n))
    _, H, a_src, a_trg = _params(n, nh, F, seed=9)
    s_src, s_trg = ops.gat_scores(H, a_src, a_trg, nh)
    out, alpha, _ = ops.gat_aggregate_fwd(T, H, s_src, s_trg, nh, act, 0.2, "segment")
    assert torch.equal(out, H[src.long()]) and (alpha == 1).all()
    out, _, _ = ops.gat_aggregate_fwd(T, H, s_src, s_trg, nh, act, 0.2, "global")
    assert ((out - H[src.long()]).abs() <= 2.0**-22 * H[src.long()].abs()).all()


def test_gat_negative_zero_scores_global_shift(cuda):
    """s_src = s_trg = -0.0: every LeakyReLU score is -0.0, the global max must be ±0 (not -inf) and the output the neighbour mean."""
    from dance_b200 import ops
    n, nh, F = 3000, 2, 16
    T, _, _, src, trg = _graph(n)
    _, H, _, _ = _params(n, nh, F, seed=3)
    s = torch.full((n, nh), -0.0, device="cuda")
    out, _, gmax = ops.gat_aggregate_fwd(T, H, s, s.clone(), nh, "leakyrelu", 0.2, "global")
    assert gmax.item() == 0.0
    assert torch.isfinite(out).all()
    deg = _indeg(T).double().clamp(min=1).unsqueeze(1)
    mean = torch.zeros(n, nh * F, dtype=torch.float64, device="cuda").index_add_(0, trg, H.double()[src]) / deg
    assert row_err(out, mean) < 1e-5


@pytest.mark.parametrize("shift", ["global", "segment"])
def test_gat_empty_graph_and_zero_rows(cuda, shift):
    from dance_b200 import ops
    nh, F = 2, 16
    W = nh * F
    for n in (500, 0):
        T = ops.CSR(torch.zeros(n + 1, dtype=torch.int32, device="cuda"), torch.zeros(0, dtype=torch.int32, device="cuda"), None, (n, n))
        Tt, perm = ops.csr_transpose(T)
        _, H, a_src, a_trg = _params(max(n, 1), nh, F, seed=1)
        H = H[:n]
        s_src, s_trg = ops.gat_scores(H, a_src, a_trg, nh)
        out, alpha, gmax = ops.gat_aggregate_fwd(T, H, s_src, s_trg, nh, "leakyrelu", 0.2, shift)
        assert out.shape == (n, W) and (out == 0).all() and alpha.shape == (0, nh)
        dOut = torch.ones(n, W, device="cuda")
        dH, da_src, da_trg = ops.gat_aggregate_bwd(T, Tt, perm, H, a_src, a_trg, s_src, s_trg, alpha, dOut, nh,
                                                   gmax=gmax if shift == "global" else None)
        assert (dH == 0).all() and (da_src == 0).all() and (da_trg == 0).all()
        dH, da_src, _, dH2 = ops.gat_aggregate_bwd(T, Tt, perm, H, a_src, a_trg, s_src, s_trg, alpha, dOut, nh, H2=H, dOut2=dOut)
        assert (dH == 0).all() and (dH2 == 0).all() and (da_src == 0).all()
        comb = ops.gat_combine_fwd(out, None, None, nh, False, "elu")
        dpre, dact = ops.gat_combine_bwd(torch.ones_like(comb), comb, nh, F, False, "elu")
        assert comb.shape == (n, F) and dpre.shape == (n, W) and dact.shape == (n, F)


def test_gat_bad_arguments_raise(cuda):
    from dance_b200 import ops
    from dance_b200._lib import B2Error
    n = 3000
    T, Tt, perm, _, _ = _graph(n)
    gen = torch.Generator(device="cuda").manual_seed(0)
    H = torch.randn(n, 100, device="cuda", generator=gen)
    a = torch.randn(100, device="cuda", generator=gen)
    s = torch.zeros(n, 3, device="cuda")
    with pytest.raises(B2Error, match="multiple of nheads"):
        ops.gat_scores(H, a, a, 3)
    with pytest.raises(B2Error, match="multiple of nheads"):
        ops.gat_aggregate_fwd(T, H, s, s, 3)
    with pytest.raises(B2Error, match="multiple of nheads"):
        ops.gat_aggregate_bwd(T, Tt, perm, H, a, a, s, s, torch.zeros(T.nnz, 3, device="cuda"), H, 3)
    with pytest.raises(B2Error, match="multiple of nheads"):
        ops.gat_combine_fwd(H, None, None, 3, True)
    Hw = torch.randn(n, 520, device="cuda", generator=gen)
    with pytest.raises(B2Error):
        ops.gat_aggregate_fwd(T, Hw, torch.zeros(n, 2, device="cuda"), torch.zeros(n, 2, device="cuda"), 2, shift="segment")
    H33 = torch.randn(n, 33, device="cuda", generator=gen)
    a33 = torch.randn(33, device="cuda", generator=gen)
    s_src, s_trg = ops.gat_scores(H33, a33, a33, 33)
    _, alpha, _ = ops.gat_aggregate_fwd(T, H33, s_src, s_trg, 33, shift="segment")
    with pytest.raises(B2Error):
        ops.gat_aggregate_bwd(T, Tt, perm, H33, a33, a33, s_src, s_trg, alpha, H33, 33)


# ---------------------------------------------------------------------------------------------------------- combine
@pytest.mark.parametrize("act", [None, "relu", "elu", "tanh"])
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("skip", [False, True])
@pytest.mark.parametrize("concat", [True, False])
def test_gat_combine_fwd_bwd_matches_autograd(cuda, concat, skip, bias, act):
    """agg / skip / dout with padded leading dimensions (skip as the second half of the engine's [n, 2W] buffer)."""
    from dance_b200 import ops
    from oracle import gat_ref
    n, nh, F = 777, 3, 20
    W = nh * F
    OW = W if concat else F
    gen = torch.Generator(device="cuda").manual_seed(8 * int(concat) + 4 * int(skip) + 2 * int(bias) + len(act or ""))
    agg = torch.randn(n, W + 5, device="cuda", generator=gen)[:, :W]
    sk = torch.randn(n, 2 * W + 3, device="cuda", generator=gen)[:, W:2 * W] if skip else None
    b = torch.randn(OW, device="cuda", generator=gen) if bias else None
    dout = torch.randn(n, OW + 9, device="cuda", generator=gen)[:, :OW]
    out = ops.gat_combine_fwd(agg, sk, b, nh, concat, act)
    dpre, dact = ops.gat_combine_bwd(dout, out, nh, F, concat, act)
    leaves = [t.double().requires_grad_() if t is not None else None for t in (agg, sk)]
    pre = gat_ref.combine(leaves[0], leaves[1], b.double() if bias else None, nh, concat, None)
    pre.retain_grad()
    ref = gat_ref.combine(pre, None, None, 1, True, act)
    ref.backward(dout.double())
    assert row_err(out, ref.detach()) < 2e-6
    assert row_err(dact, pre.grad) < 2e-6 and row_err(dpre, leaves[0].grad) < 2e-6
    if skip:
        assert torch.equal(leaves[1].grad, leaves[0].grad)          # d(skip) = d(agg): the engine writes one into the other
