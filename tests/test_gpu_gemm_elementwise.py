"""The tensor-core GEMM and its CUDA-core fallback (``ops.gemm`` / ``b2_gemm_f32``) checked element by element against
float64, at the edges of its tiles, of its split-K plan, of its epilogue and of its dispatch rules.

Element-wise bound
------------------
Let a = op(A) (M x K) and b = op(B) (K x N) be the fp32 operands, ref = a·b and P = |a|·|b|, both in float64 (in bf16 mode
from the operands rounded to bfloat16 the way the kernel rounds them, ``bf16_ref.bf16``).  Before the epilogue every element
of C satisfies

    |C - ref| <= tau · P,        tau(mode, K) = u_op(mode) + c_acc(mode) · n(mode, K) · 2^-24.

u_op bounds the relative error of one product that comes from rounding its two operands:
  tf32    wgmma reads the upper 19 bits of each fp32 operand (10-bit mantissa, the rest dropped): |â - a| < 2^-10 |a|, so
          |â·b̂ - a·b| < (2·2^-10 + 2^-20) |a||b|.
  tf32x3  hi = x & 0xFFFFE000 is exact in tf32 and lo = x - hi is exact in fp32 with |lo| < 2^-10 |x|; the tensor core
          drops the low bits of lo in turn, by less than 2^-10 |lo| < 2^-20 |x|.  The product leaves out lo·lo and uses the two
          shortened lo's, each costing less than 2^-20 |a||b|: u_op = 3·2^-20.
  bf16    0 against the rounded operands: the product of two 8-bit mantissas is exact in fp32.
  fp32    0: the CUDA-core kernel multiplies the fp32 operands with fmaf.
The second term is the fp32 accumulation.  If the running sum of an element is rounded n times, each rounding errs by at
most 2^-24 (to nearest) or 2^-23 (toward zero) of a partial sum, and no partial sum exceeds P, so the error is below
n·2^-24·P, or n·2^-23·P (Higham, "Accuracy and Stability of Numerical Algorithms", 2nd ed., section 3.1).
  fp32    one fmaf per k, rounded to nearest: n = K, c_acc = 1.
  tensor  one accumulator update per wgmma k-step of 8 (tf32, tf32x3) or 16 (bf16) products, and the tensor cores have been
  cores   found to truncate, not round, in their accumulation (Fasi, Higham, Mikaitis & Pranesh, "Numerical behavior of
          NVIDIA tensor cores", PeerJ Comput. Sci. 7:e330, 2021): n = ceil(K / k-step) + 2, c_acc = 2.  The + 2 is fitted,
          not derived: with it, the measured ratio below stays between 0.7 and 1.1 from K = 8 to K = 100 000 in tf32 and
          tf32x3 (in bf16 it rises from 0.6 to 1.5).  A split-K plan gives each split a shorter chain, and its reduction
          adds `splits` rounded sums, fewer than the k-steps it saves.
No data sheet states how the tensor cores accumulate, so the model is checked against H100 runs of this file, measured
against ref_k, the exact float64 product of the operands as the kernel rounds them (tf32: upper 19 bits; tf32x3: hi·hi +
lo'·hi + hi·lo' with lo' the upper 19 bits of lo; bf16: round to nearest even; fp32: unchanged), so that the operand
rounding does not hide it.  The largest measured ratio max |C - ref_k| / (n·2^-24·P) over every case of this file, on an
H100 80 GB HBM3 (SXM5, 700 W power limit):

    fp32 0.44 (K = 7), tf32x3 1.09 (K = 224), tf32 1.07 (K = 224), bf16 1.51 (K = 100 000)

so each c_acc is at least its mode's ratio and at most 4x it.  On one-signed sums (below) the tensor cores' error does grow
linearly in K, about one 2^-24 of P per k-step, while round-to-nearest fmaf stays far below its bound as K grows.  Every case asserts
|C - ref_k| <= c_acc·n·2^-24·P and, which follows from it because |ref_k - ref| <= u_op·P, |C - ref| <= tau·P.

The epilogue (bias, activation, ReLU mask, accumulate) is applied to ref and ref_k in float64.  bias, relu, elu and tanh are
1-Lipschitz, so the accumulation error passes through them unchanged; the kernel's own fp32 epilogue adds at most
2^-21·(|ref| + |bias| + |C0|): one rounding of the bias sum, tanhf / expm1f within 2 ulps (CUDA C++ Programming Guide,
single-precision mathematical functions) and one rounding of the accumulate.

Rows of op(A) are scaled by 2^20, 1 and 2^-20 and columns of op(B) by 1, 2^8 and 2^-8 in turn, so that the hi / lo split
and the rounding run at exponents far from 1; the bound scales with P, so none of them needs a looser tau.  Every fifth row
of op(A) and every fourth column of op(B) are made non-negative: where they meet, the K terms have one sign, |ref| = P, and
the accumulation error relative to P is largest (over terms of random sign it barely grows with K).

Exact checks
------------
- A masked-out element (mask <= 0, -0.0 or NaN: the kernels test !(m > 0)) is exactly 0, or exactly C0 with accumulate.
- ``out`` is an M x N view into a NaN buffer with two more rows, spare columns and, where its base is one float past a
  16-byte boundary, one float before it: nothing outside the view changes.
- Operands are stored with leading dimensions padded to multiples of 4 (so odd M, N, K reach the tensor cores in every
  layout), and the padding is NaN: a read of it would poison the result.
- Shapes the tensor-core kernel does not take give a result bit-identical to precision="fp32"; every shape meant for it
  gives a result that is not.  Two calls give bit-identical results, split-K included.

The split-K plan of ``make_plan`` (csrc/gemm_tc.cu) is restated in :func:`plan`, checked against
``b2_gemm_workspace_bytes`` and used to place shapes on both sides of each of its boundaries."""
from typing import NamedTuple

import pytest
import torch

from bf16_ref import bf16

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
U_OP = {"fp32": 0.0, "tf32x3": 3 * 2.0 ** -20, "tf32": 2 * 2.0 ** -10 + 2.0 ** -20, "bf16": 0.0}
C_ACC = {"fp32": 1.0, "tf32x3": 2.0, "tf32": 2.0, "bf16": 2.0}
K_STEP = {"tf32x3": 8, "tf32": 8, "bf16": 16}       # products per wgmma k-step
EPILOGUE_ROUNDING = 2.0 ** -21


def roundings(precision, K):
    """n: how many times the running sum of one element is rounded (see the module docstring)"""
    return K if precision == "fp32" else -(-K // K_STEP[precision]) + 2

TC = ["tf32x3", "tf32", "bf16"]
LAYOUTS = [(0, 1), (0, 0), (1, 0), (1, 1)]
ACTS = ["none", "relu", "elu", "tanh"]
OUTS = ["aligned", "odd_ldc", "offset"]
NAN_BITS = torch.tensor(float("nan")).view(torch.int32).item()


def cdiv(a, b):
    return -(-a // b)


def pad4(n):
    return cdiv(n, 4) * 4


# ---------------------------------------------------------------------------------------------------- split-K plan
BM, BK = 128, 32


class Plan(NamedTuple):
    BN: int
    tiles: int
    kb_total: int
    wanted: int          # splits that would give every SM a CTA, before the kb_total / 4 cap
    splits: int
    kb_per_split: int


def plan(M, N, K, sms):
    """make_plan of csrc/gemm_tc.cu: the tile width, the 128 x BN output tiles, the 32-wide k-blocks and the split-K plan
    (the same in every precision).  Split only when the tiles fill less than 0.6 of the SMs and there are at least 8
    k-blocks; then aim at one CTA per SM, with at least 4 k-blocks per split, and drop the splits left empty by rounding."""
    BN = 32 if N <= 32 else (64 if N <= 64 else 128)
    tiles = cdiv(M, BM) * cdiv(N, BN)
    kb_total = cdiv(K, BK)
    wanted = cdiv(sms, tiles)
    splits = 1
    if tiles * 10 < sms * 6 and kb_total >= 8:
        splits = max(1, min(wanted, kb_total // 4))
    kb_per_split = cdiv(kb_total, splits)
    return Plan(BN, tiles, kb_total, wanted, cdiv(kb_total, kb_per_split), kb_per_split)


def plan_workspace_bytes(M, N, K, sms):
    p = plan(M, N, K, sms)
    return p.splits * M * N * 4 if p.splits > 1 else 0


def workspace_bytes(M, N, K, transA, transB, precision):
    from dance_b200 import ops
    return int(ops.lib().b2_gemm_workspace_bytes(M, N, K, int(transA), int(transB), ops.PREC[precision]))


@pytest.fixture(scope="module")
def sms(cuda):
    from dance_b200 import ops
    return ops.device_info()[0]


# ---------------------------------------------------------------------------------------------------- operands and canvas
def _matrix(rows, cols, g, dev, ld=None, off=0):
    """rows x cols standard normal fp32, in a NaN buffer with leading dimension ld (default: cols padded to a multiple of
    4), starting `off` floats into it"""
    ld = pad4(cols) if ld is None else ld
    buf = torch.full((off + rows * ld,), float("nan"), device=dev)
    view = buf[off:].view(rows, ld)[:, :cols]
    view.copy_(torch.randn(rows, cols, generator=g, device=dev))
    return view


def _cycle(values, n, dev):
    return torch.tensor(values, dtype=torch.float32, device=dev)[torch.arange(n, device=dev) % len(values)]


def _mask(M, N, g, dev):
    """ReLU-mask operand (leading dimension N + 3): normal values with exact zeros, -0.0 and NaNs among them"""
    v = torch.randn(M * N, generator=g, device=dev)
    v[::7] = 0.0
    v[3::11] = -0.0
    v[5::13] = float("nan")
    buf = torch.full((M, N + 3), float("nan"), device=dev)
    buf[:, :N] = v.view(M, N)
    return buf[:, :N]


class Canvas:
    """``out``: an M x N view into a NaN buffer with two more rows and spare columns.  aligned: even ldc, 16-byte aligned
    base; odd_ldc: odd ldc; offset: base one float past a 16-byte boundary, with one float before it."""

    def __init__(self, M, N, kind, dev):
        off = 1 if kind == "offset" else 0
        ld = N + 1 + N % 2 if kind == "odd_ldc" else pad4(N) + 4
        self.buf = torch.full((off + (M + 2) * ld,), float("nan"), device=dev)
        self.out = self.buf[off:off + M * ld].view(M, ld)[:, :N]
        self.inside = torch.zeros(self.buf.shape, dtype=torch.bool, device=dev)
        self.inside[off:off + M * ld].view(M, ld)[:, :N] = True
        assert self.out.data_ptr() % 16 == (4 if kind == "offset" else 0) and (ld % 2 == 1) == (kind == "odd_ldc")

    def assert_outside_untouched(self):
        bits = self.buf.view(torch.int32)[~self.inside]
        written = int((bits != NAN_BITS).sum())
        assert written == 0, f"{written} floats outside `out` were written"

    def bits(self):
        return self.buf.view(torch.int32)


# ---------------------------------------------------------------------------------------------------- references
def _tf32(x):
    """x with the low 13 of its 23 mantissa bits cleared: the tf32 operand wgmma reads"""
    return (x.contiguous().view(torch.int32) & -8192).view(torch.float32)


def _references(a, b, precision):
    """(ref, ref_k, P) in float64: the exact product, the exact product of the operands as the kernel rounds them, |a|·|b|"""
    if precision == "bf16":
        ad, bd = bf16(a), bf16(b)
        ref = ad @ bd
        return ref, ref, ad.abs() @ bd.abs()
    ad, bd = a.double(), b.double()
    ref, P = ad @ bd, ad.abs() @ bd.abs()
    if precision == "fp32":
        return ref, ref, P
    ha, hb = _tf32(a), _tf32(b)
    if precision == "tf32":
        return ref, ha.double() @ hb.double(), P
    la, lb = _tf32(a - ha).double(), _tf32(b - hb).double()
    ha, hb = ha.double(), hb.double()
    return ref, ha @ hb + (la @ hb + ha @ lb), P


def _epilogue(x, bias, act, mask, C0):
    if bias is not None:
        x = x + bias.double()
    if act == "relu":
        x = torch.relu(x)
    elif act == "elu":
        x = torch.nn.functional.elu(x)
    elif act == "tanh":
        x = torch.tanh(x)
    if mask is not None:
        x = torch.where(mask > 0, x, 0.0)
    return x if C0 is None else x + C0.double()


def _check(C, ref, ref_k, P, precision, K, slack, live):
    """Assert both element-wise bounds on the elements in `live`; returns the largest |C - ref_k| net of `slack`, over
    n·2^-24·P (the measured accumulation ratio)."""
    C = C.double()
    acc = roundings(precision, K) * U * P
    bound_k = C_ACC[precision] * acc + slack
    bound = U_OP[precision] * P + bound_k
    err_k, err = (C - ref_k).abs(), (C - ref).abs()
    for what, e, bnd in (("ref_k", err_k, bound_k), ("ref", err, bound)):
        bad = ~(e <= bnd) & live                     # a NaN counts as a violation
        n = int(bad.sum())
        if n:
            i, j = (int(v) for v in bad.nonzero()[0])
            pytest.fail(f"{precision}: {n} of {int(live.sum())} elements outside the bound against {what}; first at "
                        f"({i}, {j}): C = {C[i, j].item()!r}, {what} = {(ref_k if what == 'ref_k' else ref)[i, j].item()!r}, "
                        f"bound {bnd[i, j].item():.3g}, error {e[i, j].item():.3g}")
    ratio = ((err_k - slack).clamp_min(0) / acc)[live & (acc > 0)]
    return ratio.max().item() if ratio.numel() else 0.0


class Case:
    """Seeded operands and epilogue inputs of one GEMM, run on a NaN canvas and checked against float64."""

    def __init__(self, dev, M, N, K, transA=0, transB=1, seed=0, bias=False, act="none", mask=False, accumulate=False,
                 lda=None, ldb=None, a_off=0, b_off=0):
        self.dev, self.M, self.N, self.K, self.transA, self.transB, self.act = dev, M, N, K, transA, transB, act
        g = torch.Generator(device=dev).manual_seed(seed)
        self.A = _matrix(K, M, g, dev, lda, a_off) if transA else _matrix(M, K, g, dev, lda, a_off)
        self.B = _matrix(N, K, g, dev, ldb, b_off) if transB else _matrix(K, N, g, dev, ldb, b_off)
        self.a, self.b = (self.A.t() if transA else self.A), (self.B.t() if transB else self.B)
        self.a.mul_(_cycle([2.0 ** 20, 1.0, 2.0 ** -20], M, dev)[:, None])
        self.b.mul_(_cycle([1.0, 2.0 ** 8, 2.0 ** -8], N, dev)[None, :])
        self.a[::5].abs_()
        self.b[:, ::4].abs_()
        self.bias = torch.randn(N, generator=g, device=dev) if bias else None
        self.mask = _mask(M, N, g, dev) if mask else None
        self.C0 = torch.randn(M, N, generator=g, device=dev) if accumulate else None

    def run(self, precision, out="aligned"):
        from dance_b200 import ops
        cv = Canvas(self.M, self.N, out, self.dev)
        if self.C0 is not None:
            cv.out.copy_(self.C0)
        ops.gemm(self.A, self.B, transA=bool(self.transA), transB=bool(self.transB), bias=self.bias, act=self.act,
                 mask=self.mask, out=cv.out, accumulate=self.C0 is not None, precision=precision)
        return cv

    def check(self, cv, precision):
        """All checks of one result; returns the measured accumulation ratio"""
        cv.assert_outside_untouched()
        C = cv.out
        live = torch.ones(C.shape, dtype=torch.bool, device=self.dev)
        if self.mask is not None:
            live = self.mask > 0
            dead = ~live
            if self.C0 is None:
                assert bool((C[dead] == 0).all()), f"{int((C[dead] != 0).sum())} masked-out elements are not 0"
            else:
                assert torch.equal(C[dead].view(torch.int32), self.C0[dead].view(torch.int32)), \
                    f"{int((C[dead] != self.C0[dead]).sum())} masked-out elements are not C0"
        ref, ref_k, P = _references(self.a, self.b, precision)
        slack = 0.0
        if self.bias is not None or self.act != "none" or self.mask is not None or self.C0 is not None:
            slack = EPILOGUE_ROUNDING * (ref.abs() + (0 if self.bias is None else self.bias.double().abs())
                                         + (0 if self.C0 is None else self.C0.double().abs()))
            ref, ref_k = (_epilogue(x, self.bias, self.act, self.mask, self.C0) for x in (ref, ref_k))
        return _check(C, ref, ref_k, P, precision, self.K, slack, live)


def _run_checked(case, precision, out="aligned", computed_as=None):
    """Run, check (as `computed_as`, the precision of the kernel expected to run), run again: the second result must be
    bit-identical, canvas included"""
    cv = case.run(precision, out)
    case.check(cv, computed_as or precision)
    again = case.run(precision, out)
    assert torch.equal(again.bits(), cv.bits()), f"{precision}: two calls differ"
    return cv


def _assert_tensor_cores_ran(case, cv, precision, out="aligned"):
    """The CUDA-core kernel's result (itself checked) differs from the tensor-core one: no silent fall-back"""
    ref = case.run("fp32", out)
    case.check(ref, "fp32")
    assert not torch.equal(cv.out.view(torch.int32), ref.out.view(torch.int32)), \
        f"{precision} gave the CUDA-core kernel's result bit for bit: the tensor cores did not run"


# ---------------------------------------------------------------------------------------------------- split-K plan tests
def test_split_k_plan_matches_workspace_bytes(cuda, sms):
    """The restated plan gives the workspace b2_gemm_workspace_bytes asks for, over a grid of shapes on both sides of the
    split decision, in every precision and layout."""
    got = {}
    split = unsplit = 0
    for M in (1, 127, 128, 129, 640, 4000, 10113):
        for N in (1, 32, 33, 64, 65, 128, 129, 1000):
            for K in (1, 8, 224, 225, 256, 1300, 12800, 100_000):
                want = plan_workspace_bytes(M, N, K, sms)
                split, unsplit = split + (want > 0), unsplit + (want == 0)
                for precision in TC:
                    for transA, transB in LAYOUTS:
                        have = workspace_bytes(M, N, K, transA, transB, precision)
                        if have != want:
                            got[(M, N, K, precision, transA, transB)] = (have, want)
    assert not got, f"{len(got)} shapes differ from the restated plan, e.g. {next(iter(got.items()))}"
    assert split > 100 and unsplit > 100


def _last_split_one_k_block(p):
    return p.splits > 2 and p.kb_total - (p.splits - 1) * p.kb_per_split == 1


def _boundary_shapes(sms):
    """Shapes one step either side of each boundary of the split-K plan on this device's SM count:
    name -> (M, N, K, what the plan must show)"""
    t = cdiv(6 * sms, 10) - 1                  # the most tiles with tiles·10 < sms·6
    s = cdiv(sms, 12)                          # splits wanted by 12 tiles of 128 x 128 (384 x 511)
    # 128 x 129 (2 tiles): the first K whose last split holds a single k-block, that k-block holding one element of K
    k_one = next(32 * (kb - 1) + 1 for kb in range(8, 4096) if _last_split_one_k_block(plan(128, 129, 32 * kb, sms)))
    return {
        "kb_total=7_unsplit": (128, 129, 224, lambda p: p.kb_total == 7 and p.splits == 1),
        "kb_total=8_split": (128, 129, 225, lambda p: p.kb_total == 8 and p.splits == 2),
        "tiles_below_0.6_sms_split": (128 * (t - 1) + 1, 33, 256, lambda p: p.tiles * 10 < 6 * sms and p.splits == 2),
        "tiles_at_0.6_sms_unsplit": (128 * t + 1, 33, 256, lambda p: p.tiles * 10 >= 6 * sms and p.splits == 1),
        "splits_not_capped": (384, 511, 32 * 4 * s - 31,
                              lambda p: p.tiles == 12 and p.kb_total // 4 == p.wanted and p.splits == p.wanted),
        "splits_capped_by_kb_total/4": (384, 511, 32 * (4 * s - 1),
                                        lambda p: p.tiles == 12 and p.kb_total // 4 == p.wanted - 1 and p.splits < p.wanted),
        "last_split_one_k_block": (128, 129, k_one, _last_split_one_k_block),
    }


BOUNDARIES = ["kb_total=7_unsplit", "kb_total=8_split", "tiles_below_0.6_sms_split", "tiles_at_0.6_sms_unsplit",
              "splits_not_capped", "splits_capped_by_kb_total/4", "last_split_one_k_block"]


@pytest.mark.parametrize("precision", TC)
@pytest.mark.parametrize("transA,transB", LAYOUTS)
@pytest.mark.parametrize("boundary", BOUNDARIES)
def test_split_k_plan_boundary(cuda, sms, boundary, transA, transB, precision):
    M, N, K, side = _boundary_shapes(sms)[boundary]
    p = plan(M, N, K, sms)
    assert side(p), f"{boundary}: {(M, N, K)} gives {p}"
    assert workspace_bytes(M, N, K, transA, transB, precision) == plan_workspace_bytes(M, N, K, sms)
    case = Case(cuda, M, N, K, transA, transB, seed=M + 3 * N + 7 * K + transA)
    cv = _run_checked(case, precision)
    _assert_tensor_cores_ran(case, cv, precision)


@pytest.mark.parametrize("precision", TC)
@pytest.mark.parametrize("shape", [(1152, 1152, 100_000), (128, 128, 100_000)], ids=["unsplit", "most_splits"])
def test_long_k(cuda, sms, shape, precision):
    """K = 100 000 in the weight-gradient layout (transA): 3 125 k-blocks through the rings of one CTA per tile, and the
    same K over as many splits as the plan allows."""
    M, N, K = shape
    p = plan(M, N, K, sms)
    if M == 1152:
        assert plan(M, N, K, 132).splits == 1 and p.splits == 1
    else:
        assert p.tiles == 1 and p.wanted == sms <= p.kb_total // 4 and p.splits == cdiv(p.kb_total, cdiv(p.kb_total, sms))
    assert workspace_bytes(M, N, K, 1, 0, precision) == plan_workspace_bytes(M, N, K, sms)
    case = Case(cuda, M, N, K, transA=1, transB=0, seed=17)
    _run_checked(case, precision)


# ---------------------------------------------------------------------------------------------------- edges of the tiles
# 7 k-blocks (no split) and 42 / 66 k-blocks on a few tiles (split-K); M·N·K >= 2^18 throughout
EDGE_SHAPES = (
    [(1200, n, 224) for n in (1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 257)]      # BN = 32 / 64 / 128, odd N
    + [(200, n, 1320) for n in (1, 2, 31, 33, 63, 65, 127, 129, 257)]                  # the same through split-K
    + [(m, 1201, 224) for m in (1, 63, 64, 65, 127, 128, 129)]                         # second consumer warpgroup
    + [(m, 129, 2100) for m in (1, 63, 64, 65, 127, 128, 129)]
    + [(257, 131, k) for k in (8, 9, 31, 33, 63, 65)]                                  # K tails, K = 8 alone
)


@pytest.mark.parametrize("precision", TC)
@pytest.mark.parametrize("transA,transB", LAYOUTS)
@pytest.mark.parametrize("shape", EDGE_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_edge_shapes(cuda, shape, transA, transB, precision):
    """Each shape in all four layouts; `out` is aligned, has an odd ldc or starts one float past a 16-byte boundary,
    in turn with the layout, so that every shape meets the vector and the scalar stores."""
    M, N, K = shape
    out = OUTS[LAYOUTS.index((transA, transB)) % 3]
    case = Case(cuda, M, N, K, transA, transB, seed=M * 7 + N * 3 + K + 1000 * transA + 2000 * transB)
    cv = _run_checked(case, precision, out)
    _assert_tensor_cores_ran(case, cv, precision, out)


# ---------------------------------------------------------------------------------------------------- epilogue
EPILOGUE_SHAPES = {"unsplit": (333, 257, 200, "odd_ldc"), "split": (200, 129, 1000, "offset")}


@pytest.mark.parametrize("precision", ["fp32"] + TC)
@pytest.mark.parametrize("accumulate", [False, True], ids=["store", "accumulate"])
@pytest.mark.parametrize("mask", [False, True], ids=["nomask", "mask"])
@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("bias", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("shape", list(EPILOGUE_SHAPES))
def test_epilogue(cuda, sms, shape, bias, act, mask, accumulate, precision):
    """bias x activation x mask x accumulate, straight from the accumulators (one ragged tile row and column, odd N, odd
    ldc) and through the split-K reduction (odd N, `out` one float past a 16-byte boundary)."""
    M, N, K, out = EPILOGUE_SHAPES[shape]
    assert (plan(M, N, K, sms).splits > 1) == (shape == "split")
    case = Case(cuda, M, N, K, 0, 1, seed=5, bias=bias, act=act, mask=mask, accumulate=accumulate)
    case.check(case.run(precision, out), precision)


# ---------------------------------------------------------------------------------------------------- dispatch
# (M, N, K), storage of A [M, K] and B [K, N], whether the tensor-core kernel takes it
DISPATCH = {
    "K=7_cuda_cores": ((256, 256, 7), {}, False),
    "K=8_tensor_cores": ((256, 256, 8), {}, True),
    "MNK=2^18-1_cuda_cores": ((133, 73, 27), {}, False),
    "MNK=2^18_tensor_cores": ((64, 64, 64), {}, True),
    "A_base_plus_4_bytes_cuda_cores": ((256, 128, 64), {"a_off": 1}, False),
    "B_base_plus_4_bytes_cuda_cores": ((256, 128, 64), {"b_off": 1}, False),
    "lda=65_cuda_cores": ((256, 128, 64), {"lda": 65}, False),
    "ldb=129_cuda_cores": ((256, 128, 64), {"ldb": 129}, False),
    "aligned_lda=64_ldb=128_tensor_cores": ((256, 128, 64), {}, True),
}


@pytest.mark.parametrize("precision", TC)
@pytest.mark.parametrize("case_name", list(DISPATCH))
def test_dispatch_boundary(cuda, case_name, precision):
    """One element either side of each rule that sends a shape to the CUDA-core kernel: K >= 8, M·N·K >= 2^18, 16-byte
    aligned A and B, lda and ldb multiples of 4.  A shape that falls back is bit-identical to precision="fp32"."""
    (M, N, K), storage, tensor_cores = DISPATCH[case_name]
    case = Case(cuda, M, N, K, 0, 0, seed=M + N + K, **storage)
    cv = _run_checked(case, precision, computed_as=precision if tensor_cores else "fp32")
    if tensor_cores:
        _assert_tensor_cores_ran(case, cv, precision)
    else:
        fp32 = case.run("fp32")
        assert torch.equal(cv.bits(), fp32.bits()), f"{case_name}: {precision} differs from the CUDA-core kernel"
