"""The triangle sweep (gae_tri_tc_kernel in gae_tc.cu) runs its dZ_J products on a warpgroup of their own, checked in the SASS
without a GPU.

dZ_J += Gᵀ·Z_I reads both operands from shared memory (HGMMA.64xDPx8 / 64x(2·DP)x8 with a descriptor A), while the consumer
warpgroups' dZ_I += G·Z_J takes A = G from registers.  So no commit group that holds a dZ_I product may hold a shared-A product,
and the dZ_J products form groups of their own: 2·8 HGMMAs per consumer warpgroup's half of a tile, both halves written out.
The dZ_J warpgroup sets its register count with setmaxnreg like the producer, and the four warpgroups fit the register file."""
import re

import pytest

from test_decoder_triangle_overlap_codegen import TRI, sass  # noqa: F401  (sass: the compiled-kernel fixture)
from test_decoder_triangle_overlap_codegen import pytestmark  # noqa: F401  (needs nvcc and cuobjdump)
from test_decoder_triangle_overlap_codegen import test_triangle_dz_and_s_in_flight_together as _in_flight

_HGMMA = re.compile(r"\bHGMMA\.64x(\d+)x8\S*\s+R\d+,\s*(gdesc|R\d+)[^;]*?(gsb0)?\s*;")


def commit_groups(code: str):
    """HGMMAs in code order, cut after each one that closes a commit group (gsb0): lists of (N, A from registers)."""
    groups, cur = [], []
    for m in _HGMMA.finditer(code):
        cur.append((int(m.group(1)), m.group(2) != "gdesc"))
        if m.group(3):
            groups.append(cur)
            cur = []
    assert not cur, "HGMMAs after the last gsb0"
    return groups


@pytest.mark.parametrize("dp", sorted(TRI))
def test_consumer_batches_hold_no_dzj_product(sass, dp):  # noqa: F811
    groups = commit_groups(sass(TRI[dp]))
    dzi = [g for g in groups if any(reg for _, reg in g)]
    assert dzi, f"DP = {dp}: no dZ_I batch (register-A HGMMA)"
    for g in dzi:
        assert all(reg for _, reg in g), f"DP = {dp}: a dZ_I batch also holds shared-A products: {g}"
        assert len(g) == 16, f"DP = {dp}: dZ_I batch of {len(g)} HGMMAs, expected 2·8"
    s = [g for g in groups if g == [(64, False)] * (3 * dp // 8)]
    dzj = [g for g in groups if g not in dzi and g not in s]
    assert len(dzj) >= 2, f"DP = {dp}: expected both halves of the dZ_J product written out, found {len(dzj)} groups"
    for g in dzj:
        assert sorted(g) == sorted([(dp, False)] * 8 + [(2 * dp, False)] * 8), f"DP = {dp}: unexpected dZ_J group {g}"


@pytest.mark.parametrize("dp", sorted(TRI))
def test_dzj_warpgroup_sets_its_registers(sass, dp):  # noqa: F811
    code = sass(TRI[dp])
    dealloc = [int(x, 16) for x in re.findall(r"USETMAXREG\.DEALLOC\.CTAPOOL (0x[0-9a-f]+)", code)]
    alloc = [int(x, 16) for x in re.findall(r"USETMAXREG\.TRY_ALLOC\.CTAPOOL \S+ (0x[0-9a-f]+)", code)]
    assert len(dealloc) == 2, f"DP = {dp}: expected setmaxnreg.dec in the producer and the dZ_J warpgroup, found {dealloc}"
    assert len(set(alloc)) == 1, f"DP = {dp}: expected one consumer register count, found {alloc}"
    assert 128 * (sum(dealloc) + 2 * alloc[0]) <= 65536, f"DP = {dp}: {dealloc} + 2 x {alloc[0]} registers exceed the SM"


@pytest.mark.parametrize("dp", (16, 32))
def test_triangle_double_buffers_s_at_every_dp(sass, dp):  # noqa: F811
    """With the dZ_J accumulators gone from the consumers, DP = 16 and 32 also keep dZ_I and the next S in flight together."""
    _in_flight(sass, dp)
