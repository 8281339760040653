"""The order in which the tensor-core decoder's warpgroups issue, wait and hand the tensor cores over (gae_tc.cu), checked in
the SASS without a GPU (see kernel_codegen.py; spills and serialised wgmmas are checked in test_kernel_codegen.py).

Triangle (gae_tri_tc_kernel), every instantiation:
- S keeps the tf32 product (3·DP/8 HGMMA.64x64x8); the gradient products are fp16 k16.  Each S and dZ batch ends in one
  WARPGROUP.DEPBAR, not one per HGMMA: at most 9 in the whole kernel.
- A warpgroup passes its turn (BAR.ARV) as soon as its S batch is committed, before the WARPGROUP.DEPBAR that waits for that
  S, so that the other warpgroup's dZ batch queues behind it.
- S is double-buffered: within a turn the dZ batch of the previous tile and the S batch of the next one go out with no
  WARPGROUP.DEPBAR between them, and dZ is waited for alone (DEPBAR.LE gsb0, 0x1) while S still runs.
- The dZ_J products run on a warpgroup of their own.  dZ_I += G·Z_J takes A = G from registers: one commit group per tile of
  4 HGMMA.64x(2·DP)x16 ([hi·hi | hi·lo]) and 4 HGMMA.64xDPx16 (lo·hi), with no shared-A product in it.  dZ_J += Gᵀ·Z_I reads
  both operands from shared memory: per consumer warpgroup's half of a tile, one group of the same 4 + 4 shapes with a
  descriptor A, both halves written out.  The dZ_J warpgroup sets its register count with setmaxnreg like the producer, and
  the four warpgroups fit the register file.
- The wgmma descriptors stay in uniform registers.  The per-warpgroup operands (Gᵀ, Z_Iᵀ, the warpgroup's rows of Z_I) sit
  at addresses derived from the warpgroup index; when ptxas cannot tell that index is the same across a warp, it keeps the
  descriptors in ordinary registers and copies them with R2URs before the HGMMAs, which costs consumer registers and issue
  slots in every turn.  The kernel broadcasts the index from lane 0, so only a handful of
  R2UR remain.
Full sweep (gae_allpairs_tc_kernel): its HGMMA / DEPBAR / BAR sequence is the one pinned in
tests/golden/gae_allpairs_sync_order.json (the schedule the triangle's changes leave alone)."""
import json
import re
from pathlib import Path

import pytest

from kernel_codegen import compiled, needs_cuobjdump

pytestmark = needs_cuobjdump

GOLDEN = Path(__file__).resolve().parent / "golden" / "gae_allpairs_sync_order.json"
DPS = (8, 16, 32)
TRI = {dp: f"_ZN2b23gtc17gae_tri_tc_kernelILi{dp}EEEvNS0_6ParamsE" for dp in DPS}
ALLPAIRS = {dp: f"_ZN2b23gtc22gae_allpairs_tc_kernelILi{dp}EEEvNS0_6ParamsE" for dp in DPS}
S_NK = (64, 8)                # the triangle's S product is m64n64k8

_EVENT = re.compile(r"\b(HGMMA\.64x\d+x(?:8|16)\S*)[^;]*?(gsb0)?\s*;|\b(WARPGROUP\.DEPBAR\.LE) gsb0, (0x\d+)|\b(BAR\.SYNC|BAR\.ARV)\b")
_HGMMA = re.compile(r"\bHGMMA\.64x(\d+)x(8|16)\S*\s+R\d+,\s*(gdesc|R\d+)[^;]*?(gsb0)?\s*;")


def sass(name):
    return compiled("gae_tc.cu").sass(name)


def sync_events(code: str):
    """The kernel's HGMMA, WARPGROUP.DEPBAR and named-barrier instructions in code order, as short strings:
    'HGMMA.64xNxK... [gsb0]', 'DEPBAR 0xK', 'BAR.SYNC', 'BAR.ARV'."""
    out = []
    for line in code.splitlines():
        m = _EVENT.search(line)
        if not m:
            continue
        if m.group(1):
            out.append(m.group(1) + (" gsb0" if m.group(2) else ""))
        elif m.group(3):
            out.append(f"DEPBAR {m.group(4)}")
        else:
            out.append(m.group(5))
    return out


def hgmma_nk(ev: str):
    """(N, K) of an HGMMA event, None for any other"""
    m = re.match(r"HGMMA\.64x(\d+)x(\d+)", ev)
    return (int(m.group(1)), int(m.group(2))) if m else None


def s_batches(ev, dp):
    """(first, last) event index of every S batch: 3·DP/8 HGMMA.64x64x8 ending in gsb0 (a dZ batch is 8 k16 HGMMAs)"""
    out, first = [], None
    for k, e in enumerate(ev):
        if hgmma_nk(e) is None:
            continue
        if first is None:
            first = k
        if e.endswith("gsb0"):
            run = [x for x in ev[first:k + 1] if hgmma_nk(x) is not None]
            if len(run) == 3 * dp // 8 and all(hgmma_nk(x) == S_NK for x in run):
                out.append((first, k))
            first = None
    return out


def commit_groups(code: str):
    """HGMMAs in code order, cut after each one that closes a commit group (gsb0): lists of (N, K, A from registers)."""
    groups, cur = [], []
    for m in _HGMMA.finditer(code):
        cur.append((int(m.group(1)), int(m.group(2)), m.group(3) != "gdesc"))
        if m.group(4):
            groups.append(cur)
            cur = []
    assert not cur, "HGMMAs after the last gsb0"
    return groups


def _count(pattern, code):
    return len(re.findall(pattern, code))


@pytest.mark.parametrize("dp", DPS)
def test_triangle_waits_at_most_nine_times(dp):
    """S (3·DP/8 HGMMAs), dZ_I (8) and each half of dZ_J (8) end in one wait each, not one per HGMMA."""
    code = sass(TRI[dp])
    hgmma, depbar = _count(r"\bHGMMA\.", code), _count(r"\bWARPGROUP\.DEPBAR\b", code)
    assert hgmma >= 2 * (3 * dp // 8 + 16), f"expected the S and dZ batches in the SASS, found {hgmma} HGMMA"
    assert depbar <= 9, f"DP = {dp}: {depbar} WARPGROUP.DEPBAR for {hgmma} HGMMA"


@pytest.mark.parametrize("dp", DPS)
def test_triangle_passes_the_turn_before_waiting_for_s(dp):
    ev = sync_events(sass(TRI[dp]))
    s_ends = [last for _, last in s_batches(ev, dp)]
    assert s_ends, f"no S batch (HGMMA.64x{S_NK[0]}x{S_NK[1]}) in the triangle, DP = {dp}"
    for k in s_ends:
        nxt = next(e for e in ev[k + 1:] if e == "BAR.ARV" or e.startswith("DEPBAR"))
        assert nxt == "BAR.ARV", f"DP = {dp}: the S batch ending at event {k} is waited for before the turn is passed: {ev[k:k + 4]}"


@pytest.mark.parametrize("dp", DPS)
def test_triangle_fp16_dz_and_s_in_flight_together(dp):
    ev = sync_events(sass(TRI[dp]))
    assert "DEPBAR 0x1" in ev, f"DP = {dp}: no WARPGROUP.DEPBAR.LE gsb0, 0x1 (dZ waited for while S runs)"
    # every S batch issued in the same turn as a dZ batch (no BAR between them) follows it with no DEPBAR in between
    in_turn = 0
    for k, _ in s_batches(ev, dp):
        j = k - 1
        while j >= 0 and hgmma_nk(ev[j]) is None and not ev[j].startswith("BAR."):
            j -= 1
        if j >= 0 and hgmma_nk(ev[j]) is not None:
            assert not any(x.startswith("DEPBAR") for x in ev[j + 1:k]), f"DP = {dp}: DEPBAR between dZ and S: {ev[j:k + 1]}"
            in_turn += 1
    assert in_turn >= 2, f"DP = {dp}: expected the two unrolled turns to issue dZ and S back to back, found {in_turn}"


@pytest.mark.parametrize("dp", DPS)
def test_triangle_fp16_gradient_groups(dp):
    groups = commit_groups(sass(TRI[dp]))
    s = [g for g in groups if g == [(*S_NK, False)] * (3 * dp // 8)]
    dzi = [g for g in groups if any(reg for *_, reg in g)]
    dzj = [g for g in groups if g not in s and g not in dzi]
    assert len(s) >= 2 and len(dzi) >= 2, f"DP = {dp}: {len(s)} S and {len(dzi)} dZ_I (register-A) batches"
    assert len(dzj) >= 2, f"DP = {dp}: expected both halves of the dZ_J product written out, found {len(dzj)} groups"
    for g in dzi:
        assert all(reg for *_, reg in g), f"DP = {dp}: a dZ_I batch also holds shared-A products: {g}"
        assert sorted(g) == sorted([(dp, 16, True)] * 4 + [(2 * dp, 16, True)] * 4), f"DP = {dp}: unexpected dZ_I group {g}"
    for g in dzj:
        assert sorted(g) == sorted([(dp, 16, False)] * 4 + [(2 * dp, 16, False)] * 4), f"DP = {dp}: unexpected dZ_J group {g}"


@pytest.mark.parametrize("dp", DPS)
def test_dzj_warpgroup_sets_its_registers(dp):
    code = sass(TRI[dp])
    dealloc = [int(x, 16) for x in re.findall(r"USETMAXREG\.DEALLOC\.CTAPOOL (0x[0-9a-f]+)", code)]
    alloc = [int(x, 16) for x in re.findall(r"USETMAXREG\.TRY_ALLOC\.CTAPOOL \S+ (0x[0-9a-f]+)", code)]
    assert len(dealloc) == 2, f"DP = {dp}: expected setmaxnreg.dec in the producer and the dZ_J warpgroup, found {dealloc}"
    assert len(set(alloc)) == 1, f"DP = {dp}: expected one consumer register count, found {alloc}"
    assert 128 * (sum(dealloc) + 2 * alloc[0]) <= 65536, f"DP = {dp}: {dealloc} + 2 x {alloc[0]} registers exceed the SM"


@pytest.mark.parametrize("dp", DPS)
def test_triangle_fp16_descriptors_stay_in_uniform_registers(dp):
    code = sass(TRI[dp])
    hgmma, r2ur = _count(r"\bHGMMA\.", code), _count(r"\bR2UR\b", code)
    assert hgmma >= 2 * (3 * dp // 8 + 16), f"DP = {dp}: expected the S and dZ batches in the SASS, found {hgmma} HGMMA"
    assert 4 * r2ur <= hgmma, f"DP = {dp}: {r2ur} R2UR for {hgmma} HGMMA (descriptors moved from ordinary registers)"


def test_decoder_dp16_waits_once_per_batch():
    """Full sweep: one wait per batch (S: 6 HGMMAs, dZ: 48) instead of one per HGMMA."""
    code = sass(ALLPAIRS[16])
    hgmma, depbar = _count(r"\bHGMMA\.", code), _count(r"\bWARPGROUP\.DEPBAR\b", code)
    assert hgmma >= 54, f"expected the S and dZ batches in the SASS, found {hgmma} HGMMA"
    assert depbar * 8 <= hgmma, f"{depbar} WARPGROUP.DEPBAR for {hgmma} HGMMA"


@pytest.mark.parametrize("dp", DPS)
def test_full_sweep_schedule_unchanged(dp):
    pinned = json.loads(GOLDEN.read_text())[str(dp)]
    assert sync_events(sass(ALLPAIRS[dp])) == pinned
