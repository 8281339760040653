"""The order in which the tensor-core decoder's warpgroups issue, wait and hand the tensor cores over (gae_tc.cu), checked in
the SASS without a GPU (see kernel_codegen.py; spills and serialised wgmmas are checked in test_kernel_codegen.py).

Triangle (gae_tri_tc_kernel), every instantiation:
- Each S and dZ batch ends in one WARPGROUP.DEPBAR, not one per HGMMA.
- A warpgroup passes its turn (BAR.ARV) as soon as its S batch is committed, before the WARPGROUP.DEPBAR that waits for that
  S, so that the other warpgroup's dZ batch queues behind it.
- S is double-buffered: within a turn the dZ batch of the previous tile and the S batch of the next one go out with no
  WARPGROUP.DEPBAR between them, and dZ is waited for alone (DEPBAR.LE gsb0, 0x1) while S still runs.
- The dZ_J products run on a warpgroup of their own.  dZ_J += Gᵀ·Z_I reads both operands from shared memory (HGMMA.64xDPx8 /
  64x(2·DP)x8 with a descriptor A), while the consumer warpgroups' dZ_I += G·Z_J takes A = G from registers.  So no commit
  group that holds a dZ_I product may hold a shared-A product, and the dZ_J products form groups of their own: 2·8 HGMMAs per
  consumer warpgroup's half of a tile, both halves written out.  The dZ_J warpgroup sets its register count with setmaxnreg
  like the producer, and the four warpgroups fit the register file.
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
S_N = 64                      # the triangle's S product is m64n64k8

_EVENT = re.compile(r"\b(HGMMA\.64x(\d+)x8\S*)[^;]*?(gsb0)?\s*;|\b(WARPGROUP\.DEPBAR\.LE) gsb0, (0x\d+)|\b(BAR\.SYNC|BAR\.ARV)\b")
_HGMMA = re.compile(r"\bHGMMA\.64x(\d+)x8\S*\s+R\d+,\s*(gdesc|R\d+)[^;]*?(gsb0)?\s*;")


def sass(name):
    return compiled("gae_tc.cu").sass(name)


def sync_events(code: str):
    """The kernel's HGMMA, WARPGROUP.DEPBAR and named-barrier instructions in code order, as short strings:
    'HGMMA.64xNx8... [gsb0]', 'DEPBAR 0xK', 'BAR.SYNC', 'BAR.ARV'."""
    out = []
    for line in code.splitlines():
        m = _EVENT.search(line)
        if not m:
            continue
        if m.group(1):
            out.append(m.group(1) + (" gsb0" if m.group(3) else ""))
        elif m.group(4):
            out.append(f"DEPBAR {m.group(5)}")
        else:
            out.append(m.group(6))
    return out


def hgmma_n(ev: str):
    m = re.match(r"HGMMA\.64x(\d+)x8", ev)
    return int(m.group(1)) if m else None


def s_batches(ev, dp):
    """(first, last) event index of every S batch: 3·DP/8 HGMMA.64x64x8 ending in gsb0 (a dZ batch is 32 HGMMAs)"""
    out, first = [], None
    for k, e in enumerate(ev):
        if hgmma_n(e) is None:
            continue
        if first is None:
            first = k
        if e.endswith("gsb0"):
            run = [x for x in ev[first:k + 1] if hgmma_n(x) is not None]
            if len(run) == 3 * dp // 8 and all(hgmma_n(x) == S_N for x in run):
                out.append((first, k))
            first = None
    return out


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


@pytest.mark.parametrize("dp", DPS)
def test_triangle_waits_once_per_batch(dp):
    """S (3·DP/8 HGMMAs) and dZ_I + dZ_J (2·8 + 2·8) each end in one wait, not one per HGMMA."""
    code = sass(TRI[dp])
    hgmma = len(re.findall(r"\bHGMMA\.", code))
    depbar = len(re.findall(r"\bWARPGROUP\.DEPBAR\b", code))
    assert hgmma >= 2 * (3 * dp // 8 + 32), f"expected the S and dZ batches in the SASS, found {hgmma} HGMMA"
    assert depbar * 8 <= hgmma, f"{depbar} WARPGROUP.DEPBAR for {hgmma} HGMMA"


@pytest.mark.parametrize("dp", DPS)
def test_triangle_passes_the_turn_before_waiting_for_s(dp):
    ev = sync_events(sass(TRI[dp]))
    s_ends = [last for _, last in s_batches(ev, dp)]
    assert s_ends, f"no S batch (HGMMA.64x{S_N}x8) in the triangle, DP = {dp}"
    for k in s_ends:
        nxt = next(e for e in ev[k + 1:] if e == "BAR.ARV" or e.startswith("DEPBAR"))
        assert nxt == "BAR.ARV", f"DP = {dp}: the S batch ending at event {k} is waited for before the turn is passed: {ev[k:k + 4]}"


@pytest.mark.parametrize("dp", DPS)
def test_triangle_dz_and_s_in_flight_together(dp):
    ev = sync_events(sass(TRI[dp]))
    assert "DEPBAR 0x1" in ev, f"DP = {dp}: no WARPGROUP.DEPBAR.LE gsb0, 0x1 (dZ waited for while S runs)"
    # every S batch issued in the same turn as a dZ batch (no BAR between them) follows it with no DEPBAR in between
    in_turn = 0
    for k, _ in s_batches(ev, dp):
        j = k - 1
        while j >= 0 and hgmma_n(ev[j]) is None and not ev[j].startswith("BAR."):
            j -= 1
        if j >= 0 and hgmma_n(ev[j]) is not None:
            assert not any(x.startswith("DEPBAR") for x in ev[j + 1:k]), f"DP = {dp}: DEPBAR between dZ and S: {ev[j:k + 1]}"
            in_turn += 1
    assert in_turn >= 2, f"DP = {dp}: expected the two unrolled turns to issue dZ and S back to back, found {in_turn}"


@pytest.mark.parametrize("dp", DPS)
def test_consumer_batches_hold_no_dzj_product(dp):
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


@pytest.mark.parametrize("dp", DPS)
def test_dzj_warpgroup_sets_its_registers(dp):
    code = sass(TRI[dp])
    dealloc = [int(x, 16) for x in re.findall(r"USETMAXREG\.DEALLOC\.CTAPOOL (0x[0-9a-f]+)", code)]
    alloc = [int(x, 16) for x in re.findall(r"USETMAXREG\.TRY_ALLOC\.CTAPOOL \S+ (0x[0-9a-f]+)", code)]
    assert len(dealloc) == 2, f"DP = {dp}: expected setmaxnreg.dec in the producer and the dZ_J warpgroup, found {dealloc}"
    assert len(set(alloc)) == 1, f"DP = {dp}: expected one consumer register count, found {alloc}"
    assert 128 * (sum(dealloc) + 2 * alloc[0]) <= 65536, f"DP = {dp}: {dealloc} + 2 x {alloc[0]} registers exceed the SM"


@pytest.mark.parametrize("dp", DPS)
def test_triangle_descriptors_stay_in_uniform_registers(dp):
    code = sass(TRI[dp])
    hgmma = len(re.findall(r"\bHGMMA\.", code))
    r2ur = len(re.findall(r"\bR2UR\b", code))
    assert hgmma >= 2 * (3 * dp // 8 + 32), f"DP = {dp}: expected the S and dZ batches in the SASS, found {hgmma} HGMMA"
    assert 4 * r2ur <= hgmma, f"DP = {dp}: {r2ur} R2UR for {hgmma} HGMMA (descriptors moved from ordinary registers)"


def test_decoder_dp16_waits_once_per_batch():
    """Full sweep: one wait per batch (S: 6 HGMMAs, dZ: 48) instead of one per HGMMA."""
    code = sass(ALLPAIRS[16])
    hgmma = len(re.findall(r"\bHGMMA\.", code))
    depbar = len(re.findall(r"\bWARPGROUP\.DEPBAR\b", code))
    assert hgmma >= 54, f"expected the S and dZ batches in the SASS, found {hgmma} HGMMA"
    assert depbar * 8 <= hgmma, f"{depbar} WARPGROUP.DEPBAR for {hgmma} HGMMA"


@pytest.mark.parametrize("dp", DPS)
def test_full_sweep_schedule_unchanged(dp):
    pinned = json.loads(GOLDEN.read_text())[str(dp)]
    assert sync_events(sass(ALLPAIRS[dp])) == pinned
