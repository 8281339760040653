"""The order in which the decoder's warpgroups issue, wait and hand the tensor cores over (gae_tc.cu), checked in the SASS
without a GPU.

Triangle (gae_tri_tc_kernel), every instantiation: a warpgroup passes its turn (BAR.ARV) as soon as its S batch is committed,
before the WARPGROUP.DEPBAR that waits for that S, so that the other warpgroup's dZ batch queues behind it.
Triangle at DP = 8, where S is double-buffered: within a turn the dZ batch of the previous tile and the S batch of the next one
go out with no WARPGROUP.DEPBAR between them, and dZ is waited for alone (DEPBAR.LE gsb0, 0x1) while S still runs.
Full sweep (gae_allpairs_tc_kernel): its HGMMA / DEPBAR / BAR sequence is the one pinned in
tests/golden/gae_allpairs_sync_order.json (the schedule the triangle's changes leave alone)."""
import json
import re
import shutil
import subprocess
from pathlib import Path

import pytest

from dance_b200.build import CSRC, NVCC_FLAGS, PKG

NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CUOBJDUMP = str(Path(NVCC).with_name("cuobjdump"))
GOLDEN = Path(__file__).resolve().parent / "golden" / "gae_allpairs_sync_order.json"
TRI = {dp: f"_ZN2b23gtc17gae_tri_tc_kernelILi{dp}EEEvNS0_6ParamsE" for dp in (8, 16, 32)}
ALLPAIRS = {dp: f"_ZN2b23gtc22gae_allpairs_tc_kernelILi{dp}EEEvNS0_6ParamsE" for dp in (8, 16, 32)}
OVERLAP_DP = (8,)             # instantiations with the double-buffered S
S_N = 64                      # the triangle's S product is m64n64k8

pytestmark = pytest.mark.skipif(not (Path(NVCC).exists() and Path(CUOBJDUMP).exists()), reason="needs nvcc and cuobjdump")

_EVENT = re.compile(r"\b(HGMMA\.64x(\d+)x8\S*)[^;]*?(gsb0)?\s*;|\b(WARPGROUP\.DEPBAR\.LE) gsb0, (0x\d+)|\b(BAR\.SYNC|BAR\.ARV)\b")


def sync_events(sass: str):
    """The kernel's HGMMA, WARPGROUP.DEPBAR and named-barrier instructions in code order, as short strings:
    'HGMMA.64xNx8... [gsb0]', 'DEPBAR 0xK', 'BAR.SYNC', 'BAR.ARV'."""
    out = []
    for line in sass.splitlines():
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


@pytest.fixture(scope="module")
def sass(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("gae_overlap")
    obj = tmp / "gae_tc.o"
    cmd = [NVCC, *NVCC_FLAGS, "-I", str(PKG.parent / "include"), "-c", str(CSRC / "gae_tc.cu"), "-o", str(obj)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr

    def get(name):
        return subprocess.run([CUOBJDUMP, "-sass", "-fun", name, str(obj)], capture_output=True, text=True, check=True).stdout
    return get


@pytest.mark.parametrize("dp", sorted(TRI))
def test_triangle_passes_the_turn_before_waiting_for_s(sass, dp):
    ev = sync_events(sass(TRI[dp]))
    s_ends = [last for _, last in s_batches(ev, dp)]
    assert s_ends, f"no S batch (HGMMA.64x{S_N}x8) in the triangle, DP = {dp}"
    for k in s_ends:
        nxt = next(e for e in ev[k + 1:] if e == "BAR.ARV" or e.startswith("DEPBAR"))
        assert nxt == "BAR.ARV", f"DP = {dp}: the S batch ending at event {k} is waited for before the turn is passed: {ev[k:k + 4]}"


@pytest.mark.parametrize("dp", OVERLAP_DP)
def test_triangle_dz_and_s_in_flight_together(sass, dp):
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


@pytest.mark.parametrize("dp", sorted(ALLPAIRS))
def test_full_sweep_schedule_unchanged(sass, dp):
    pinned = json.loads(GOLDEN.read_text())[str(dp)]
    assert sync_events(sass(ALLPAIRS[dp])) == pinned
