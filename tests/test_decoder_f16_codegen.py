"""The fp16-gradient triangle (gae_tri_f16_tc_kernel) in the SASS and the ptxas report, without a GPU (see kernel_codegen.py).

- dZ_I is one commit group of 8 register-A HGMMA.64xNx16 per tile (4 k-steps of [hi·hi | hi·lo] at N = 2·DP and lo·hi at
  N = DP), with no shared-A product in it.
- dZ_J runs on its own warpgroup: per consumer warpgroup's half of a tile, one group of 4 + 4 shared-A HGMMA.64xNx16.
- S keeps the tf32 triangle's product (3·DP/8 HGMMA.64x64x8 tf32); each batch ends in one WARPGROUP.DEPBAR, the turn is passed
  (BAR.ARV) before S is waited for, and dZ_I is waited for alone (DEPBAR 0x1) while S still runs.
- No stack frame or spills, no serialised wgmmas, and the descriptors in uniform registers."""
import re

import pytest

from kernel_codegen import compiled, needs_cuobjdump

pytestmark = needs_cuobjdump

DPS = (8, 16, 32)
F16 = {dp: f"_ZN2b23gtc21gae_tri_f16_tc_kernelILi{dp}EEEvNS0_6ParamsE" for dp in DPS}
_HGMMA = re.compile(r"\bHGMMA\.64x(\d+)x(8|16)\S*\s+R\d+,\s*(gdesc|R\d+)[^;]*?(gsb0)?\s*;")
_EVENT = re.compile(r"\bHGMMA\.64x\d+x8\S*[^;]*?(gsb0)\s*;|\bWARPGROUP\.DEPBAR\.LE gsb0, (0x\d+)|\b(BAR\.ARV)\b")


def groups(code):
    """commit groups in code order: lists of (N, K, A from registers)"""
    out, cur = [], []
    for m in _HGMMA.finditer(code):
        cur.append((int(m.group(1)), int(m.group(2)), m.group(3) != "gdesc"))
        if m.group(4):
            out.append(cur)
            cur = []
    assert not cur, "HGMMAs after the last gsb0"
    return out


@pytest.mark.parametrize("dp", DPS)
def test_f16_triangle_gradient_groups(dp):
    gs = groups(compiled("gae_tc.cu").sass(F16[dp]))
    s = [g for g in gs if g == [(64, 8, False)] * (3 * dp // 8)]
    dzi = [g for g in gs if any(reg for *_, reg in g)]
    dzj = [g for g in gs if g not in s and g not in dzi]
    assert len(s) >= 2 and len(dzi) >= 2 and len(dzj) >= 2, (len(s), len(dzi), len(dzj))
    for g in dzi:
        assert sorted(g) == sorted([(dp, 16, True)] * 4 + [(2 * dp, 16, True)] * 4), f"DP = {dp}: dZ_I group {g}"
    for g in dzj:
        assert sorted(g) == sorted([(dp, 16, False)] * 4 + [(2 * dp, 16, False)] * 4), f"DP = {dp}: dZ_J group {g}"


@pytest.mark.parametrize("dp", DPS)
def test_f16_triangle_turn_and_waits(dp):
    code = compiled("gae_tc.cu").sass(F16[dp])
    hgmma = len(re.findall(r"\bHGMMA\.", code))
    depbar = len(re.findall(r"\bWARPGROUP\.DEPBAR\b", code))
    assert depbar * 6 <= hgmma, f"DP = {dp}: {depbar} WARPGROUP.DEPBAR for {hgmma} HGMMA"
    ev = [m.group(0) for m in _EVENT.finditer(code)]
    s_ends = [k for k, e in enumerate(ev) if e.startswith("HGMMA")]
    assert s_ends, f"DP = {dp}: no S batch"
    for k in s_ends:
        nxt = next(e for e in ev[k + 1:] if e == "BAR.ARV" or e.startswith("WARPGROUP"))
        assert nxt == "BAR.ARV", f"DP = {dp}: S waited for before the turn is passed"
    assert "WARPGROUP.DEPBAR.LE gsb0, 0x1" in ev, f"DP = {dp}: dZ_I not waited for alone while S runs"


@pytest.mark.parametrize("dp", DPS)
def test_f16_triangle_registers(dp):
    c = compiled("gae_tc.cu")
    assert c.frame(F16[dp]) == (0, 0, 0), f"DP = {dp}: stack frame / spills {c.frame(F16[dp])}"
    assert not c.serialised(F16[dp]), c.serialised(F16[dp])
    code = c.sass(F16[dp])
    assert 4 * len(re.findall(r"\bR2UR\b", code)) <= len(re.findall(r"\bHGMMA\.", code)), f"DP = {dp}: descriptors moved"
