"""The triangle decoder's σ / softplus phase and its Gᵀ stores (gae_tc.cu, gae_tri_tc_kernel), checked in the SASS without a
GPU (see kernel_codegen.py; spills and serialised wgmmas are checked in test_kernel_codegen.py).

In that phase one warp per SM sub-partition works (the four warps of one consumer warpgroup), so its length is its instruction
count.  How the numbers below were counted: `cuobjdump -sass` of the kernel compiled with the library's own flags, one count
per opcode over the whole kernel (predicated instructions included, operand suffixes ignored).  The kernel holds six copies of
the elementwise loop (masked and unmasked tiles, at the first tile and in each of the two unrolled turns), each over a thread's
32 logits of a 64 x 64 warpgroup tile; the MUFU they issue (32 ex2 + 32 rcp + 2 lg2 per 32 logits, the SFU floor of
benchmarks/decoder.py) is all the kernel's MUFU.
- Gᵀ is written with stmatrix .trans (STSM.16.MT88.4): 4 per plane and tile per thread instead of a PRMT and a 32-bit STS
  per column and plane.  No PRMT is left in the kernel.
- The fp16 scale 2^14 of G rides in the reciprocal's argument and the product of the (1 + e) is one FFMA per logit, so the
  FMUL + FADD + FFMA count falls by one per logit in every copy, except at the first logit of each of the two product chains
  (one per lg2), where 1 + e used to share its FADD with the reciprocal's argument and now takes one of its own: at least
  30 per 32 logits and copy.
The counts the kernel had before these changes, per DP, are recorded below (same nvcc, same flags)."""
import collections
import re

import pytest

from kernel_codegen import compiled, needs_cuobjdump

pytestmark = needs_cuobjdump

DPS = (8, 16, 32)
TRI = {dp: f"_ZN2b23gtc17gae_tri_tc_kernelILi{dp}EEEvNS0_6ParamsE" for dp in DPS}
COPIES, LOGITS = 6, 32                                       # elementwise copies, logits per thread and copy
FP32_BEFORE = {8: 1487, 16: 1617, 32: 1685}                  # FMUL + FADD + FFMA with the PRMT / STS Gᵀ path and 1 + e
MUFU_BEFORE = {"EX2": 194, "RCP": 190, "LG2": 12}            # every DP

_OP = re.compile(r"^\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P[T0-9]\s+)?([A-Z][A-Z0-9_]*)((?:\.[A-Z0-9_]+)*)")


def opcodes(dp):
    """Counter of (opcode, suffixes) over the kernel's SASS, e.g. ('MUFU', '.EX2'), ('STSM', '.16.MT88.4')."""
    out = collections.Counter()
    for line in compiled("gae_tc.cu").sass(TRI[dp]).splitlines():
        m = _OP.match(line)
        if m:
            out[(m.group(1), m.group(2))] += 1
    return out


def total(ops, name):
    return sum(n for (op, _), n in ops.items() if op == name)


@pytest.mark.parametrize("dp", DPS)
def test_gt_is_written_with_transposing_stmatrix(dp):
    ops = opcodes(dp)
    stsm = {suffix: n for (op, suffix), n in ops.items() if op == "STSM"}
    # two planes x 4 per tile in each of the three copies that hand Gᵀ over
    assert stsm == {".16.MT88.4": 3 * 2 * 4}, f"DP = {dp}: STSM {stsm}"
    assert total(ops, "PRMT") == 0, f"DP = {dp}: {total(ops, 'PRMT')} PRMT left in the triangle"


@pytest.mark.parametrize("dp", DPS)
def test_mufu_count_unchanged(dp):
    ops = opcodes(dp)
    mufu = {suffix.lstrip("."): n for (op, suffix), n in ops.items() if op == "MUFU"}
    assert mufu == MUFU_BEFORE, f"DP = {dp}: MUFU {mufu}"
    assert sum(mufu.values()) == COPIES * (32 + 32 + 2) * LOGITS // 32


@pytest.mark.parametrize("dp", DPS)
def test_fewer_fp32_instructions_per_logit(dp):
    ops = opcodes(dp)
    fp32 = sum(total(ops, op) for op in ("FMUL", "FADD", "FFMA"))
    saved = FP32_BEFORE[dp] - fp32
    assert saved >= COPIES * (LOGITS - 2), f"DP = {dp}: FMUL + FADD + FFMA {fp32}, {saved} below {FP32_BEFORE[dp]}"
