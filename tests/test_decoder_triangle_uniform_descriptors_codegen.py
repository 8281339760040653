"""The triangle sweep (gae_tri_tc_kernel in gae_tc.cu) keeps its wgmma descriptors in uniform registers, checked in the SASS
without a GPU.

An HGMMA takes its shared-memory descriptors from uniform registers.  The triangle's per-warpgroup operands (Gᵀ, Z_Iᵀ, and
the warpgroup's rows of Z_I) sit at addresses derived from the warpgroup index; when ptxas cannot tell that index is the same
across a warp, it keeps the descriptors in ordinary registers and copies them with an R2UR before each HGMMA (about two per
HGMMA at every DP), which costs consumer registers and issue slots in every turn.  The kernel broadcasts the index from lane 0,
so only a handful of R2UR remain."""
import re

import pytest

from test_decoder_triangle_overlap_codegen import TRI, sass  # noqa: F401  (sass: the compiled-kernel fixture)
from test_decoder_triangle_overlap_codegen import pytestmark  # noqa: F401  (needs nvcc and cuobjdump)


@pytest.mark.parametrize("dp", sorted(TRI))
def test_triangle_descriptors_stay_in_uniform_registers(sass, dp):  # noqa: F811
    code = sass(TRI[dp])
    hgmma = len(re.findall(r"\bHGMMA\.", code))
    r2ur = len(re.findall(r"\bR2UR\b", code))
    assert hgmma >= 2 * (3 * dp // 8 + 32), f"DP = {dp}: expected the S and dZ batches in the SASS, found {hgmma} HGMMA"
    assert 4 * r2ur <= hgmma, f"DP = {dp}: {r2ur} R2UR for {hgmma} HGMMA (descriptors moved from ordinary registers)"
