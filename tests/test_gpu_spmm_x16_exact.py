"""The row-group aggregate builds the same fmaf chain per output feature, in CSR order, whatever the operand's element type and
the lane layout (G lanes per row, VPL 16-byte vectors per lane).  So a bf16 / fp16 operand must give exactly the result of the
same values stored as fp32, although the two run different (G, VPL) instantiations, and the 16-bit copy of the result must be
the fp32 result rounded to nearest even."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

pytestmark = pytest.mark.gpu


def _graph(n_rows, n_cols, seed):
    rng = np.random.default_rng(seed)
    deg = rng.integers(0, 40, n_rows)
    deg[[3, 4, 5, n_rows - 1]] = 0          # empty rows, one at the end
    deg[7] = 3000                            # hub row: many full G-entry chunks after the prefetched ones
    rows = np.repeat(np.arange(n_rows), deg)
    cols = np.concatenate([rng.choice(n_cols, d, replace=False) for d in deg])
    m = sp.csr_matrix((rng.normal(size=rows.size).astype(np.float32), (rows, cols)), shape=(n_rows, n_cols))
    m.sort_indices()
    return m


# 16-bit G = 4 (F = 8 … 32), 8, 16, 32; the fp32 copies run G = 4 … 32 with VPL = 1 and G = 32 with VPL = 2
@pytest.mark.parametrize("F", [8, 16, 24, 32, 48, 64, 104, 128, 192, 256])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_rowgroup_16bit_operand_equals_fp32_operand_bit_for_bit(cuda, F, dtype):
    from dance_b200 import ops
    m = _graph(600, 4000, seed=F)
    X16 = ops.to_x16(torch.randn(4000, F, device=cuda), dtype)
    X32 = X16.float()
    bias = torch.randn(F, device=cuda)
    graphs = {"weighted": ops.CSR.from_scipy(m, cuda), "unit": ops.CSR.from_scipy(m, cuda, with_values=False)}
    try:
        ops.set_path("spmm", "rowgroup")
        for gname, A in graphs.items():
            for reduce in ("sum", "mean"):
                for act in (None, "relu", "elu", "tanh"):
                    for b in (None, bias):
                        what = f"{gname} {reduce} act={act} bias={b is not None}"
                        Y32 = ops.spmm(A, X32, reduce=reduce, act=act, bias=b)
                        out16 = torch.empty(600, F, dtype=dtype, device=cuda)
                        Y = ops.spmm(A, X16, reduce=reduce, act=act, bias=b, out=torch.empty_like(Y32), out16=out16)
                        assert torch.equal(Y, Y32), what
                        assert torch.equal(out16, Y.to(dtype)), what
    finally:
        ops.set_path("spmm", "auto")
