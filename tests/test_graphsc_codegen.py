"""The graph-sc kernels (csrc/graphsc.cu) compile for sm_90a without a stack frame or spills."""
import pytest

from kernel_codegen import compiled, needs_nvcc

KERNELS = ("block_degrees_kernel", "block_aggregate_kernel", "batch_decoder_kernel", "scatter_rows_kernel")


@needs_nvcc
@pytest.mark.parametrize("kernel", KERNELS)
def test_graphsc_kernels_spill_nothing(kernel):
    c = compiled("graphsc.cu")
    for name in c.kernels(kernel):
        assert c.frame(name) == (0, 0, 0), name
