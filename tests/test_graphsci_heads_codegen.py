"""The fused GraphSCI heads kernels and the BatchNorm statistics kernels (csrc/graphsci.cu) compile for sm_90a without a
stack frame or local-memory spills."""
from kernel_codegen import compiled, needs_nvcc


@needs_nvcc
def test_graphsci_heads_kernels_spill_nothing():
    c = compiled("graphsci.cu")
    names = c.kernels("heads_train_kernel") + c.kernels("heads_eval_kernel") + c.kernels("bn_stats_kernel") + c.kernels("bn_finalize_kernel")
    assert len(names) == 5
    for name in names:
        assert c.frame(name) == (0, 0, 0), name
