"""The Leiden kernels (csrc/leiden.cu) compile for sm_90a without a stack frame or spills."""
from kernel_codegen import compiled, needs_nvcc


@needs_nvcc
def test_leiden_kernels_spill_nothing():
    c = compiled("leiden.cu")
    names = c.kernels("ld_")
    assert len(names) >= 20
    for name in names:
        assert c.frame(name) == (0, 0, 0), name
