"""The large-k kNN kernels (csrc/knn.cu) and the warp-per-cell UMAP smoothing kernel (csrc/umap.cu) compile for sm_90a without a
stack frame or spills."""
from kernel_codegen import compiled, needs_nvcc


@needs_nvcc
def test_large_k_kernels_spill_nothing():
    names = compiled("knn.cu").kernels("knn_lk_")
    assert len(names) == 4
    for name in names:
        assert compiled("knn.cu").frame(name) == (0, 0, 0), name
    warp = compiled("umap.cu").kernels("um_smooth_warp_kernel")
    assert len(warp) == 1 and compiled("umap.cu").frame(warp[0]) == (0, 0, 0)
