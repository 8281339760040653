"""ctypes binding of ``libdance_b200.so`` (the C-ABI declared in ``include/dance_b200.h``).

There is no CPU fallback: if the shared library is missing, :func:`lib` raises and tells
the user to run ``python -m dance_b200.build``.  Tensors cross the boundary as raw
device pointers + sizes; the CUDA stream is torch's current stream.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

_LIB_PATH = Path(__file__).resolve().parent / "lib" / "libdance_b200.so"
_lib = None

c_i32, c_i64, c_f32, c_vp, c_sz, c_u32 = C.c_int32, C.c_int64, C.c_float, C.c_void_p, C.c_size_t, C.c_uint32

# name -> (restype, argtypes); mirrors include/dance_b200.h declaration by declaration
_SIGNATURES = {
    "b2_last_error": (C.c_char_p, []),
    "b2_version": (C.c_int, []),
    "b2_set_path": (C.c_int, [C.c_int, C.c_int]),
    "b2_get_path": (C.c_int, [C.c_int]),
    "b2_set_tuning": (C.c_int, [C.c_int, C.c_int]),
    "b2_launch_count": (c_i64, []),
    "b2_device_info": (C.c_int, [C.POINTER(C.c_int)] * 3),
    "b2_spmm_csr_f32": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_i64, c_vp, c_i64, c_i32, c_i32, c_i32, C.c_int, C.c_int, c_vp, c_vp]),
    "b2_spmm_csr_bf16": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_i32, c_i32, c_i32, C.c_int, C.c_int, c_vp, c_vp]),
    "b2_spmm_csr_f16": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_i32, c_i32, c_i32, C.c_int, C.c_int, c_vp, c_vp]),
    "b2_convert_f32_to_x16": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_i64, c_i32, C.c_int, c_vp]),
    "b2_comm_available": (C.c_int, []),
    "b2_comm_version": (C.c_int, []),
    "b2_comm_unique_id": (C.c_int, [c_vp]),
    "b2_comm_init_rank": (C.c_int, [C.POINTER(c_vp), c_vp, C.c_int, C.c_int]),
    "b2_comm_destroy": (C.c_int, [c_vp]),
    "b2_comm_world": (C.c_int, [c_vp]),
    "b2_comm_rank": (C.c_int, [c_vp]),
    "b2_allreduce_sum_f32": (C.c_int, [c_vp, c_vp, c_i64, c_vp]),
    "b2_allgather_f32": (C.c_int, [c_vp, c_vp, c_vp, c_i64, c_vp]),
    "b2_gene_stats_f32": (C.c_int, [c_vp, c_i64, c_i64, c_i32, c_vp, c_vp, c_vp, c_vp]),
    "b2_cell_stats_f32": (C.c_int, [c_vp, c_i64, c_i64, c_i32, c_vp, c_vp, c_vp]),
    "b2_subset_f32": (C.c_int, [c_vp, c_i64, c_vp, c_vp, c_i64, c_i32, c_vp, c_i64, c_vp]),
    "b2_cellwise_mask_u8": (C.c_int, [c_vp, c_i64, c_i64, c_i32, c_f32, c_i32, C.c_int, C.c_int, C.c_uint32, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2_kmeans_workspace_bytes": (c_sz, [c_i32, c_i32]),
    "b2_kmeans_step_f32": (C.c_int, [c_vp, c_i64, c_i32, c_i32, c_vp, c_i32, c_vp, C.c_int, c_vp, c_vp, c_sz, c_vp]),
    "b2_graph_regu_weights_f32": (C.c_int, [c_vp, c_vp, c_vp, c_i32, c_i32, c_vp, c_vp, c_vp]),
    "b2_graph_regu_weights_weighted_f32": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_i32, c_i32, c_vp, c_vp, c_vp]),
    "b2_quantiles_workspace_bytes": (c_sz, []),
    "b2_quantiles_f32": (C.c_int, [c_vp, c_i64, c_i64, c_i32, c_vp, c_i32, c_vp, c_vp, c_sz, c_vp]),
    "b2_col_minmax_workspace_bytes": (c_sz, [c_i32]),
    "b2_col_minmax_f32": (C.c_int, [c_vp, c_i64, c_i64, c_i32, c_vp, c_vp, c_vp, c_vp, c_sz, c_vp]),
    "b2_concat_scaled_workspace_bytes": (c_sz, [c_i32]),
    "b2_concat_scaled_f32": (C.c_int, [c_vp, c_i64, c_i32, c_vp, c_i64, c_i32, c_i64, c_vp, c_vp, c_f32, c_f32, C.c_int, c_vp, c_i64,
                                       c_vp, c_sz, c_vp]),
    "b2_celltype_loss_grad_f32": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_i64, c_i32, c_i32, C.c_int, c_vp, c_vp, c_vp, c_vp]),
    "b2_l1_grad_add_f32": (C.c_int, [c_vp, c_vp, c_i64, c_f32, c_vp, c_vp]),
    "b2_louvain_csr_host": (C.c_int, [c_vp, c_vp, c_vp, c_i32, c_vp, C.POINTER(c_i32), C.POINTER(C.c_double), C.c_int, C.c_double]),
    "b2_csr_transpose_workspace_bytes": (c_sz, [c_i32, c_i32, c_i64]),
    "b2_csr_transpose": (C.c_int, [c_vp, c_vp, c_vp, c_i32, c_i32, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_sz, c_vp]),
    "b2_gemm_workspace_bytes": (c_sz, [C.c_int] * 6),
    "b2_gemm_f32": (C.c_int, [c_vp, c_i64, C.c_int, c_vp, c_i64, C.c_int, c_vp, c_i64, C.c_int, C.c_int, C.c_int,
                              c_vp, C.c_int, c_vp, c_i64, c_f32, C.c_int, c_vp, c_sz, c_vp]),
    "b2_colsum_workspace_bytes": (c_sz, [C.c_int, C.c_int]),
    "b2_colsum_f32": (C.c_int, [c_vp, c_i64, C.c_int, C.c_int, c_vp, c_f32, c_vp, c_sz, c_vp]),
    "b2_mse_sum_loss_grad_f32": (C.c_int, [c_vp, c_vp, c_vp, c_f32, C.c_int, c_vp, c_vp, c_i64, c_vp]),
    "b2_gae_loss_workspace_bytes": (c_sz, [c_i32, c_i32]),
    "b2_gae_loss_grad_f32": (C.c_int, [c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_f32, c_f32, C.c_int,
                                       c_vp, c_vp, c_vp, c_i64, c_vp, c_vp, c_sz, c_vp]),
    "b2_gae_loss_grad_weighted_f32": (C.c_int, [c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i32, c_i32, c_i32,
                                                c_i32, c_f32, c_f32, C.c_int, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp, c_sz, c_vp]),
    "b2_gae_sym_super_blocks": (C.c_int, [c_i32]),
    "b2_gae_loss_grad_sym_f32": (C.c_int, [c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_vp, c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, c_f32, c_f32,
                                           C.c_int, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp, c_sz, c_vp]),
    "b2_gae_loss_grad_sym_weighted_f32": (C.c_int, [c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i32, c_i32,
                                                    c_i32, c_i32, c_i32, c_i32, c_f32, c_f32, C.c_int, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp,
                                                    c_sz, c_vp]),
    "b2_adam_step_f32": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_i64, c_f32, c_f32, c_f32, c_f32, c_f32, c_i32, c_vp]),
    "b2_relu_bwd_f32": (C.c_int, [c_vp, c_vp, c_vp, c_i64, c_vp]),
    "b2_reparam_fwd_f32": (C.c_int, [c_vp, c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_i64, c_i32, c_vp]),
    "b2_reparam_bwd_f32": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_i64, c_i64, c_i32, c_vp]),
    "b2_knn_workspace_bytes": (c_sz, [c_i32, c_i32, c_i32, c_i32]),
    "b2_knn_l2_f32": (C.c_int, [c_vp, c_i64, c_i32, c_i32, c_i32, c_i32, c_i32, C.c_int, c_vp, c_vp, c_vp, c_sz, c_vp]),
    "b2_pairwise_l2_dense_f32": (C.c_int, [c_vp, c_i64, c_i32, c_i32, c_vp, c_i64, c_vp]),
    "b2_knn_graph_workspace_bytes": (c_sz, [c_i32, c_i32]),
    "b2_knn_graph_build": (C.c_int, [c_vp, c_i32, c_i32, c_vp, c_vp, c_vp, c_i64, C.POINTER(c_i64), c_vp, c_sz, c_vp]),
    "b2_knn_graph_weighted_workspace_bytes": (c_sz, [c_i32, c_i32]),
    "b2_knn_graph_weighted_build": (C.c_int, [c_vp, c_vp, c_i32, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64,
                                              C.POINTER(c_i64), c_vp, c_sz, c_vp]),
    "b2_gat_scores_f32": (C.c_int, [c_vp, c_i64, c_vp, c_vp, c_i32, c_i32, c_i32, c_vp, c_vp, c_vp]),
    "b2_gat_edge_max_f32": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_i32, c_i32, C.c_int, c_f32, c_vp, c_vp]),
    "b2_gat_aggregate_fwd_f32": (C.c_int, [c_vp, c_vp, c_vp, c_i64, c_vp, c_vp, c_i32, c_i32, c_i32, C.c_int, c_f32, C.c_int,
                                           c_vp, c_vp, c_i64, c_vp, c_vp]),
    "b2_gat_aggregate_bwd_f32": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64,
                                           c_i32, c_i32, c_i32, C.c_int, c_f32, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp,
                                           c_vp, c_vp]),
    "b2_gat_aggregate_bwd_tied_f32": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64,
                                                c_vp, c_i64, c_vp, c_i64, c_i32, c_i32, c_i32, C.c_int, c_f32, c_vp, c_vp, c_i64, c_vp,
                                                c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2_gat_combine_fwd_f32": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_i32, c_i32, c_i32, C.c_int, C.c_int, c_vp, c_i64, c_vp]),
    "b2_gat_combine_bwd_f32": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_i32, c_i32, c_i32, C.c_int, C.c_int, c_vp, c_i64, c_vp, c_i64,
                                         c_vp]),
    "b2_gat_combine_fwd_identity_f32": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_i32, c_i32, c_i32, C.c_int, C.c_int, c_vp, c_i64,
                                                  c_vp]),
    "b2_gat_combine_bwd_identity_f32": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_i32, c_i32, c_i32, C.c_int, C.c_int, c_vp, c_i64, c_vp,
                                                  c_i64, c_vp, c_i64, c_vp]),
    "b2_dropout_f32": (C.c_int, [c_vp, c_i64, c_i64, c_i32, c_f32, c_u32, c_u32, c_vp, c_i64, c_vp]),
    "b2_gat_aggregate_fwd_drop_f32": (C.c_int, [c_vp, c_vp, c_vp, c_i64, c_vp, c_vp, c_i32, c_i32, c_i32, C.c_int, c_f32, C.c_int,
                                                c_vp, c_vp, c_i64, c_vp, c_f32, c_u32, c_u32, c_vp]),
    "b2_gat_aggregate_bwd_drop_f32": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64,
                                                c_i32, c_i32, c_i32, C.c_int, c_f32, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp,
                                                c_vp, c_f32, c_u32, c_u32, c_vp]),
    "b2_cellgene_graph_workspace_bytes": (c_sz, [c_i32, c_i32]),
    "b2_cellgene_graph_count": (C.c_int, [c_vp, c_i64, c_i32, c_i32, C.POINTER(c_i64), c_vp, c_sz, c_vp]),
    "b2_cellgene_graph_fill": (C.c_int, [c_vp, c_i64, c_i32, c_i32, C.c_int, c_i64, c_vp, c_vp, c_vp, c_vp, c_sz, c_vp]),
    "b2_sage_edge_values_f32": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_i32, c_i32, c_vp, c_vp]),
    "b2_softmax_ce_sum_f32": (C.c_int, [c_vp, c_i64, c_vp, c_i32, c_i32, c_vp, c_i64, c_vp, c_vp]),
    "b2_sym_eig_jacobi_f32": (C.c_int, [c_vp, c_vp, c_i32, c_i32, c_f32, c_vp, C.POINTER(c_i32), c_vp, c_sz, c_vp]),
    "b2_cov_rank1_sub_f32": (C.c_int, [c_vp, c_vp, c_i32, c_f32, c_vp]),
    "b2_row_center_f32": (C.c_int, [c_vp, c_i64, c_i32, c_i32, c_vp, c_i64, c_vp]),
    "b2_dec_q_f32": (C.c_int, [c_vp, c_i64, c_vp, c_i32, c_i32, c_i32, c_f32, c_vp, c_i64, c_vp]),
    "b2_dec_target_f32": (C.c_int, [c_vp, c_i64, c_vp, c_i32, c_i32, c_vp, c_i64, c_vp]),
    "b2_dec_kl_grad_f32": (C.c_int, [c_vp, c_i64, c_vp, c_vp, c_i64, c_i32, c_i32, c_i32, c_f32, c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp]),
    "b2_matrix_normalize_workspace_bytes": (c_sz, [c_i32, c_i32, C.c_int]),
    "b2_matrix_normalize_f32": (C.c_int, [c_vp, c_i64, c_i32, c_i32, C.c_int, C.c_int, c_f32, c_vp, c_i64, c_vp, c_sz, c_vp]),
    "b2_pearson_corr_workspace_bytes": (c_sz, [c_i32]),
    "b2_pearson_corr_f32": (C.c_int, [c_vp, c_i64, c_i32, c_i32, c_vp, c_i64, c_vp, c_sz, c_vp]),
    "b2_threshold_graph_workspace_bytes": (c_sz, [c_i32]),
    "b2_threshold_graph_count": (C.c_int, [c_vp, c_i64, c_i32, c_f32, C.c_int, c_vp, c_vp, c_vp, c_sz, c_vp]),
    "b2_threshold_graph_fill": (C.c_int, [c_vp, c_i64, c_i32, c_f32, C.c_int, c_vp, C.c_int, c_vp, c_vp, c_vp, c_vp, c_sz, c_vp]),
    "b2_umap_fuzzy_knn_f32": (C.c_int, [c_vp, c_vp, c_i32, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "b2_fuzzy_union_workspace_bytes": (c_sz, [c_i32]),
    "b2_fuzzy_union_count": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i32, c_vp, c_vp, c_vp, c_sz, c_vp]),
    "b2_fuzzy_union_fill": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i32, c_vp, c_vp, c_vp, c_vp]),
    "b2_batchnorm_workspace_bytes": (c_sz, [c_i32]),
    "b2_batchnorm_fwd_f32": (C.c_int, [c_vp, c_i64, c_i32, c_i32, c_vp, c_vp, c_vp, c_vp, C.c_int, c_f32, c_f32, C.c_int, c_vp, c_i64,
                                       c_vp, c_vp, c_vp, c_sz, c_vp]),
    "b2_batchnorm_bwd_f32": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_vp, c_i64, c_i32, c_i32, c_vp, c_vp, c_vp, C.c_int, C.c_int, c_vp,
                                       c_i64, c_vp, c_vp, c_vp, c_sz, c_vp]),
    "b2_zinb_loss_grad_f32": (C.c_int, [c_vp, c_vp, c_vp, c_i64, c_vp, c_i64, c_vp, c_vp, c_i64, c_i32, c_i32, c_f32, c_f32, c_vp, c_vp,
                                        c_vp, c_i64, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp]),
    "b2_adj_sample_f32": (C.c_int, [c_vp, c_vp, c_vp, c_i64, c_vp, c_vp]),
    "b2_adj_loss_grad_f32": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_i32, c_f32, c_vp, c_vp, c_vp]),
    "b2_adj_reparam_bwd_f32": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_i64, c_f32, c_vp, c_vp, c_vp]),
    "b2_clip_grad_norm_f32": (C.c_int, [c_vp, c_i64, c_f32, c_f32, c_vp, c_vp, c_vp]),
    "b2_radius_graph_workspace_bytes": (c_sz, [c_i32]),
    "b2_radius_graph_count": (C.c_int, [c_vp, c_i64, c_i32, c_i32, C.c_double, c_vp, c_vp, c_vp, c_sz, c_vp]),
    "b2_radius_graph_fill": (C.c_int, [c_vp, c_i64, c_i32, c_i32, C.c_double, c_vp, c_vp, c_vp]),
    "b2_sgd_momentum_step_f32": (C.c_int, [c_vp, c_vp, c_vp, c_i64, c_f32, c_f32, c_f32, c_i32, c_vp]),
    "b2_exp_adj_f32": (C.c_int, [c_vp, c_vp, c_i64, C.c_double, c_vp, c_vp]),
    "b2_normalize_total_workspace_bytes": (c_sz, [c_i32, c_i32]),
    "b2_normalize_total_log1p_f32": (C.c_int, [c_vp, c_i64, c_i32, c_i32, c_f32, c_f32, C.c_int, C.c_int, c_f32, c_vp,
                                               c_sz, c_vp]),
}


class B2Error(RuntimeError):
    """A C-ABI call returned a negative status."""


def lib_path() -> Path:
    return _LIB_PATH


def declared_symbols():
    return sorted(_SIGNATURES)


def lib():
    """Return the loaded shared library (loads it on first use; no fallback if absent)."""
    global _lib
    if _lib is None:
        if not _LIB_PATH.exists():
            raise B2Error(f"{_LIB_PATH} not found: build the CUDA extension first with "
                          "`python -m dance_b200.build` (there is no CPU fallback).")
        handle = C.CDLL(str(_LIB_PATH))
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(handle, name)
            fn.restype = res
            fn.argtypes = args
        _lib = handle
        # A/B selector of the decoder kernel for a whole process (read once at load; tests switch paths with ops.set_path):
        #   B2_FORCE_GAE_PATH = cuda | tc
        import os
        forced = os.environ.get("B2_FORCE_GAE_PATH")
        if forced:
            modes = {"auto": 0, "cuda": 1, "tc": 2}
            if forced not in modes:
                raise B2Error(f"B2_FORCE_GAE_PATH={forced!r}: expected one of {sorted(modes)}")
            handle.b2_set_path(0, modes[forced])
    return _lib


def check(status: int, what: str = ""):
    if status != 0:
        msg = lib().b2_last_error().decode("utf-8", "replace")
        raise B2Error(f"{what or 'dance_b200'} failed with status {status}: {msg}")
