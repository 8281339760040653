/*
 * dance_b200 — C-ABI of the H100-native (sm_90a) GNN message-passing hot path.
 *
 * This header is the drop-in boundary (SURVEY.md §8b.4).  The reference
 * (OmicsML/dance) has no FFI of its own: its hot path bottoms out in calls
 * into torch / DGL / PyG / scanpy / scipy kernels.  Every entry point below
 * names the reference call site(s) it replaces (paths relative to the
 * reference repository root).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in `_host`;
 *   - the library never allocates or frees caller-visible memory: scratch is
 *     passed in, sized by the matching `*_workspace_bytes` query;
 *   - `stream` is a `cudaStream_t` passed as `void*`; work is enqueued on it
 *     and the call returns without synchronising (unless documented);
 *   - return value 0 = success, negative = error; `b2_last_error()` returns
 *     a thread-local human-readable message for the last failing call;
 *   - matrices are row-major with an explicit leading dimension (in elements);
 *   - index types: CSR `rowptr`/`colidx` are int32 (nnz < 2^31).
 */
#ifndef DANCE_B200_H_
#define DANCE_B200_H_

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2_OK 0
#define B2_ERR_INVALID (-1)
#define B2_ERR_CUDA (-2)
#define B2_ERR_UNSUPPORTED (-3)
#define B2_ERR_WORKSPACE (-4)

/* activation codes shared by GEMM / SpMM epilogues (NONE..TANH); LEAKY_RELU and GELU are taken by b2_act_f32 / b2_act_bwd_f32
 * only (graph-sc's activations, graphsc.py:324-331) */
#define B2_ACT_NONE 0
#define B2_ACT_RELU 1
#define B2_ACT_ELU 2
#define B2_ACT_TANH 3
#define B2_ACT_LEAKY_RELU 4 /* F.leaky_relu, negative slope 0.01 */
#define B2_ACT_GELU 5       /* F.gelu, exact (erf) form */

/* GEMM precision modes */
#define B2_PREC_FP32_SIMT 0 /* CUDA-core FFMA, exact fp32 accumulate            */
#define B2_PREC_TF32X3 1    /* wgmma tf32, 3-product split, ~fp32 accuracy      */
#define B2_PREC_TF32 2      /* wgmma tf32, single product                        */
#define B2_PREC_BF16 3      /* wgmma bf16 (operands rounded RNE), fp32 accumulate */

/* Kernel-path selectors for A/B tests: every selectable path returns the same result (bit-exact for the kNN filter, to
 * rounding for the decoder); mode 0 = automatic choice by problem size. */
#define B2_PATH_GAE_DECODER 0 /* 1 CUDA cores · 2 tensor cores (S in wgmma tf32, 3-product split; the call over all rows takes
                                 its gradient products in fp16 hi / lo with a power-of-two scale per tile) */
#define B2_PATH_KNN_FILTER 1  /* 1 SIMT candidate filter */
#define B2_PATH_SPMM 2        /* 1 row-per-lane-group kernels for every shape (default: the nnz-stream kernel where it applies) */
#define B2_PATH_COUNT 3
int b2_set_path(int which, int mode);
int b2_get_path(int which);
/* Scheduling knob of the tensor-core decoder (timing experiments; results do not depend on it beyond summation order). */
#define B2_TUNE_GAE_SPLITS 0      /* step ranges (CTAs) per 128-row block of the decoder's J sweep (0 = automatic: fill a wave of SMs) */
#define B2_TUNE_COUNT 1
int b2_set_tuning(int which, int value);

const char* b2_last_error(void);
int b2_version(void);
/* Number of CUDA kernels this library has launched in the calling process (bench.py's `gpu_launches`). */
int64_t b2_launch_count(void);
/* Fills SM count and compute capability of the current device. */
int b2_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ------------------------------------------------------------------------
 * K1/K2  CSR SpMM  Y[n_rows,F] = act( reduce(A · X) + bias )
 * replaces: torch.spmm(adj, support)      scgnn2.py:500, spagcn.py:359,
 *           scdsc.py:498; DGL update_all(u_mul_e, sum|mean)  gnn.py:90,
 *           graphsc.py:463-465.
 *   vals      : nnz edge weights, or NULL for an unweighted (0/1) graph
 *   reduce    : 0 = sum, 1 = mean over the row's nnz (0 for empty rows)
 *   act       : B2_ACT_* applied to the output row
 *   F must be a multiple of 4; X/Y rows and bias must be 16-byte aligned.
 *   F > 512 returns B2_ERR_UNSUPPORTED.
 * ---------------------------------------------------------------------- */
int b2_spmm_csr_f32(const int32_t* rowptr, const int32_t* colidx, const float* vals,
                    const float* X, int64_t ldx, float* Y, int64_t ldy,
                    int32_t n_rows, int32_t n_cols, int32_t F,
                    int reduce, int act, const float* bias /* length F or NULL, added before act */, void* stream);

/* The same aggregate with a 16-bit dense operand (bf16 / fp16 storage, fp32 accumulation) — the reduced-precision
 * configurations (BASELINE config 3 "GraphSCI … bf16"; dglnn.GraphConv under autocast, graphsci.py:112-115) and the
 * bandwidth-optimised form of torch.spmm(adj, support) scgnn2.py:500: every non-zero gathers F·2 instead of F·4 bytes.
 *   X       : [n_cols, F] bf16 / fp16, leading dimension ldx (elements), rows 16-byte aligned, F % 8 == 0, F <= 256
 *   Y       : fp32 output or NULL;  Y16 : output in the operand's 16-bit type (round-to-nearest-even) or NULL (feeds the next
 *             layer's aggregate without a conversion pass); at least one of the two, rows 16-byte aligned.
 *   bias    : length F or NULL, 4-byte alignment suffices. */
int b2_spmm_csr_bf16(const int32_t* rowptr, const int32_t* colidx, const float* vals,
                     const void* X, int64_t ldx, float* Y, int64_t ldy, void* Y16, int64_t ldy16,
                     int32_t n_rows, int32_t n_cols, int32_t F, int reduce, int act, const float* bias, void* stream);
int b2_spmm_csr_f16(const int32_t* rowptr, const int32_t* colidx, const float* vals,
                    const void* X, int64_t ldx, float* Y, int64_t ldy, void* Y16, int64_t ldy16,
                    int32_t n_rows, int32_t n_cols, int32_t F, int reduce, int act, const float* bias, void* stream);
/* fp32 [rows, cols] -> bf16 (dtype 0) / fp16 (dtype 1), round-to-nearest-even; replaces tensor.to(torch.bfloat16). */
int b2_convert_f32_to_x16(const float* src, int64_t lds, void* dst, int64_t ldd, int64_t rows, int32_t cols, int dtype, void* stream);

/* CSR transpose (deterministic: entries of each output row ordered by source
 * row).  Used to obtain Aᵀ for the SpMM backward of non-symmetric graphs
 * (GAT edge lists, cell→gene / gene→cell halves of CellFeatureGraph).
 * perm_out (optional, nnz int32): position of each transposed entry in the
 * source arrays, so per-edge data can be permuted the same way. */
size_t b2_csr_transpose_workspace_bytes(int32_t n_rows, int32_t n_cols, int64_t nnz);
int b2_csr_transpose(const int32_t* rowptr, const int32_t* colidx, const float* vals,
                     int32_t n_rows, int32_t n_cols, int64_t nnz,
                     int32_t* t_rowptr, int32_t* t_colidx, float* t_vals, int32_t* perm_out,
                     void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------
 * K5  dense projection GEMM with fused epilogue
 *     C[M,N] = act( op(A)[M,K] · op(B)[K,N] + bias[N] ) ⊙ (mask > 0 ? 1 : 0)
 * replaces: torch.mm / nn.Linear   scgnn2.py:352-355,364-370,499;
 *           spagcn.py:358; gnn.py:57; scdeepsort.py:81; graphsci.py:41,73,81
 *   transA = 0: A is [M,K] row-major (lda ≥ K); 1: A is stored [K,M] (lda ≥ M)
 *   transB = 0: B is [K,N] row-major (ldb ≥ N); 1: B is stored [N,K] (ldb ≥ K)
 *            (nn.Linear weight [out,in] is the transB = 1 case)
 *   bias   : length N or NULL
 *   mask   : optional [M,N] (ldmask) — output is zeroed where mask <= 0
 *            (ReLU backward fused into the dX GEMM)
 *   beta   : 0 overwrite, 1 accumulate into C (weight-gradient accumulation)
 *   colsum : optional length-N output, += column sums of the epilogue result
 *            is NOT provided here; see b2_colsum_f32.
 *   precision: B2_PREC_*.  A, B, C, bias and mask are fp32 in every mode; the mode
 *            bounds how the operands are rounded for the tensor cores (BF16:
 *            round-to-nearest-even to bfloat16, fp32 accumulate).  Shapes the
 *            tensor-core kernel does not take (K < 8, M·N·K < 2^18, a base not
 *            16-byte aligned or a row pitch not a multiple of 4 elements) run on
 *            the CUDA-core fp32 kernel in every mode.
 * ---------------------------------------------------------------------- */
size_t b2_gemm_workspace_bytes(int M, int N, int K, int transA, int transB, int precision);
int b2_gemm_f32(const float* A, int64_t lda, int transA,
                const float* B, int64_t ldb, int transB,
                float* C, int64_t ldc, int M, int N, int K,
                const float* bias, int act,
                const float* mask, int64_t ldmask,
                float beta, int precision,
                void* workspace, size_t workspace_bytes, void* stream);

/* column sums: out[N] = (beta ? out : 0) + Σ_rows X[M,N]   (bias gradients) */
size_t b2_colsum_workspace_bytes(int M, int N);
int b2_colsum_f32(const float* X, int64_t ldx, int M, int N, float* out, float beta,
                  void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------
 * Losses (forward value + gradient w.r.t. the prediction, one pass)
 * ---------------------------------------------------------------------- */
/* Feature-AE reconstruction loss: loss_function_graph, scgnn2.py:1298-1328
 *   regularizer "LTMG"  :  (1-s)·Σ(r-x)² + s·Σ (r-x)²·T    (T = LTMG_regu; NULL = all zeros)
 *   regularizer "noregu":  Σ (r-x)²                       (pass s = 0)
 * loss_out[0] += value (per-block fp64 partial sums, fp32 running total);
 * grad = d loss / d recon, additionally masked by recon>0 when relu_mask!=0
 * (the decoder's final ReLU, scgnn2.py:362). */
int b2_mse_sum_loss_grad_f32(const float* recon, const float* target, const float* ltmg_regu,
                             float regu_strength, int relu_mask,
                             float* grad, float* loss_out, int64_t n_elem, void* stream);

/* Graph-AE loss, exact and matrix-free: gae_loss_function, scgnn2.py:603-615
 * with InnerProductDecoder scgnn2.py:423-426 (logits = z zᵀ never stored).
 *   cost = norm · mean_{ij} BCEwithLogits(z_i·z_j, L_ij, pos_weight=L_ij·pw)
 *   L = A + I given as CSR (rowptr/colidx, unit entries; diagonal included)
 *   lab_vals = NULL : unit labels; L must be symmetric (it always is: scgnn2.py:658-664) and labt_* are ignored.
 *   lab_vals set    : real-valued, asymmetric labels y (graph_AE_retain_weights, scgnn2.py:555-569): lab_* are the local
 *     rows of L (entries (i, j), values y_ij, diagonal included), labt_* (all three required) the local rows of Lᵀ (row i
 *     holds the j with (j, i) in L, values y_ji), n_rows+1 row pointers, global column ids.  Per entry
 *     ℓ = (1−y)·softplus(x) + y²·pw·softplus(−x) (pos_weight = labels·pw); use_pos_weight = 0: ℓ = softplus(x) − y·x.
 *   KLD  = -0.5/n · mean_i Σ_d (1 + 2·logvar - mu² - exp(logvar)²)
 *   loss_out[0] = cost + KLD ; dz [n,d] dense, dmu/dlogvar [n,d] with leading
 *   dimension ldd are OVERWRITTEN with d loss / d z (decoder part) and the KLD
 *   parts respectively.
 *   Row sharding (cell-sharded multi-GPU): z holds all n rows; this call handles rows
 *   [row_begin, row_begin+n_rows): lab_rowptr has n_rows+1 entries (global column ids),
 *   mu/logvar/dz/dmu/dlogvar are the n_rows local rows, and loss_out receives this
 *   shard's additive share of the loss (constants use the global n).
 *   mu/logvar may be NULL (plain GAE: cost only).
 *   When use_pos_weight == 0 computes loss_function (scgnn2.py:618-619):
 *   plain mean BCE (GAT branch), norm ignored.
 *   d ∈ {8, 16, 32, 64}; any other d returns B2_ERR_UNSUPPORTED. */
size_t b2_gae_loss_workspace_bytes(int32_t n, int32_t d);
int b2_gae_loss_grad_f32(const float* z, int64_t ldz, const float* mu, const float* logvar, int64_t ldm,
                         const int32_t* lab_rowptr, const int32_t* lab_colidx, const float* lab_vals,
                         const int32_t* labt_rowptr, const int32_t* labt_colidx, const float* labt_vals,
                         int32_t n, int32_t d, int32_t row_begin, int32_t n_rows,
                         float norm, float pos_weight, int use_pos_weight,
                         float* dz, float* dmu, float* dlogvar, int64_t ldd, float* loss_out,
                         void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------
 * Optimiser: torch.optim.Adam semantics (scgnn2.py:301,573; default eps 1e-8,
 * betas (0.9,0.999), no amsgrad, L2 weight_decay added to grad).
 * `step` is the 1-based step count AFTER this update.
 * ---------------------------------------------------------------------- */
int b2_adam_step_f32(float* param, const float* grad, float* exp_avg, float* exp_avg_sq,
                     int64_t n, float lr, float beta1, float beta2, float eps,
                     float weight_decay, int32_t step, void* stream);
/* torch.nn.utils.clip_grad_norm_ on one flat gradient bucket (stagate.py:221):
 *   g ← pre_scale·g ; total = ||g||₂ ; g ← g·min(1, max_norm/(total+1e-6))   (max_norm <= 0: scale only)
 * sumsq_ws: one device double of scratch; norm_out (device, optional) receives the total norm. */
int b2_clip_grad_norm_f32(float* grad, int64_t n, float pre_scale, float max_norm, double* sumsq_ws,
                          float* norm_out, void* stream);

/* ------------------------------------------------------------------------
 * Elementwise helpers on the GCN path
 * ---------------------------------------------------------------------- */
/* Standalone activations over strided [rows, cols] matrices, for every B2_ACT_* code (the activations the GEMM / SpMM
 * epilogues do not take, and the backward of those they do):
 *   b2_act_f32     : y = act(x); in place allowed.
 *   b2_act_bwd_f32 : dx = dy ⊙ act'(·): from the output y for relu / elu / tanh / leaky_relu, from the pre-activation x for
 *       gelu (the other may be NULL; NONE reads neither and copies dy); in place allowed.  relu is torch's threshold_backward,
 *       dx = y > 0 ? dy : 0, so dx is +0 wherever y <= 0 whatever dy is.  The backward of the activation of the GCN layers
 *       (GraphConvolution, scgnn2.py:497-502; dgl's GraphConv), of nn.ReLU / nn.Tanh in GraphSCI (graphsci.py:37-45,
 *       68-87,111-112), of F.elu in STAGATE (stagate.py:191,197) and of graph-sc's activations (graphsc.py:324-331). */
int b2_act_f32(const float* x, int64_t ldx, int64_t rows, int32_t cols, int act, float* y, int64_t ldy, void* stream);
int b2_act_bwd_f32(const float* dy, int64_t lddy, const float* y, int64_t ldy, const float* x, int64_t ldx, int64_t rows,
                   int32_t cols, int act, float* dx, int64_t lddx, void* stream);
/* z = mu + eps ⊙ exp(logvar)  (Graph_AE.reparameterize, scgnn2.py:394-400); [n,d] with leading dims */
int b2_reparam_fwd_f32(const float* mu, const float* logvar, int64_t ldm, const float* eps, int64_t lde,
                       float* z, int64_t ldz, int64_t n, int32_t d, void* stream);
/* dmu += dz ; dlogvar += dz ⊙ eps ⊙ exp(logvar) */
int b2_reparam_bwd_f32(const float* dz, int64_t lddz, const float* logvar, int64_t ldm, const float* eps, int64_t lde,
                       float* dmu, float* dlogvar, int64_t ldd, int64_t n, int32_t d, void* stream);

/* ------------------------------------------------------------------------
 * K7  exact k-nearest-neighbour search (euclidean)
 * replaces: calculateKNNgraphDistanceMatrixStatsSingleThread scgnn2.py:675-689
 *           (scipy cdist in fp64 + argsort, ranks 1..k), NeighborGraph
 *           (neighbor_graph.py:50-57), StagateGraph kNN (spatial_graph.py:147-149)
 *   X [n,d] fp32 reference set (queries = rows q_begin..q_end of the same set)
 *   idx_out  [n_q, k] int32 — neighbours sorted by (fp64 distance, index)
 *   dist_out [n_q, k] fp64 euclidean distances (may be NULL)
 *   include_rank0 = 0: drop sorted rank 0 (the reference's "self" slot) and
 *   return ranks 1..k; 1: return ranks 0..k-1.
 *   Distances are ranked in fp64 exactly like the reference; ties broken by
 *   the smaller index.
 *   Limits: 1 <= k, k + r0 <= n (r0 = 0 with include_rank0, else 1), any d.
 *   k + r0 + 8 <= 64 keeps per-query candidate lists; larger k runs a batched
 *   path (tf32x3 GEMM estimate in [bq, n] blocks of at most 2 GiB, radix
 *   select, fp64 refine) that synchronises the stream once per batch.
 *   b2_knn_workspace_bytes gives what either path needs.
 * ---------------------------------------------------------------------- */
size_t b2_knn_workspace_bytes(int32_t n, int32_t d, int32_t k, int32_t n_queries);
int b2_knn_l2_f32(const float* X, int64_t ldx, int32_t n, int32_t d, int32_t k,
                  int32_t q_begin, int32_t q_end, int include_rank0,
                  int32_t* idx_out, double* dist_out,
                  void* workspace, size_t workspace_bytes, void* stream);

/* Dense pairwise euclidean distance matrix, fp32 (small N only)
 * replaces: dance.utils.matrix.pairwise_distance (utils/matrix.py:164-180) */
int b2_pairwise_l2_dense_f32(const float* X, int64_t ldx, int32_t n, int32_t d,
                             float* D, int64_t ldd, void* stream);

/* ------------------------------------------------------------------------
 * Graph assembly for scGNN: feature2adj (scgnn2.py:650-672, union-symmetrise,
 * drop diagonal) + preprocess_graph (scgnn2.py:1191-1198,  Â = D^-1/2 (A+I) D^-1/2)
 *   knn_idx [n,k] → CSR of (A ∪ Aᵀ) + I with sorted columns.
 *   Two-phase: `count` returns nnz (host int64), then `fill` writes arrays.
 *   vals_norm : Â values;  the same rowptr/colidx serve as the label matrix
 *   L = A + I for b2_gae_loss_grad_f32.  Σ A (no diagonal) = nnz - n.
 * ---------------------------------------------------------------------- */
size_t b2_knn_graph_workspace_bytes(int32_t n, int32_t k);
int b2_knn_graph_build(const int32_t* knn_idx, int32_t n, int32_t k,
                       int32_t* rowptr /* n+1 */, int32_t* colidx /* cap */, float* vals_norm /* cap */,
                       int64_t capacity, int64_t* nnz_out_host,
                       void* workspace, size_t workspace_bytes, void* stream);

/* Weighted, directed kNN graph: feature2adj(retain_weights=True) (scgnn2.py:659-670) + preprocess_graph (scgnn2.py:1191-1198).
 *   knn_idx [n,k] int32 (distinct neighbours per row), knn_dist [n,k] fp64 → W[i,j] = 1/(d_ij + 1e-16) in fp64, directed, no
 *   clamping (a zero distance gives 1e16).  adj_train = W without its diagonal (a row listing itself drops that slot).
 *   L = adj_train + I with sorted columns, in two orientations of nnz entries each (capacity >= n·(k+1)):
 *     rowptr/colidx  : rows = source i;  y = float32(L[i,j]) (the decoder labels),  norm_t = Âᵀ[i,j]
 *     t_rowptr/...   : rows = target j;  t_y = float32(L[i,j]) at (j, i),            norm   = Â[j,i]
 *   Â[i,j] = adj_[j,i]·r_i^-1/2·r_j^-1/2 with adj_ = adj_train + I and r = rowsum(adj_) (the out-weight + 1), the products in
 *   fp64 in the reference's order ((adj_·Dm)ᵀ·Dm), cast to fp32.  (Lᵀ rows, norm) is the CSR of Â for the forward aggregate,
 *   (L rows, norm_t) the CSR of Âᵀ for the backward.  sum_w: one device double, ΣW = adj_train.sum().  Synchronises the stream;
 *   *nnz_out_host = nnz. */
size_t b2_knn_graph_weighted_workspace_bytes(int32_t n, int32_t k);
int b2_knn_graph_weighted_build(const int32_t* knn_idx, const double* knn_dist, int32_t n, int32_t k,
                                int32_t* rowptr /* n+1 */, int32_t* colidx, float* y, float* norm_t,
                                int32_t* t_rowptr /* n+1 */, int32_t* t_colidx, float* t_y, float* norm,
                                double* sum_w, int64_t capacity, int64_t* nnz_out_host,
                                void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------
 * K9  normalize_total (+ optional log1p), in place on dense X [n,g]
 * replaces: scanpy.pp.normalize_total / log1p via AnnDataTransform
 *           (transforms/interface.py:67-68), NormalizeTotal (normalize.py:569-628),
 *           Log1P (normalize.py:531-564), NormalizeTotalLog1P (:664-679)
 *   target_sum <= 0 → median of the (included-gene) totals over cells with
 *   total > 0 (computed on device; this call then synchronises the stream).
 *   max_fraction < 1 → genes that exceed that fraction of ANY cell's total are
 *   excluded from the totals (scanpy exclude_highly_expressed).
 *   Rows with total == 0 are left unchanged (scanpy ≥1.10.1).
 *   do_log1p: 0 none, 1 natural log1p; base > 0 divides by ln(base).
 * ---------------------------------------------------------------------- */
size_t b2_normalize_total_workspace_bytes(int32_t n, int32_t g);
int b2_normalize_total_log1p_f32(float* X, int64_t ldx, int32_t n, int32_t g,
                                 float target_sum, float max_fraction,
                                 int do_normalize, int do_log1p, float base,
                                 void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------
 * K4  GAT layer (scGNN GATLayer scgnn2.py:989-1215; STAGATE GATConv stagate.py:61-125)
 *   Graph = CSR indexed by TARGET node: row v lists the sources u of its in-edges.
 *   H [n, nheads*F] projected features; s_src/s_trg [n, nheads] dense.
 *   e = score_act(s_src[u] + s_trg[v]); α = softmax over the in-edges of v; out[v] = Σ α·H[u]
 *   score_act : 0 LeakyReLU(slope) (scgnn2.py:1023), 1 sigmoid (stagate.py:119)
 *   shift_mode: 0 subtract the GLOBAL max over all edges/heads (scgnn2.py:1076; value in
 *               gmax_dev[0], produced by b2_gat_edge_max_f32), 1 per-target max (PyG softmax)
 *   alpha_out [nnz, nheads] or NULL (needed by the backward pass).  nheads*F <= 512.
 * ---------------------------------------------------------------------- */
int b2_gat_scores_f32(const float* H, int64_t ldh, const float* a_src, const float* a_trg,
                      int32_t n, int32_t nheads, int32_t F, float* s_src, float* s_trg, void* stream);
int b2_gat_edge_max_f32(const int32_t* rowptr, const int32_t* colidx,
                        const float* s_src, const float* s_trg, int32_t n, int32_t nheads,
                        int score_act, float slope, float* gmax_dev, void* stream);
/* Attention dropout (GATLayer, scgnn2.py:1029: α' = drop(α) after the softmax): drop_p in [0, 1], otherwise an error.
 *   drop_p = 0 is the plain aggregate (seed and key are not read); drop_p > 0 needs nheads <= 32 and drops (edge, head) with
 *   the keep bit of b2_dropout_f32 at r = the edge's position in the target CSR, c = the head.  alpha_out stays the
 *   UNDROPPED α, which is what the backward takes with the same (drop_p, seed, key). */
int b2_gat_aggregate_fwd_f32(const int32_t* rowptr, const int32_t* colidx,
                             const float* H, int64_t ldh, const float* s_src, const float* s_trg,
                             int32_t n, int32_t nheads, int32_t F,
                             int score_act, float slope, int shift_mode, const float* gmax_dev,
                             float* out, int64_t ldo, float* alpha_out,
                             float drop_p, uint32_t seed, uint32_t key, void* stream);
/* Backward of scores + aggregate.  (t_rowptr, t_colidx, t_perm) = b2_csr_transpose of the target
 * CSR.  Outputs: dH [n, nheads*F] (overwritten: message path + score path), da_src/da_trg
 * [nheads*F] (overwritten).  ds_src_ws/ds_trg_ws [n*nheads] and dpre_edge_ws [nnz*nheads] are
 * caller-provided scratch.  nheads <= 32.
 *   gmax_dev : the forward's global shift (shift_mode 0) or NULL (per-target shift, whose max is detached
 *              as in PyG).  The global max is NOT detached in scgnn2.py:1076; since α = p/(Σp + 1e-16) is
 *              shift-invariant only up to the 1e-16, its gradient reaches the argmax score(s) — split evenly
 *              over ties, as torch's max — and matters for targets whose scores lie ~37+ below the max.
 *   shift_ws : [2] caller-provided scratch, needed when gmax_dev is set.
 *   H2       : NULL, or tied attention (STAGATE, stagate.py:197: conv3 reuses conv1's node scores, so the SAME edge
 *              coefficients α weight two layers' messages): the second layer's projected features H2 with its upstream
 *              gradient dOut2 (required):  dα_e = <dOut[v],H[u]> + <dOut2[v],H2[u]> ;  dH2[u] = Σ α dOut2[v] (message path
 *              only — the scores depend on H; pass dH2 = NULL when the caller already has it).  No attention dropout.
 *   drop_p, seed, key : the forward's attention dropout. */
int b2_gat_aggregate_bwd_f32(const int32_t* rowptr, const int32_t* colidx,
                             const int32_t* t_rowptr, const int32_t* t_colidx, const int32_t* t_perm,
                             const float* H, int64_t ldh, const float* a_src, const float* a_trg,
                             const float* s_src, const float* s_trg, const float* alpha,
                             const float* dOut, int64_t lddo, const float* H2, int64_t ldh2,
                             const float* dOut2, int64_t lddo2, int32_t n, int32_t nheads, int32_t F,
                             int score_act, float slope, const float* gmax_dev,
                             float* dH, int64_t lddh, float* dH2, int64_t lddh2, float* da_src, float* da_trg,
                             float* ds_src_ws, float* ds_trg_ws, float* dpre_edge_ws, float* shift_ws,
                             float drop_p, uint32_t seed, uint32_t key, void* stream);
/* skip connection + concat | head-mean + bias + activation (scgnn2.py:1189-1215):
 *   concat: out[n, nheads*F] = act(agg + skip + bias) ; else out[n,F] = act(mean_h(agg + skip) + bias)
 *   skip may be NULL.  identity_skip != 0 (GATLayer with FIN == FOUT, scgnn2.py:1167-1171): skip is the raw input
 *   x [n, F] (required, ldskip >= F), added to every head as skip[n, h*F + f] = x[n, f].
 *   act: B2_ACT_NONE..B2_ACT_TANH.
 *   Backward: dpre [n, nheads*F] = d(agg) = d(skip); dact [n, OW] (optional) is the gradient before the bias add (its column
 *   sums are the bias gradient); dx_skip NULL, or for an identity skip dx_skip[n, F] = Σ_h dpre[n, h*F:(h+1)*F] (overwritten,
 *   ldx >= F). */
int b2_gat_combine_fwd_f32(const float* agg, int64_t ldagg, const float* skip, int64_t ldskip, const float* bias,
                           int32_t n, int32_t nheads, int32_t F, int concat, int act, int identity_skip,
                           float* out, int64_t ldo, void* stream);
int b2_gat_combine_bwd_f32(const float* dout, int64_t lddo, const float* out, int64_t ldo,
                           int32_t n, int32_t nheads, int32_t F, int concat, int act,
                           float* dpre, int64_t ldp, float* dact, int64_t ldact,
                           float* dx_skip, int64_t ldx, void* stream);

/* Dropout (scGNN GATLayer, scgnn2.py:1005 / :1010 / :1029: one nn.Dropout(p) at the input, the projection and the
 * attention coefficients).  Keep bits are counter-based, keep(seed, key, r, c) = uniform01(seed, key, r, c) >= p with the
 * hash of CellwiseMaskData: the masks follow torch's distribution (independent Bernoulli(1 - p), kept values scaled by
 * 1 / (1 - p), p = 1 gives zeros) but are not torch's masks.  The backward regenerates them from the same (seed, key).
 *   b2_dropout_f32 : y[r, c] = keep(r, c) ? x[r, c] / (1 - p) : 0 over a strided [rows, cols] matrix; y may be x.
 *   0 <= p <= 1, otherwise an error.  The attention site is the drop_p of b2_gat_aggregate_fwd_f32 / _bwd_f32. */
int b2_dropout_f32(const float* x, int64_t ldx, int64_t rows, int32_t cols, float p, uint32_t seed, uint32_t key,
                   float* y, int64_t ldy, void* stream);

/* ------------------------------------------------------------------------
 * NeighborGraph connectivities (transforms/graph/neighbor_graph.py:50-57 → scanpy.pp.neighbors(method="umap") →
 * umap fuzzy_simplicial_set; third-party algorithm restated, see csrc/umap.cu)
 *   b2_umap_fuzzy_knn_f32 : knn_idx/knn_dist [n,k] (column 0 = the cell itself, ascending distances, k >= 2; a thread per
 *                           cell for k <= 64, a warp per cell above)
 *                           → membership strengths vals [n,k], sigmas [n], rhos [n]; sum_ws = one device double.
 *   b2_fuzzy_union_*      : C = A + Aᵀ - A∘Aᵀ from A and Aᵀ in CSR with ascending columns (b2_csr_transpose gives both),
 *                           zeros dropped; `count` writes rowptr_out and returns nnz (synchronises), `fill` the rest.
 * ---------------------------------------------------------------------- */
int b2_umap_fuzzy_knn_f32(const int32_t* knn_idx, const float* knn_dist, int32_t n, int32_t k, float* vals,
                          float* sigmas, float* rhos, double* sum_ws, void* stream);
size_t b2_fuzzy_union_workspace_bytes(int32_t n);
int b2_fuzzy_union_count(const int32_t* rowptr_a, const int32_t* colidx_a, const float* vals_a,
                         const int32_t* rowptr_t, const int32_t* colidx_t, const float* vals_t, int32_t n,
                         int32_t* rowptr_out, int64_t* nnz_host, void* workspace, size_t workspace_bytes, void* stream);
int b2_fuzzy_union_fill(const int32_t* rowptr_a, const int32_t* colidx_a, const float* vals_a,
                        const int32_t* rowptr_t, const int32_t* colidx_t, const float* vals_t, int32_t n,
                        const int32_t* rowptr_out, int32_t* colidx_out, float* vals_out, void* stream);

/* ------------------------------------------------------------------------
 * dance.utils.matrix.normalize (utils/matrix.py:8-67), out-of-place, along axis 0 (columns) or 1 (rows):
 *   mode 0 "normalize" x/Σx, 1 "standardize" (x-mean)/std (population), 2 "minmax", 3 "l2" x/sqrt(Σx²)
 *   eps == -1: zero denominators → 1 ; eps > 0: denominator + eps ; anything else is an error (:61).
 * Statistics are accumulated in fp64.  out may alias X.
 * ---------------------------------------------------------------------- */
size_t b2_matrix_normalize_workspace_bytes(int32_t n_rows, int32_t n_cols, int axis);
int b2_matrix_normalize_f32(const float* X, int64_t ldx, int32_t n_rows, int32_t n_cols, int mode, int axis, float eps,
                            float* out, int64_t ldo, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------
 * FeatureFeatureGraph (transforms/graph/feature_feature_graph.py:45-87)
 *   b2_pearson_corr_f32      : adj [g,g] fp32 = float32(np.corrcoef(X.T)) for X [n cells, g genes]; fp64 arithmetic
 *                              (:49), zero-variance genes give NaN rows/columns exactly as numpy does.
 *   b2_threshold_graph_count : keeps entries with NOT(-thr < a < thr) (and a >= 0 if positive_only) that are nonzero
 *                              (:62-69; NaN is kept); writes rowptr [g+1], returns nnz (synchronises).
 *   b2_threshold_graph_fill  : COO edges in row-major order (int32 src/dst, :68-69) and weights: 1, or with
 *                              normalize_edges dgl EdgeWeightNorm("both") = outdeg(src)^-1/2 · indeg(dst)^-1/2 (:75-78).
 *                              Must be given the workspace `count` filled.
 * ---------------------------------------------------------------------- */
size_t b2_pearson_corr_workspace_bytes(int32_t g);
int b2_pearson_corr_f32(const float* X, int64_t ldx, int32_t n, int32_t g, float* adj, int64_t lda,
                        void* workspace, size_t workspace_bytes, void* stream);
size_t b2_threshold_graph_workspace_bytes(int32_t g);
int b2_threshold_graph_count(const float* adj, int64_t lda, int32_t g, float threshold, int positive_only,
                             int32_t* rowptr, int64_t* nnz_host, void* workspace, size_t workspace_bytes, void* stream);
int b2_threshold_graph_fill(const float* adj, int64_t lda, int32_t g, float threshold, int positive_only,
                            const int32_t* rowptr, int normalize_edges, int32_t* src, int32_t* dst, float* w,
                            void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------
 * Radius graph over spot coordinates — StagateGraph(model_name="radius"):
 * NearestNeighbors(radius=r).fit(X).radius_neighbors_graph(X) (transforms/graph/spatial_graph.py:143-151).
 *   X [n, d] fp64 (1 <= d <= 4), A_ij = 1 iff Σ_c (x_ic - x_jc)² <= r² in fp64 (sklearn's reduced-distance test), self
 *   included.  `count` writes rowptr [n+1] and returns nnz (synchronises); `fill` writes colidx [nnz], ascending per row.
 * ---------------------------------------------------------------------- */
size_t b2_radius_graph_workspace_bytes(int32_t n);
int b2_radius_graph_count(const double* X, int64_t ldx, int32_t n, int32_t d, double radius, int32_t* rowptr,
                          int64_t* nnz_host, void* workspace, size_t workspace_bytes, void* stream);
int b2_radius_graph_fill(const double* X, int64_t ldx, int32_t n, int32_t d, double radius, const int32_t* rowptr,
                         int32_t* colidx, void* stream);

/* ------------------------------------------------------------------------
 * K10 CellFeatureGraph (transforms/graph/cell_feature_graph.py:34-79)
 *   dense X [n_cells, n_genes] → COO edge list in the reference's order
 *   [cell→gene ×nnz ; gene→cell ×nnz ; self ×(G+N)] (gene nodes first: ids 0..G-1, cell c = G+c),
 *   int64 src/dst, fp32 w, with the per-destination renormalisation w ← indeg·w/Σ_in w (:62-68)
 *   and unit self loops (:69).  `count` (synchronises) returns nnz; `fill` writes 2·nnz+G+N edges
 *   and must be given the same workspace `count` filled.
 * ---------------------------------------------------------------------- */
size_t b2_cellgene_graph_workspace_bytes(int32_t n_cells, int32_t n_genes);
int b2_cellgene_graph_count(const float* X, int64_t ldx, int32_t n_cells, int32_t n_genes,
                            int64_t* nnz_out_host, void* workspace, size_t workspace_bytes, void* stream);
int b2_cellgene_graph_fill(const float* X, int64_t ldx, int32_t n_cells, int32_t n_genes,
                           int normalize_edges, int64_t nnz, int64_t* src, int64_t* dst, float* w,
                           void* workspace, size_t workspace_bytes, void* stream);
/* AdaptiveSAGE.message_func edge scalars (models/nn/gnn.py:62-82) on a destination-indexed CSR
 * (node ids < n_genes are genes): out[p] = w[p] · alpha[idx(p)].  The mean aggregate (gnn.py:90) is
 * b2_spmm_csr_f32(vals = out, reduce = 1). */
int b2_sage_edge_values_f32(const int32_t* rowptr, const int32_t* colidx, const float* w, const float* alpha,
                            int32_t n_nodes, int32_t n_genes, float* out, void* stream);
/* nn.CrossEntropyLoss(reduction="sum") (scdeepsort.py:185): loss_out[0] += Σ_rows CE ; dlogits = softmax - onehot
 * (dlogits may be NULL for evaluation). */
int b2_softmax_ce_sum_f32(const float* logits, int64_t ld, const int64_t* labels, int32_t n, int32_t c,
                          float* dlogits, int64_t ldd, float* loss_out, void* stream);

/* ------------------------------------------------------------------------
 * K8  PCA building blocks (WeightedFeaturePCA / CellPCA, transforms/cell_feature.py:49-75,168-194;
 *     replaces sklearn.decomposition.PCA).  PCA = eigen-decomposition of the small Gram / covariance matrix
 *     (built with b2_gemm_f32) by a parallel one-sided Jacobi iteration.
 *   b2_sym_eig_jacobi_f32: W [g,g] symmetric (OVERWRITTEN), V [g,g] out: row i of V = eigenvector i,
 *     evals[i] = eigenvalue i (unsorted).  Stops when every |<w_p,w_q>|/(|w_p||w_q|) <= tol or after
 *     max_sweeps; synchronises the stream once per sweep.  workspace: 64 bytes.
 *   b2_cov_rank1_sub_f32: C[i,j] -= n·mean[i]·mean[j]  (XᵀX → centred second moment)
 *   b2_row_center_f32   : out[i,:] = X[i,:] - mean(X[i,:])
 * ---------------------------------------------------------------------- */
int b2_sym_eig_jacobi_f32(float* W, float* V, int32_t g, int32_t max_sweeps, float tol, float* evals,
                          int32_t* sweeps_done_host, void* workspace, size_t workspace_bytes, void* stream);
int b2_cov_rank1_sub_f32(float* C, const float* mean, int32_t g, float n, void* stream);
int b2_row_center_f32(const float* X, int64_t ldx, int32_t n, int32_t g, float* out, int64_t ldo, void* stream);

/* ------------------------------------------------------------------------
 * SpaGCN deep-embedded-clustering head (modules/spatial/spatial_domain/spagcn.py:369-425, K <= 64 clusters)
 *   b2_dec_q_f32       : q_ij = u_ij / Σ_j u_ij, u = ((1 + |z_i-mu_j|²/alpha) + 1e-8)^-(alpha+1) / 2       (:391-397)
 *   b2_dec_target_f32  : p = (q² / colsum(q)) row-normalised                                             (:408-425)
 *   b2_dec_kl_grad_f32 : loss = mean_i Σ_j p log(p/(q+1e-6)) (:399-406) and its gradients dz [n,h], dmu [K,h]
 *                        (both overwritten); q_out and labels_out (= argmax_j q_ij, first maximum, :527) optional.
 *   b2_sgd_momentum_step_f32 : torch.optim.SGD(momentum, weight_decay) as used at spagcn.py:463; step is 1-based.
 *   b2_exp_adj_f32     : out = exp(-D²/(2 l²)) elementwise (spagcn.py:807-809) and/or its total sum in fp64
 *                        (calculate_p / search_l, spagcn.py:249-251).
 * ---------------------------------------------------------------------- */
int b2_dec_q_f32(const float* z, int64_t ldz, const float* mu, int32_t n, int32_t K, int32_t h, float alpha,
                 float* q, int64_t ldq, void* stream);
int b2_dec_target_f32(const float* q, int64_t ldq, const float* colsum, int32_t n, int32_t K, float* p, int64_t ldp, void* stream);
int b2_dec_kl_grad_f32(const float* z, int64_t ldz, const float* mu, const float* p, int64_t ldp, int32_t n, int32_t K, int32_t h,
                       float alpha, float* q_out, int64_t ldq, float* dz, int64_t lddz, float* dmu, float* loss_out,
                       int32_t* labels_out, void* stream);
int b2_sgd_momentum_step_f32(float* param, const float* grad, float* momentum_buf, int64_t n, float lr, float momentum,
                             float weight_decay, int32_t step, void* stream);
int b2_exp_adj_f32(const float* D, float* out, int64_t n_elem, double l, double* sum_out_dev, void* stream);

/* ------------------------------------------------------------------------
 * SpaGCN's spot graph from the coordinates, never forming the N×N matrices.  rows [n_rows, d] and cols [n_cols, d] are
 * contiguous fp32 coordinate sets (1 <= d <= 4); a pair's distance D_rc and weight W_rc = exp(-D_rc²/(2 l²)) are the bits
 * b2_pairwise_l2_dense_f32 and b2_exp_adj_f32 give for the same pair.
 *   b2_spatial_exp_adj_mm_f32  : AX [n_rows, F] = W · X, X [n_cols, F] (tf32x3 tensor cores, ~2^-21 of W·|X|).  Replaces
 *       adj_exp · X of GraphConvolution on calc_adj_exp's matrix (spagcn.py:337-366, 807-809).  Workspace:
 *       b2_spatial_exp_adj_mm_workspace_bytes(n_cols, F), 16-byte aligned.
 *   b2_spatial_exp_adj_sum_f32 : Σ_rc W_rc in fp64 (overwritten) — calculate_p / search_l (spagcn.py:249-287).
 *   b2_spatial_nearest_f32     : idx_out [n_rows, m], 1 <= m <= 8: per row the m columns of smallest fp32 distance, ties to
 *       the lower column index (a stable sort of the row) — the neighbours of refine (spagcn.py:290-334).
 * ---------------------------------------------------------------------- */
size_t b2_spatial_exp_adj_mm_workspace_bytes(int32_t n_cols, int32_t F);
int b2_spatial_exp_adj_mm_f32(const float* rows, int32_t n_rows, const float* cols, int32_t n_cols, int32_t d, double l,
                              const float* X, int64_t ldx, int32_t F, float* AX, int64_t ldax, void* workspace,
                              size_t workspace_bytes, void* stream);
int b2_spatial_exp_adj_sum_f32(const float* rows, int32_t n_rows, const float* cols, int32_t n_cols, int32_t d, double l,
                               double* sum_out_dev, void* stream);
int b2_spatial_nearest_f32(const float* rows, int32_t n_rows, const float* cols, int32_t n_cols, int32_t d, int32_t m,
                           int32_t* idx_out, void* stream);

/* ------------------------------------------------------------------------
 * GraphSCI (modules/single_modality/imputation/graphsci.py)
 *   b2_batchnorm_fwd/bwd_f32 : nn.BatchNorm1d over the rows of X [n, c] inside buildNetwork (:37-45); training → batch
 *       statistics (biased variance to normalise, running stats updated with momentum and the unbiased variance),
 *       eval → running statistics.  `act` 0 | 1 (ReLU) is fused after the affine transform.  save_mean / save_invstd [c]
 *       feed the backward.  Workspace: b2_batchnorm_workspace_bytes(c).
 *   b2_zinb_loss_grad_f32    : the three decoder heads' activations (Sigmoid :107, DispActivation :48-54, MeanActivation
 *       :57-63) + ZINB negative log-likelihood + reconstruction MSE over the masked entries (get_loss :463-483):
 *       acc3 = {Σ nll, Σ (mean·sf − y)², #masked}; with d_a/d_b/d_c the gradients of
 *       le·nll_mean + ke·(0.5/g)·mse_mean w.r.t. the three pre-activations.  mask: bytes [n, g] or NULL (all).
 *   b2_batchnorm_stats_f32   : the statistics half of b2_batchnorm_fwd_f32 without the apply: save_mean / save_invstd
 *       (training: from the batch, running stats updated; eval: from the running stats, X may be NULL).
 *   b2_graphsci_heads_train_f32 : the three decoder heads (Linear, BatchNorm) of AEModel :101-104 fused with get_loss's ZINB /
 *       MSE terms (:463-483), for the low-memory training schedule.  pre_pi / pre_disp / pre_mean [n, g] (common ldp) are the
 *       heads' GEMM outputs; gamma, beta, mean, invstd, dgamma, dbeta are packed [3, g] (pi, disp, mean), mean / invstd from
 *       b2_batchnorm_stats_f32.  BatchNorm, activations and loss stay in registers: acc3 as b2_zinb_loss_grad_f32, and each
 *       pre_h is overwritten IN PLACE by ∂(le·nll_mean + ke·(0.5/g)·mse_mean)/∂pre_h through the BatchNorm (batch statistics);
 *       dgamma / dbeta its affine gradients.  Two passes over the rows.  Workspace: b2_graphsci_heads_workspace_bytes(g).
 *   b2_graphsci_heads_eval_f32 : the same heads in eval mode (running statistics, mean / invstd from b2_batchnorm_stats_f32
 *       with training = 0) over n rows: acc3 (+)= {Σ nll, Σ mse, #masked} (accumulate = 1 adds to it, for row chunks) and,
 *       when z_exp is given, z_exp = mean·sf (GraphSCI.evaluate :377-381).  Read-only on pre.
 *   b2_adj_sample_f32        : z = μ + exp(log_std)·ε  (torch.normal(mean, exp(log_std)) :130 with explicit noise)
 *   b2_adj_loss_grad_f32     : acc2 = {Σ_i −Σ_c w_c t_ic log_softmax(z_i)_c, Σ (1 + 2ls − μ² − e^{2ls})} (F.cross_entropy with
 *       probability targets and class weights :461, kl_adj :479-480); dz = coef_ce·∂CE_sum/∂z (optional).
 *   b2_adj_reparam_bwd_f32   : dμ = dz − 2·coef_kl·μ ; dlog_std = dz·ε·e^{ls} + coef_kl·(2 − 2e^{2ls}).
 * ---------------------------------------------------------------------- */
size_t b2_batchnorm_workspace_bytes(int32_t c);
int b2_batchnorm_fwd_f32(const float* X, int64_t ldx, int32_t n, int32_t c, const float* gamma, const float* beta,
                         float* running_mean, float* running_var, int training, float momentum, float eps, int act,
                         float* out, int64_t ldo, float* save_mean, float* save_invstd,
                         void* workspace, size_t workspace_bytes, void* stream);
int b2_batchnorm_bwd_f32(const float* dY, int64_t lddy, const float* Y, int64_t ldy, const float* X, int64_t ldx,
                         int32_t n, int32_t c, const float* gamma, const float* save_mean, const float* save_invstd,
                         int act, int training, float* dX, int64_t lddx, float* dgamma, float* dbeta,
                         void* workspace, size_t workspace_bytes, void* stream);
int b2_zinb_loss_grad_f32(const float* a_pi, const float* b_disp, const float* c_mean, int64_t ld,
                          const float* Y, int64_t ldy, const float* size_factors, const uint8_t* mask, int64_t ldm,
                          int32_t n, int32_t g, float le, float ke, float* d_a, float* d_b, float* d_c, int64_t ldd,
                          float* mean_out, float* disp_out, float* pi_out, int64_t ldo, double* acc3, void* stream);
int b2_batchnorm_stats_f32(const float* X, int64_t ldx, int32_t n, int32_t c, float* running_mean, float* running_var,
                           int training, float momentum, float eps, float* save_mean, float* save_invstd,
                           void* workspace, size_t workspace_bytes, void* stream);
size_t b2_graphsci_heads_workspace_bytes(int32_t g);
int b2_graphsci_heads_train_f32(float* pre_pi, float* pre_disp, float* pre_mean, int64_t ldp, const float* gamma,
                                const float* beta, const float* mean, const float* invstd, const float* Y, int64_t ldy,
                                const float* size_factors, const uint8_t* mask, int64_t ldm, int32_t n, int32_t g, float le,
                                float ke, float* dgamma, float* dbeta, double* acc3, void* workspace, size_t workspace_bytes,
                                void* stream);
int b2_graphsci_heads_eval_f32(const float* pre_pi, const float* pre_disp, const float* pre_mean, int64_t ldp,
                               const float* gamma, const float* beta, const float* mean, const float* invstd, const float* Y,
                               int64_t ldy, const float* size_factors, const uint8_t* mask, int64_t ldm, int32_t n, int32_t g,
                               int accumulate, double* acc3, float* z_exp, int64_t ldz, void* stream);
int b2_adj_sample_f32(const float* mu, const float* log_std, const float* eps, int64_t n_elem, float* z, void* stream);
int b2_adj_loss_grad_f32(const float* z, const float* mu, const float* log_std, const float* target,
                         const float* class_weight, int32_t g, float coef_ce, float* dz, double* acc2, void* stream);
int b2_adj_reparam_bwd_f32(const float* dz, const float* mu, const float* log_std, const float* eps, int64_t n_elem,
                           float coef_kl, float* dmu, float* dlog_std, void* stream);

/* Pair-sharded form of b2_gae_loss_grad_f32 for multi-GPU runs (InnerProductDecoder + gae_loss_function, scgnn2.py:423-426,
 * 603-619).  The all-pairs part is partitioned into b2_gae_sym_super_blocks(n) equal-work units (super-block s = the 128-row
 * blocks s and nb-1-s): rank r takes super-blocks [sb_begin, sb_end), plus the label / KLD terms of its own rows
 * [row_begin, row_begin + n_rows).  dz_full [n, d] is zero-filled here and receives this rank's contributions: sum it over
 * ranks (all-reduce); loss_out holds this rank's share of the loss.  d <= 16.  Workspace: b2_gae_loss_workspace_bytes(n, d).
 * Labels (lab_vals NULL: unit; set: real-valued with labt_*) as in b2_gae_loss_grad_f32. */
int b2_gae_sym_super_blocks(int32_t n);
int b2_gae_loss_grad_sym_f32(const float* z, int64_t ldz, const float* mu, const float* logvar, int64_t ldm,
                             const int32_t* lab_rowptr, const int32_t* lab_colidx, const float* lab_vals,
                             const int32_t* labt_rowptr, const int32_t* labt_colidx, const float* labt_vals, int32_t n, int32_t d,
                             int32_t sb_begin, int32_t sb_end, int32_t row_begin, int32_t n_rows, float norm, float pos_weight,
                             int use_pos_weight, float* dz_full, float* dmu, float* dlogvar, int64_t ldd, float* loss_out,
                             void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------
 * scGNN EM-iteration stages (SURVEY §8f row 3)
 *   b2_kmeans_step_f32        : one Lloyd iteration of sklearn.cluster.KMeans(...).fit_predict(embed), scgnn2.py:186 —
 *       labels <- nearest centre (ties: lowest index); update != 0: centres <- cluster means (empty clusters keep theirs).
 *       stats (device, 3 doubles) = {inertia w.r.t. the old centres, ||dC||^2, number of changed labels}.
 *   b2_graph_regu_weights_f32 : graph_celltype_regu_handler + the `[clusterIndex][:, clusterIndex]` slicing of
 *       cluster_AE_handler (scgnn2.py:716-730, 844-846) without the N x N matrix.  The reference normalises an np.matrix, so its
 *       `avg_mtx * x` is a MATRIX product and adjdense[i, j] = deg_j / deg_i (dense, rank one); the column sums inside j's cluster are
 *       w_j = deg_j * sum_{i in cluster(j)} 1/deg_i.  Pattern = A or A + I CSR (the diagonal is not counted); cluster_sums: n_clusters
 *       device doubles of scratch.
 *   b2_graph_regu_weights_weighted_f32 : the same for a weighted, directed adj (graph_AE_retain_weights returns W): adjdense[i, j]
 *       = colsum_j / rowsum_i, so w_j = colsum_j * sum_{i in cluster(j)} 1/rowsum_i; a row with zero sum adds 0.  vals: fp64 CSR
 *       values; the diagonal is not counted.  scratch: n + n_clusters device doubles.
 *   b2_celltype_loss_grad_f32 : loss_function_graph(regularizer_type="Celltype"), scgnn2.py:1316-1326, with the dense
 *       `M @ mse` products folded into per-row weights: value = sum_j row_weight_j * sum_g (r-x)^2 + || (x_dropout - r)[x_dropout != 0] ||_2
 *       (callers pass row_weight = 0.3 + 0.3*w_graph + 0.1*w_celltype); grad = d value / d recon masked by recon > 0.
 *       scratch2: 2 device doubles.
 *   b2_l1_grad_add_f32        : the `loss + 1*l1` term of train_handler (scgnn2.py:1268-1274): grad += coef*sign(p).
 *   b2_louvain_csr_host       : generateLouvainCluster (scgnn2.py:193-215; networkx -> igraph.community_multilevel) as
 *       multilevel modularity optimisation on a symmetric weighted CSR in HOST memory (both directions stored).
 *       Deterministic (index order, ties keep the current community).
 * ---------------------------------------------------------------------- */
size_t b2_kmeans_workspace_bytes(int32_t k, int32_t d);
int b2_kmeans_step_f32(const float* X, int64_t ldx, int32_t n, int32_t d, float* C, int32_t k, int32_t* labels, int update,
                       double* stats, void* workspace, size_t workspace_bytes, void* stream);
int b2_graph_regu_weights_f32(const int32_t* rowptr, const int32_t* colidx, const int32_t* labels, int32_t n, int32_t n_clusters,
                              double* cluster_sums, float* w, void* stream);
int b2_graph_regu_weights_weighted_f32(const int32_t* rowptr, const int32_t* colidx, const double* vals, const int32_t* labels, int32_t n,
                                       int32_t n_clusters, double* scratch, float* w, void* stream);
int b2_celltype_loss_grad_f32(const float* recon, const float* target, const float* x_dropout, const float* row_weight,
                              int64_t rows, int32_t cols, int32_t cols_orig, int relu_mask, float* grad, float* loss_out,
                              double* scratch2, void* stream);
int b2_l1_grad_add_f32(const float* param, float* grad, int64_t n, float coef, float* l1_out, void* stream);
int b2_louvain_csr_host(const int64_t* rowptr, const int32_t* colidx, const double* weights, int32_t n, int32_t* labels_out,
                        int32_t* n_comm_out, double* modularity_out, int max_levels, double min_gain);

/* ------------------------------------------------------------------------
 * Leiden community detection (csrc/leiden.cu): SpaGCN's init="louvain" (spagcn.py:481-492 → scanpy 1.10 tl.leiden →
 * leidenalg.RBConfigurationVertexPartition with weights = the connectivities and resolution_parameter = resolution).
 *   The graph is an n×n CSR on the device that must be SYMMETRIC with both directions stored (scanpy's connectivities always
 *   are; a self-loop is stored once); vals NULL means unit weights, otherwise they must be finite and non-negative.  With
 *   W = Σ vals, k_i = row sums and K_c = Σ_{i∈c} k_i, the optimised quality is Q = Σ_c (e_c − resolution·K_c²/W), e_c the
 *   weight inside c; quality_out (host) receives Q / W, which is networkx's modularity(resolution=...) on the undirected graph.
 *   max_iterations = -1 repeats Leiden iterations until one leaves the membership unchanged (at most 100), k > 0 runs at most k.
 *   labels_out [n] (device) are 0..K-1 by decreasing community size, ties by the smallest member; *n_comm_out (host) = K.
 *   info_out (host, nullable) [2]: iterations run, most aggregation levels in one iteration.
 *   Run-to-run deterministic.  Refinement merges greedily (leidenalg samples with θ = 0.01), so labels are not leidenalg's.
 *   Synchronises the stream: each phase needs its counts on the host.  The workspace bound depends on (n, nnz) only, since no
 *   aggregated level is larger than the input; b2_leiden_workspace_bytes returns 0 for n <= 0 or nnz outside [0, 2^31).
 * ---------------------------------------------------------------------- */
size_t b2_leiden_workspace_bytes(int32_t n, int64_t nnz);
int b2_leiden_f32(const int32_t* rowptr, const int32_t* colidx, const float* vals, int32_t n, int64_t nnz, double resolution,
                  int max_iterations, int32_t* labels_out, int32_t* n_comm_out, double* quality_out, int32_t* info_out,
                  void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------
 * scGNN's normalizer(X, base) (scgnn2.py:795-805) and the concatenations that use it: *_concat_prev_embed
 * (feature_AE_handler scgnn2.py:283-294, graph_AE_handler scgnn2.py:543-546) and clustering_embed = "both" (scgnn2.py:155-157).
 *   b2_quantiles_f32     : np.quantile(base, qs[j]) over ALL rows*cols elements of the row-padded matrix base (method "linear",
 *       q cast to float32 first, so the virtual index (n-1)*q is a float32 product; numpy's _get_indexes clamp and float32 _lerp).
 *       Radix select on the order-preserving uint32 key (-0.0 keyed as +0.0): the order statistics of both quantiles come out of
 *       the same three histogram passes over base (11 / 11 / 10 bits), with 64-bit counts.  nq in {1, 2}; qs is a HOST array.
 *       out: nq + 3 DEVICE doubles, written on the stream: the nq quantiles, then min(base), max(base) and the number of
 *       non-finite elements.  Nothing is synchronised; the caller reads out once.
 *   b2_col_minmax_f32    : per-column min / max of x ignoring NaN (np.nanmin / nanmax, MinMaxScaler.partial_fit's data_min_ /
 *       data_max_); an all-NaN column gives NaN.  nonfinite (nullable): one device double, the count of non-finite elements.
 *   b2_concat_scaled_f32 : out[:, :a] = left; out[:, a:a+e] = right * scale_ + min_ (scale != 0) or right; out[:, a+e:ldo] = 0.
 *       scale_ / min_ are MinMaxScaler's, in float32: scale_ = (hi - lo) / range (range = cmax - cmin, set to 1 below 10*eps),
 *       min_ = lo - cmin * scale_; the transform is two separately rounded operations (x *= scale_; x += min_), never an FMA.
 *       ldo must be a multiple of 4 (so the row-padded result keeps the GEMM / kNN on their tensor-core paths) and out 16-byte
 *       aligned.  The workspace is used only when scale != 0.
 * ---------------------------------------------------------------------- */
size_t b2_quantiles_workspace_bytes(void);
int b2_quantiles_f32(const float* base, int64_t ldb, int64_t rows, int32_t cols, const float* qs, int32_t nq, double* out,
                     void* workspace, size_t workspace_bytes, void* stream);
size_t b2_col_minmax_workspace_bytes(int32_t cols);
int b2_col_minmax_f32(const float* x, int64_t ldx, int64_t rows, int32_t cols, float* cmin, float* cmax, double* nonfinite,
                      void* workspace, size_t workspace_bytes, void* stream);
size_t b2_concat_scaled_workspace_bytes(int32_t e);
int b2_concat_scaled_f32(const float* left, int64_t ldl, int32_t a, const float* right, int64_t ldr, int32_t e, int64_t rows,
                         const float* cmin, const float* cmax, float lo, float hi, int scale, float* out, int64_t ldo,
                         void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------
 * Cell-sharded data parallelism inside the C-ABI (SURVEY §8(b)4, §8(e)): NCCL over NVLink, resolved with dlopen at run time
 * (b2_comm_available() == 0 when libnccl.so.2 cannot be loaded).  One communicator per process / GPU:
 *   rank 0: b2_comm_unique_id(id) → ship the 128 bytes to the other ranks by any channel → every rank: b2_comm_init_rank
 *   b2_allreduce_sum_f32 : in-place sum of a flat fp32 buffer — the gradient bucket of the Feature-AE / Graph-AE engines (the
 *                          only collective of the sample-parallel paths), the partial dz of b2_gae_loss_grad_sym_f32, the loss
 *   b2_allgather_f32     : equal-sized row blocks → full operand (the N×32 support of the row-sharded aggregate, z of the decoder)
 * Collectives are enqueued on `stream`; replaces torch.distributed in dance_b200/parallel.py for non-Python binders.
 * ---------------------------------------------------------------------- */
typedef struct b2_comm b2_comm;
int b2_comm_available(void);
int b2_comm_version(void);
int b2_comm_unique_id(void* id128 /* 128 bytes */);
int b2_comm_init_rank(b2_comm** out, const void* id128, int world, int rank);
int b2_comm_destroy(b2_comm* comm);
int b2_comm_world(const b2_comm* comm);
int b2_comm_rank(const b2_comm* comm);
int b2_allreduce_sum_f32(b2_comm* comm, float* buf, int64_t n, void* stream);
int b2_allgather_f32(b2_comm* comm, const float* local, float* full, int64_t count, void* stream);

/* ------------------------------------------------------------------------
 * Pre-processing operators upstream of scGNN / GraphSCI (SURVEY §8f row 1)
 *   b2_gene_stats_f32   : per-gene Σx, Σx², #(x>0) over the cells (fp64) — sc.pp.filter_genes counts (filter.py:56-158),
 *                         FilterGenesTopK / FilterGenes summaries sum | var | cv | rv (filter.py:470-489)
 *   b2_cell_stats_f32   : per-cell Σx, #(x>0) — sc.pp.filter_cells counts
 *   b2_subset_f32       : out[i, j] = X[rows[i], cols[j]] (NULL = identity) — AnnData._inplace_subset_var / filter_by_mask
 *   b2_cellwise_mask_u8 : CellwiseMaskData.__call__ (mask.py:153-291): per cell with more than min_gene_counts stored non-zeros,
 *                         floor(n_pos·mask_rate) entries are drawn WITHOUT replacement with probability ∝ exp(−x/20) ("exp") or
 *                         uniformly; with add_test_mask max(1, round(0.1·n)) of them become validation entries, the rest test.
 *                         The draw is counter-based (hash of seed, cell, gene): same distribution as numpy's rng.choice, not the
 *                         same stream.  Masks are [n, g] bytes.
 * ---------------------------------------------------------------------- */
int b2_gene_stats_f32(const float* X, int64_t ldx, int64_t n, int32_t g, double* sum, double* sumsq, double* nnz, void* stream);
int b2_cell_stats_f32(const float* X, int64_t ldx, int64_t n, int32_t g, double* sum, double* nnz, void* stream);
int b2_subset_f32(const float* X, int64_t ldx, const int64_t* rows, const int32_t* cols, int64_t n_out, int32_t g_out,
                  float* out, int64_t ldo, void* stream);
int b2_cellwise_mask_u8(const float* X, int64_t ldx, int64_t n, int32_t g, float mask_rate, int32_t min_gene_counts,
                        int distr_exp, int add_test_mask, uint32_t seed, uint8_t* train, uint8_t* valid, uint8_t* test,
                        int32_t* overflow_rows, void* stream);

/* ------------------------------------------------------------------------
 * graph-sc (GraphSC) mini-batch training, graphsc.py:179-216 (fit), :355-411 (GCNAE, InnerProductDecoder), :428-484
 * (WeightedGraphConv.forward).
 *
 * A block is a list of destination node ids `dst` [n_dst] (entries < 0 are padding, skipped) over the parent graph's
 * destination-indexed CSR `rowptr` [n_nodes + 1] / `colidx` / `weights` (row v = sources of v's in-edges, edge weights;
 * GraphLite.csr_by_destination()).  Its in-degree is the full row length (the full-neighbour sampler keeps every in-edge),
 * its out-degree is per block.  No relabelled block CSR is built.
 *
 * Dropout: keep(seed, key, row, col) of common.cuh, as b2_dropout_f32 (so b2_dropout_f32 on a matrix of ones with the same
 * seed and key materialises any mask).  Feature dropout rows are GLOBAL node ids; decoder rows are positions in the batch.
 * GraphSCEngine's key layout: key = (step·2 + pass)·3 + site, step = mini-batch counter, pass 0 (embedding) | 1 (loss),
 * site 0 = layer-1 input, 1 = layer-2 input, 2 = decoder.
 *
 *   b2_graphsc_block_degrees       : outdeg [n_nodes] ← per-source count of edges into dst (zeroed first).  With src_list
 *       [src_cap] / src_pos [n_nodes] / n_src [1] (all or none): the block's source set, each source appended once in
 *       first-touch order (src_pos[u] = its slot), unused slots -1.  src_cap must bound the sources (Σ row lengths does).
 *   b2_graphsc_block_aggregate_f32 : transposed = 0: out[i, f] = s_v · Σ_{e: u→v} w_e · c_u · keep(u, f) · in[row(u), f] / (1 − p)
 *       with v = dst[i], c_u = clamp(outdeg[u], 1)^-1/2, s_v = clamp(indeg_v, 1)^-1/2 (· 1/indeg_v when agg_mean),
 *       row(u) = x_pos[u] (x_pos NULL: u), weights NULL = 1.  Padding slots give zero rows.
 *       transposed = 1: the adjoint: out[row(u), f] = Σ over the same terms with in[i, f] (dout) in place of in[row(u), f];
 *       out [out_rows, F] is zeroed first.  Order of the atomic sums is not fixed.
 *   b2_graphsc_batch_decoder_f32   : z [B, d], 1 ≤ d ≤ 1024: z̃ = keep(row, col) ⊙ z / (1 − p), S = z̃z̃ᵀ, labels I,
 *       pw = B − 1, norm = B / (2(B − 1)) (B = 1: pw = 0, norm = 1);  loss_out[0] = norm/B² · Σ [pw·y·softplus(−S) +
 *       (1−y)·softplus(S)] (written, on the device), dz = keep ⊙ 2·(∂loss/∂S)·z̃ / (1 − p) (overwritten).
 *   b2_graphsc_scatter_rows_f32    : out[idx[i] − offset, :] = x[i, :] (recorded embeddings in cell order).
 * ---------------------------------------------------------------------- */
int b2_graphsc_block_degrees(const int32_t* rowptr, const int32_t* colidx, int32_t n_nodes, const int32_t* dst, int32_t n_dst,
                             int32_t* outdeg, int32_t* src_list, int32_t* src_pos, int32_t* n_src, int32_t src_cap, void* stream);
int b2_graphsc_block_aggregate_f32(const int32_t* rowptr, const int32_t* colidx, const float* weights, const int32_t* dst,
                                   int32_t n_dst, const int32_t* outdeg, const float* in, int64_t ldin, const int32_t* x_pos,
                                   int32_t F, int agg_mean, float p, uint32_t seed, uint32_t key, int transposed, float* out,
                                   int64_t ldout, int64_t out_rows, void* stream);
int b2_graphsc_batch_decoder_f32(const float* z, int64_t ldz, int32_t B, int32_t d, float p, uint32_t seed, uint32_t key,
                                 float* dz, int64_t lddz, float* loss_out, void* stream);
int b2_graphsc_scatter_rows_f32(const float* x, int64_t ldx, int32_t rows, int32_t cols, const int32_t* idx, int32_t offset,
                                float* out, int64_t ldo, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DANCE_B200_H_ */
