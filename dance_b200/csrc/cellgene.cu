// scDeepSort path: cell–gene graph construction, AdaptiveSAGE edge values, softmax cross-entropy.
//
//  * b2_cellgene_graph_*   CellFeatureGraph.__call__ (reference transforms/graph/cell_feature_graph.py:34-79):
//      nonzeros of the dense cell×gene matrix → COO edges in the reference's order
//      [cell→gene ×nnz ; gene→cell ×nnz ; self ×(G+N)], per-destination renormalisation
//      w ← indeg·w / Σ_in w (:62-68), self loops with weight 1 (:69).  Gene nodes come first (ids 0..G-1).
//  * b2_sage_edge_values   AdaptiveSAGE.message_func (reference models/nn/gnn.py:62-82): per-edge scalar
//      w_e · alpha[idx(e)], idx = src gene id (gene→cell) | dst gene id (cell→gene) | G (gene self) | G+1 (cell self).
//      The aggregate itself is b2_spmm_csr_f32(reduce = mean) with these values.
//  * b2_softmax_ce_sum     nn.CrossEntropyLoss(reduction="sum") forward + gradient (scdeepsort.py:185,241).
#include "common.cuh"

#include <cub/device/device_scan.cuh>

namespace b2 {

// per cell: number of nonzeros and their sum; per gene (atomics): count and sum
__global__ void __launch_bounds__(256)
cg_count_kernel(const float* __restrict__ X, int64_t ldx, int32_t n, int32_t g, int32_t* __restrict__ row_cnt,
                float* __restrict__ row_sum, int32_t* __restrict__ col_cnt, float* __restrict__ col_sum) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < n; r += nwarps) {
    int c = 0;
    float s = 0.f;
    for (int j = lane; j < g; j += 32) {
      const float v = X[r * ldx + j];
      if (v != 0.f) {
        ++c;
        s += v;
        atomicAdd(col_cnt + j, 1);
        atomicAdd(col_sum + j, v);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    s = warp_sum(s);
    if (lane == 0) { row_cnt[r] = c; row_sum[r] = s; }
  }
}

// one warp per cell: ordered compaction of the row's nonzeros (ballot + popc keeps np.nonzero order)
__global__ void __launch_bounds__(256)
cg_fill_kernel(const float* __restrict__ X, int64_t ldx, int32_t n, int32_t g, const int64_t* __restrict__ row_off,
               const int32_t* __restrict__ row_cnt, const float* __restrict__ row_sum, const int32_t* __restrict__ col_cnt,
               const float* __restrict__ col_sum, int normalize, int64_t nnz, int64_t* __restrict__ src,
               int64_t* __restrict__ dst, float* __restrict__ w) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < n; r += nwarps) {
    int64_t pos = row_off[r];
    const float rdeg = (float)row_cnt[r], rsum = row_sum[r];
    for (int j0 = 0; j0 < g; j0 += 32) {
      const int j = j0 + lane;
      const float v = j < g ? X[r * ldx + j] : 0.f;
      const unsigned m = __ballot_sync(0xffffffffu, v != 0.f);
      if (v != 0.f) {
        const int64_t e = pos + __popc(m & ((1u << lane) - 1u));
        // cell → gene (destination = gene j): renormalised over the gene's in-edges
        src[e] = (int64_t)g + r;
        dst[e] = j;
        w[e] = normalize ? ((float)col_cnt[j] * v) / col_sum[j] : v;
        // gene → cell (destination = cell r)
        src[nnz + e] = j;
        dst[nnz + e] = (int64_t)g + r;
        w[nnz + e] = normalize ? (rdeg * v) / rsum : v;
      }
      pos += __popc(m);
    }
  }
  // self loops, weight 1 (added after the renormalisation, cell_feature_graph.py:69)
  const int64_t nodes = (int64_t)n + g;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < nodes; t += (int64_t)gridDim.x * blockDim.x) {
    src[2 * nnz + t] = t;
    dst[2 * nnz + t] = t;
    w[2 * nnz + t] = 1.f;
  }
}

__global__ void cast_i32_i64_kernel(const int32_t* in, int64_t* out, int32_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = in[i];
}

// AdaptiveSAGE edge values on a destination-indexed CSR: node ids < n_genes are genes, the rest cells
__global__ void __launch_bounds__(256)
sage_edge_values_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx,
                        const float* __restrict__ w, const float* __restrict__ alpha, int32_t n_nodes, int32_t n_genes,
                        float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t v = warp; v < n_nodes; v += nwarps) {
    const bool dst_gene = v < n_genes;
    for (int32_t p = rowptr[v] + lane; p < rowptr[v + 1]; p += 32) {
      const int32_t u = colidx[p];
      const bool src_gene = u < n_genes;
      int idx = n_genes + 1;                         // cell self loop
      if (src_gene && !dst_gene) idx = u;            // gene → cell: beta of the source gene
      if (dst_gene && !src_gene) idx = (int)v;       // cell → gene: beta of the destination gene
      if (dst_gene && src_gene) idx = n_genes;       // gene self loop
      out[p] = w[p] * alpha[idx];
    }
  }
}

// softmax cross-entropy, reduction = sum; one warp per row
__global__ void __launch_bounds__(256)
softmax_ce_kernel(const float* __restrict__ logits, int64_t ld, const int64_t* __restrict__ labels, int32_t n, int32_t c,
                  float* __restrict__ dlogits, int64_t ldd, float* __restrict__ loss_out) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  float local = 0.f;
  for (int64_t r = warp; r < n; r += nwarps) {
    float m = -3.4e38f;
    for (int j = lane; j < c; j += 32) m = fmaxf(m, logits[r * ld + j]);
    m = warp_max(m);
    float s = 0.f;
    for (int j = lane; j < c; j += 32) s += expf(logits[r * ld + j] - m);
    s = warp_sum(s);
    const float lse = m + logf(s);
    const int64_t y = labels[r];
    for (int j = lane; j < c; j += 32) {
      const float p = expf(logits[r * ld + j] - lse);
      if (dlogits) dlogits[r * ldd + j] = p - (j == y ? 1.f : 0.f);
    }
    if (lane == 0) local += lse - logits[r * ld + y];
  }
  if (lane == 0 && local != 0.f) atomicAdd(loss_out, local);
}

}  // namespace b2

using namespace b2;

// workspace layout: row_cnt[n] i32 | row_sum[n] f32 | col_cnt[g] i32 | col_sum[g] f32 | row_cnt64[n] | row_off[n+1] i64 | cub temp
static size_t cg_off(int32_t n, int32_t g, int which) {
  size_t o = 0;
  const size_t a[6] = {align_up((size_t)n * 4, 256), align_up((size_t)n * 4, 256), align_up((size_t)g * 4, 256),
                       align_up((size_t)g * 4, 256), align_up(((size_t)n + 1) * 8, 256), align_up(((size_t)n + 1) * 8, 256)};
  for (int i = 0; i < which; ++i) o += a[i];
  return o;
}

extern "C" size_t b2_cellgene_graph_workspace_bytes(int32_t n_cells, int32_t n_genes) {
  size_t temp = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, temp, (const int64_t*)nullptr, (int64_t*)nullptr, (int)n_cells + 1);
  return cg_off(n_cells, n_genes, 6) + align_up(temp, 256) + 256;
}

extern "C" int b2_cellgene_graph_count(const float* X, int64_t ldx, int32_t n_cells, int32_t n_genes, int64_t* nnz_out_host,
                                       void* workspace, size_t workspace_bytes, void* stream) {
  B2_REQUIRE(X && nnz_out_host && n_cells > 0 && n_genes > 0 && ldx >= n_genes, "b2_cellgene_graph_count: bad arguments");
  B2_REQUIRE(workspace && workspace_bytes >= b2_cellgene_graph_workspace_bytes(n_cells, n_genes),
             "b2_cellgene_graph_count: workspace too small");
  cudaStream_t st = as_stream(stream);
  char* ws = reinterpret_cast<char*>(workspace);
  int32_t* row_cnt = reinterpret_cast<int32_t*>(ws + cg_off(n_cells, n_genes, 0));
  float* row_sum = reinterpret_cast<float*>(ws + cg_off(n_cells, n_genes, 1));
  int32_t* col_cnt = reinterpret_cast<int32_t*>(ws + cg_off(n_cells, n_genes, 2));
  float* col_sum = reinterpret_cast<float*>(ws + cg_off(n_cells, n_genes, 3));
  int64_t* row_cnt64 = reinterpret_cast<int64_t*>(ws + cg_off(n_cells, n_genes, 4));
  int64_t* row_off = reinterpret_cast<int64_t*>(ws + cg_off(n_cells, n_genes, 5));
  void* d_temp = ws + cg_off(n_cells, n_genes, 6);
  size_t temp = workspace_bytes - cg_off(n_cells, n_genes, 6);
  B2_CHECK_CUDA(cudaMemsetAsync(col_cnt, 0, cg_off(n_cells, n_genes, 4) - cg_off(n_cells, n_genes, 2), st));
  cg_count_kernel<<<grid_blocks(n_cells, 8), 256, 0, st>>>(X, ldx, n_cells, n_genes, row_cnt, row_sum, col_cnt, col_sum);
  B2_CHECK_LAUNCH("cg_count_kernel");
  cast_i32_i64_kernel<<<grid_blocks(n_cells / 32 + 1, 8), 256, 0, st>>>(row_cnt, row_cnt64, n_cells);
  B2_CHECK_LAUNCH("cast_i32_i64_kernel");
  B2_CHECK_CUDA(cudaMemsetAsync(row_cnt64 + n_cells, 0, sizeof(int64_t), st));
  // exclusive scan over n_cells+1 items → row_off[n_cells] = nnz
  B2_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(d_temp, temp, row_cnt64, row_off, (int)n_cells + 1, st));
  int64_t total = 0;
  B2_CHECK_CUDA(cudaMemcpyAsync(&total, row_off + n_cells, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  B2_CHECK_CUDA(cudaStreamSynchronize(st));
  *nnz_out_host = total;
  return B2_OK;
}

extern "C" int b2_cellgene_graph_fill(const float* X, int64_t ldx, int32_t n_cells, int32_t n_genes, int normalize_edges,
                                      int64_t nnz, int64_t* src, int64_t* dst, float* w, void* workspace,
                                      size_t workspace_bytes, void* stream) {
  B2_REQUIRE(X && src && dst && w && workspace, "b2_cellgene_graph_fill: null pointer");
  B2_REQUIRE(workspace_bytes >= b2_cellgene_graph_workspace_bytes(n_cells, n_genes), "b2_cellgene_graph_fill: workspace too small");
  cudaStream_t st = as_stream(stream);
  char* ws = reinterpret_cast<char*>(workspace);
  cg_fill_kernel<<<grid_blocks(n_cells, 8), 256, 0, st>>>(
      X, ldx, n_cells, n_genes, reinterpret_cast<int64_t*>(ws + cg_off(n_cells, n_genes, 5)),
      reinterpret_cast<int32_t*>(ws + cg_off(n_cells, n_genes, 0)), reinterpret_cast<float*>(ws + cg_off(n_cells, n_genes, 1)),
      reinterpret_cast<int32_t*>(ws + cg_off(n_cells, n_genes, 2)), reinterpret_cast<float*>(ws + cg_off(n_cells, n_genes, 3)),
      normalize_edges, nnz, src, dst, w);
  B2_CHECK_LAUNCH("cg_fill_kernel");
  return B2_OK;
}

extern "C" int b2_sage_edge_values_f32(const int32_t* rowptr, const int32_t* colidx, const float* w, const float* alpha,
                                       int32_t n_nodes, int32_t n_genes, float* out, void* stream) {
  B2_REQUIRE(rowptr && colidx && w && alpha && out && n_nodes >= 0 && n_genes >= 0, "b2_sage_edge_values_f32: bad arguments");
  if (n_nodes == 0) return B2_OK;
  sage_edge_values_kernel<<<grid_blocks(n_nodes, 8), 256, 0, as_stream(stream)>>>(rowptr, colidx, w, alpha, n_nodes, n_genes, out);
  B2_CHECK_LAUNCH("sage_edge_values_kernel");
  return B2_OK;
}

extern "C" int b2_softmax_ce_sum_f32(const float* logits, int64_t ld, const int64_t* labels, int32_t n, int32_t c,
                                     float* dlogits, int64_t ldd, float* loss_out, void* stream) {
  B2_REQUIRE(logits && labels && loss_out && n >= 0 && c > 0 && ld >= c, "b2_softmax_ce_sum_f32: bad arguments");
  if (n == 0) return B2_OK;
  softmax_ce_kernel<<<grid_blocks(n, 8), 256, 0, as_stream(stream)>>>(logits, ld, labels, n, c, dlogits, ldd, loss_out);
  B2_CHECK_LAUNCH("softmax_ce_kernel");
  return B2_OK;
}
