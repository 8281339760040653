// FeatureFeatureGraph on the device (reference transforms/graph/feature_feature_graph.py:45-87):
//   1. Pearson correlation of the gene columns of X [n cells, g genes] — np.corrcoef(feat.T): fp64 throughout
//      (centre, Gram / (n-1), divide by the two standard deviations one after the other, clip to [-1, 1]), cast to fp32;
//   2. threshold: entries with -thr < r < thr are dropped, optionally all negative ones too; NaN (zero-variance genes)
//      survives both tests exactly as in numpy and therefore becomes an edge;
//   3. COO edge list in row-major order (scipy coo_matrix(dense)), unit weights, optionally dgl EdgeWeightNorm("both"):
//      w_e = outdeg(src)^-1/2 · indeg(dst)^-1/2.
// The Gram is a hand-written fp64 SIMT GEMM (64×64 tiles, 4×4 per thread, split over the cell axis with fp64 atomics):
// the result has to survive a cast to fp32 and a comparison with the threshold, so fp32 tensor-core products are not
// an option for the structure to be reproducible.  g·g·n·2 flops: 8 TFLOP fp64 at 1 M × 2 k.
#include "common.cuh"

#include <cub/device/device_scan.cuh>

namespace b2 {

constexpr int FG_T = 64;   // output tile
constexpr int FG_K = 16;   // cells per staged slab

__global__ void __launch_bounds__(256)
fg_colsum_kernel(const float* __restrict__ X, int64_t ldx, int32_t n, int32_t g, double* __restrict__ sum) {
  __shared__ double ss[8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + tx;
  const int64_t rows_per = ceil_div<int64_t>(n, gridDim.y);
  const int64_t r0 = (int64_t)blockIdx.y * rows_per;
  const int64_t r1 = (r0 + rows_per < (int64_t)n) ? r0 + rows_per : (int64_t)n;
  double s = 0.0;
  if (c < g) for (int64_t r = r0 + ty; r < r1; r += 8) s += (double)X[r * ldx + c];
  ss[ty][tx] = s;
  __syncthreads();
  if (ty == 0 && c < g) {
    for (int i = 1; i < 8; ++i) s += ss[i][tx];
    atomicAdd(sum + c, s);
  }
}

// mean = sum / n by DIVISION, as np.average does: a constant gene must centre to exact zeros (→ NaN correlations)
__global__ void fg_mean_kernel(double* __restrict__ sum, int32_t g, int32_t n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < g; i += gridDim.x * blockDim.x) sum[i] = sum[i] / (double)n;
}

// C[i,j] += Σ_r (X[r,i]-m_i)(X[r,j]-m_j) over this block's slice of cells; upper-triangular tiles only (bi <= bj)
__global__ void __launch_bounds__(256)
fg_gram_kernel(const float* __restrict__ X, int64_t ldx, int32_t n, int32_t g, const double* __restrict__ mean,
               double* __restrict__ Cm) {
  const int bi = blockIdx.y, bj = blockIdx.x;
  if (bi > bj) return;
  __shared__ double sa[FG_K][FG_T + 1], sb[FG_K][FG_T + 1];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;   // 16 × 16 threads, 4×4 outputs each
  const int64_t rows_per = ceil_div<int64_t>(ceil_div<int64_t>(n, gridDim.z), FG_K) * FG_K;
  const int64_t r0 = (int64_t)blockIdx.z * rows_per;
  const int64_t r1 = (r0 + rows_per < (int64_t)n) ? r0 + rows_per : (int64_t)n;
  double acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
  for (int64_t rb = r0; rb < r1; rb += FG_K) {
    // stage FG_K cells × 64 genes for both tile sides, centred in fp64
    for (int t = threadIdx.x; t < FG_K * FG_T; t += 256) {
      const int kk = t / FG_T, cc = t % FG_T;
      const int64_t r = rb + kk;
      const int ci = bi * FG_T + cc, cj = bj * FG_T + cc;
      sa[kk][cc] = (r < r1 && ci < g) ? (double)X[r * ldx + ci] - mean[ci] : 0.0;
      sb[kk][cc] = (r < r1 && cj < g) ? (double)X[r * ldx + cj] - mean[cj] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < FG_K; ++kk) {
      double av[4], bv[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) { av[a] = sa[kk][ty + 16 * a]; bv[a] = sb[kk][tx + 16 * a]; }
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = fma(av[a], bv[b], acc[a][b]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int i = bi * FG_T + ty + 16 * a, j = bj * FG_T + tx + 16 * b;
      if (i < g && j < g && (bi < bj || i <= j)) {
        if (gridDim.z == 1) Cm[(int64_t)i * g + j] = acc[a][b];
        else atomicAdd(Cm + (int64_t)i * g + j, acc[a][b]);
      }
    }
}

// corr = clip((c_ij/(n-1)) / sd_i / sd_j) → fp32, mirrored from the upper triangle
__global__ void __launch_bounds__(256)
fg_corr_kernel(const double* __restrict__ Cm, int32_t g, int32_t n, float* __restrict__ adj, int64_t lda) {
  const int64_t total = (int64_t)g * g;
  const double fact = 1.0 / (double)(n - 1);      // np.cov: c *= np.true_divide(1, fact)
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int i = (int)(t / g), j = (int)(t % g);
    const int a = i <= j ? i : j, b = i <= j ? j : i;
    const double sdi = sqrt(Cm[(int64_t)i * g + i] * fact), sdj = sqrt(Cm[(int64_t)j * g + j] * fact);
    double v = Cm[(int64_t)a * g + b] * fact;
    v /= sdi;                                      // c /= stddev[:, None]
    v /= sdj;                                      // c /= stddev[None, :]
    v = v < -1.0 ? -1.0 : (v > 1.0 ? 1.0 : v);     // np.clip keeps NaN
    adj[(int64_t)i * lda + j] = (float)v;
  }
}

__device__ __forceinline__ bool fg_keep(float v, float thr, int positive_only) {
  if (v > -thr && v < thr) return false;           // adj[(adj > -thr) & (adj < thr)] = 0
  if (positive_only && v < 0.f) return false;      // adj[adj < 0] = 0
  return v != 0.f;                                 // coo_matrix(adj): stored entries are the nonzeros (NaN != 0 → kept)
}

// one warp per row: count kept entries; column in-degrees through atomics
__global__ void __launch_bounds__(256)
fg_count_kernel(const float* __restrict__ adj, int64_t lda, int32_t g, float thr, int positive_only,
                int32_t* __restrict__ row_cnt, int32_t* __restrict__ col_cnt) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = warp; i < g; i += nwarps) {
    int cnt = 0;
    for (int j = lane; j < g; j += 32)
      if (fg_keep(adj[i * lda + j], thr, positive_only)) { ++cnt; atomicAdd(col_cnt + j, 1); }
    cnt = __reduce_add_sync(0xffffffffu, cnt);
    if (lane == 0) row_cnt[i] = cnt;
  }
}

__global__ void __launch_bounds__(256)
fg_fill_kernel(const float* __restrict__ adj, int64_t lda, int32_t g, float thr, int positive_only,
               const int32_t* __restrict__ rowptr, const int32_t* __restrict__ col_cnt, int normalize,
               int32_t* __restrict__ src, int32_t* __restrict__ dst, float* __restrict__ w) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = warp; i < g; i += nwarps) {
    int32_t wp = rowptr[i];
    const float out_norm = normalize ? powf((float)(rowptr[i + 1] - rowptr[i]), -0.5f) : 1.f;
    for (int j0 = 0; j0 < g; j0 += 32) {
      const int j = j0 + lane;
      const bool k = j < g && fg_keep(adj[i * lda + j], thr, positive_only);
      const unsigned m = __ballot_sync(0xffffffffu, k);
      if (k) {
        const int32_t p = wp + __popc(m & ((1u << lane) - 1u));
        src[p] = (int32_t)i;
        dst[p] = j;
        w[p] = normalize ? out_norm * powf((float)col_cnt[j], -0.5f) : 1.f;
      }
      wp += __popc(m);
    }
  }
}

}  // namespace b2

using namespace b2;

extern "C" size_t b2_pearson_corr_workspace_bytes(int32_t g) {
  return align_up(sizeof(double) * (size_t)g * g, 256) + align_up(sizeof(double) * (size_t)g, 256);
}

extern "C" int b2_pearson_corr_f32(const float* X, int64_t ldx, int32_t n, int32_t g, float* adj, int64_t lda,
                                   void* workspace, size_t workspace_bytes, void* stream) {
  B2_REQUIRE(X && adj && n >= 2 && g >= 1 && ldx >= g && lda >= g, "b2_pearson_corr_f32: bad arguments (n >= 2)");
  B2_REQUIRE(workspace && workspace_bytes >= b2_pearson_corr_workspace_bytes(g), "b2_pearson_corr_f32: workspace too small");
  cudaStream_t st = as_stream(stream);
  char* base = reinterpret_cast<char*>(workspace);
  double* Cm = reinterpret_cast<double*>(base);
  double* sum = reinterpret_cast<double*>(base + align_up(sizeof(double) * (size_t)g * g, 256));
  B2_CHECK_CUDA(cudaMemsetAsync(sum, 0, sizeof(double) * g, st));
  {
    const int col_tiles = ceil_div(g, 32);
    dim3 grid(col_tiles, row_splits(col_tiles, n, 64, 4));
    fg_colsum_kernel<<<grid, 256, 0, st>>>(X, ldx, n, g, sum);
    B2_CHECK_LAUNCH("fg_colsum_kernel");
    fg_mean_kernel<<<ceil_div(g, 256), 256, 0, st>>>(sum, g, n);
    B2_CHECK_LAUNCH("fg_mean_kernel");
  }
  const int tiles = ceil_div(g, FG_T);
  const int tri = tiles * (tiles + 1) / 2;
  const int splits = row_splits(tri, n, 256, 2);
  if (splits > 1) B2_CHECK_CUDA(cudaMemsetAsync(Cm, 0, sizeof(double) * (size_t)g * g, st));
  dim3 grid(tiles, tiles, splits);
  fg_gram_kernel<<<grid, 256, 0, st>>>(X, ldx, n, g, sum, Cm);
  B2_CHECK_LAUNCH("fg_gram_kernel");
  fg_corr_kernel<<<grid_blocks((int64_t)g * g, 1024), 256, 0, st>>>(Cm, g, n, adj, lda);
  B2_CHECK_LAUNCH("fg_corr_kernel");
  return B2_OK;
}

extern "C" size_t b2_threshold_graph_workspace_bytes(int32_t g) {
  size_t temp = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, temp, (const int32_t*)nullptr, (int32_t*)nullptr, g + 1);
  return align_up(temp, 256) + 2 * align_up(sizeof(int32_t) * ((size_t)g + 1), 256);
}

extern "C" int b2_threshold_graph_count(const float* adj, int64_t lda, int32_t g, float threshold, int positive_only,
                                        int32_t* rowptr, int64_t* nnz_host, void* workspace, size_t workspace_bytes,
                                        void* stream) {
  B2_REQUIRE(adj && rowptr && nnz_host && g >= 1 && lda >= g, "b2_threshold_graph_count: bad arguments");
  B2_REQUIRE(workspace && workspace_bytes >= b2_threshold_graph_workspace_bytes(g), "b2_threshold_graph_count: workspace too small");
  cudaStream_t st = as_stream(stream);
  size_t temp = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, temp, (const int32_t*)nullptr, (int32_t*)nullptr, g + 1);
  char* base = reinterpret_cast<char*>(workspace);
  const size_t cnt_bytes = align_up(sizeof(int32_t) * ((size_t)g + 1), 256);
  int32_t* row_cnt = reinterpret_cast<int32_t*>(base + align_up(temp, 256));
  int32_t* col_cnt = reinterpret_cast<int32_t*>(base + align_up(temp, 256) + cnt_bytes);
  B2_CHECK_CUDA(cudaMemsetAsync(row_cnt, 0, 2 * cnt_bytes, st));
  fg_count_kernel<<<grid_blocks(g, 8), 256, 0, st>>>(adj, lda, g, threshold, positive_only, row_cnt, col_cnt);
  B2_CHECK_LAUNCH("fg_count_kernel");
  B2_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(base, temp, row_cnt, rowptr, g + 1, st));
  int32_t total = 0;
  B2_CHECK_CUDA(cudaMemcpyAsync(&total, rowptr + g, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  B2_CHECK_CUDA(cudaStreamSynchronize(st));
  *nnz_host = total;
  return B2_OK;
}

extern "C" int b2_threshold_graph_fill(const float* adj, int64_t lda, int32_t g, float threshold, int positive_only,
                                       const int32_t* rowptr, int normalize_edges, int32_t* src, int32_t* dst, float* w,
                                       void* workspace, size_t workspace_bytes, void* stream) {
  B2_REQUIRE(adj && rowptr && src && dst && w && g >= 1 && lda >= g, "b2_threshold_graph_fill: bad arguments");
  B2_REQUIRE(workspace && workspace_bytes >= b2_threshold_graph_workspace_bytes(g), "b2_threshold_graph_fill: workspace too small");
  size_t temp = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, temp, (const int32_t*)nullptr, (int32_t*)nullptr, g + 1);
  char* base = reinterpret_cast<char*>(workspace);
  const size_t cnt_bytes = align_up(sizeof(int32_t) * ((size_t)g + 1), 256);
  const int32_t* col_cnt = reinterpret_cast<const int32_t*>(base + align_up(temp, 256) + cnt_bytes);   // left there by `count`
  fg_fill_kernel<<<grid_blocks(g, 8), 256, 0, as_stream(stream)>>>(adj, lda, g, threshold, positive_only, rowptr, col_cnt,
                                                                   normalize_edges, src, dst, w);
  B2_CHECK_LAUNCH("fg_fill_kernel");
  return B2_OK;
}
