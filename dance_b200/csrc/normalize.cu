// normalize_total (+ log1p) on a dense cell×gene matrix, in place.
// Replaces scanpy.pp.normalize_total / scanpy.pp.log1p as called through
// AnnDataTransform (reference transforms/interface.py:67-68), NormalizeTotal
// (normalize.py:569-628), Log1P (normalize.py:531-564), NormalizeTotalLog1P (:664-679).
// Semantics restated from scanpy 1.10.1 (SURVEY.md App. A), pinned by the reference's
// tests/transforms/test_normalize.py:8-43.
//
// One warp per cell.  The common configuration (no highly-expressed-gene exclusion,
// explicit target_sum) is a single kernel: sweep 1 sums the row, sweep 2 re-reads it
// (an 8–20 KB row, L1/L2 resident) scales, applies log1p and stores → one HBM read +
// one HBM write of X.
#include "common.cuh"

#include <cub/device/device_radix_sort.cuh>
#include <math_constants.h>

namespace b2 {

__device__ __forceinline__ float row_sum_warp(const float* __restrict__ row, int g, const int32_t* __restrict__ excl,
                                              int lane) {
  float s = 0.f;
  if (((reinterpret_cast<uintptr_t>(row) & 15) == 0) && !excl) {
    const int g4 = g >> 2;
    const float4* r4 = reinterpret_cast<const float4*>(row);
    for (int c = lane; c < g4; c += 32) { const float4 v = r4[c]; s += (v.x + v.y) + (v.z + v.w); }
    for (int c = (g4 << 2) + lane; c < g; c += 32) s += row[c];
  } else {
    for (int c = lane; c < g; c += 32) if (!excl || !excl[c]) s += row[c];
  }
  return warp_sum(s);
}

// pass A (only with exclusion): totals over all genes, then flag genes above the fraction in this cell
__global__ void __launch_bounds__(256)
norm_flag_kernel(const float* __restrict__ X, int64_t ldx, int32_t n, int32_t g, float max_fraction,
                 int32_t* __restrict__ excl) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < n; r += nwarps) {
    const float* row = X + r * ldx;
    const float total = row_sum_warp(row, g, nullptr, lane);
    const float lim = total * max_fraction;   // X > counts_per_cell[:, None] * max_fraction
    for (int c = lane; c < g; c += 32) if (row[c] > lim) excl[c] = 1;
  }
}

// pass B: per-cell counts over the included genes; positives copied for the median
__global__ void __launch_bounds__(256)
norm_counts_kernel(const float* __restrict__ X, int64_t ldx, int32_t n, int32_t g, const int32_t* __restrict__ excl,
                   float* __restrict__ counts, float* __restrict__ pos_keys, int32_t* __restrict__ n_pos) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  int local_pos = 0;
  for (int64_t r = warp; r < n; r += nwarps) {
    const float c = row_sum_warp(X + r * ldx, g, excl, lane);
    if (lane == 0) {
      counts[r] = c;
      if (pos_keys) pos_keys[r] = c > 0.f ? c : CUDART_INF_F;
      local_pos += c > 0.f ? 1 : 0;
    }
  }
  if (lane == 0 && n_pos && local_pos) atomicAdd(n_pos, local_pos);
}

__global__ void norm_median_kernel(const float* __restrict__ sorted, const int32_t* __restrict__ n_pos,
                                   float* __restrict__ target) {
  const int m = *n_pos;
  if (m <= 0) { *target = 1.f; return; }
  const float a = sorted[(m - 1) / 2], b = sorted[m / 2];
  *target = (m & 1) ? a : (a + b) * 0.5f;   // np.median on float32
}

// pass C / fused single pass
__global__ void __launch_bounds__(256)
norm_apply_kernel(float* __restrict__ X, int64_t ldx, int32_t n, int32_t g, const float* __restrict__ counts,
                  const float* __restrict__ target_dev, float target_val, int do_normalize, int do_log1p,
                  float inv_log_base_div) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const float target = target_dev ? *target_dev : target_val;
  for (int64_t r = warp; r < n; r += nwarps) {
    float* row = X + r * ldx;
    float scale = 1.f;
    if (do_normalize) {
      const float c = counts ? counts[r] : row_sum_warp(row, g, nullptr, lane);
      scale = c / target;              // counts_per_cell / after
      if (scale == 0.f) scale = 1.f;   // zero-count cells are left unchanged (scanpy >= 1.10.1)
    }
    const bool vec = (reinterpret_cast<uintptr_t>(row) & 15) == 0;
    auto f = [&](float v) {
      if (do_normalize) v = v / scale;
      if (do_log1p) { v = log1pf(v); if (inv_log_base_div != 0.f) v = v / inv_log_base_div; }
      return v;
    };
    if (vec) {
      const int g4 = g >> 2;
      float4* r4 = reinterpret_cast<float4*>(row);
      for (int c = lane; c < g4; c += 32) {
        float4 v = r4[c];
        v.x = f(v.x); v.y = f(v.y); v.z = f(v.z); v.w = f(v.w);
        r4[c] = v;
      }
      for (int c = (g4 << 2) + lane; c < g; c += 32) row[c] = f(row[c]);
    } else {
      for (int c = lane; c < g; c += 32) row[c] = f(row[c]);
    }
  }
}

}  // namespace b2

using namespace b2;

extern "C" size_t b2_normalize_total_workspace_bytes(int32_t n, int32_t g) {
  size_t temp = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, temp, (const float*)nullptr, (float*)nullptr, (int)n);
  return align_up(temp, 256) + 3 * align_up((size_t)n * 4, 256) + align_up((size_t)g * 4, 256) + 1024;
}

extern "C" int b2_normalize_total_log1p_f32(float* X, int64_t ldx, int32_t n, int32_t g, float target_sum,
                                            float max_fraction, int do_normalize, int do_log1p, float base,
                                            void* workspace, size_t workspace_bytes, void* stream) {
  B2_REQUIRE(X && n >= 0 && g > 0 && ldx >= g, "b2_normalize_total_log1p_f32: bad arguments");
  if (n == 0) return B2_OK;
  cudaStream_t st = as_stream(stream);
  const float log_base = (do_log1p && base > 0.f) ? (float)log((double)base) : 0.f;
  const bool exclude = do_normalize && max_fraction < 1.f;
  const bool median = do_normalize && !(target_sum > 0.f);
  if (!exclude && !median) {
    norm_apply_kernel<<<grid_blocks(n, 8), 256, 0, st>>>(X, ldx, n, g, nullptr, nullptr, target_sum, do_normalize, do_log1p,
                                                         log_base);
    B2_CHECK_LAUNCH("norm_apply_kernel");
    return B2_OK;
  }
  B2_REQUIRE(workspace && workspace_bytes >= b2_normalize_total_workspace_bytes(n, g),
             "b2_normalize_total_log1p_f32: workspace too small");
  char* ws = reinterpret_cast<char*>(workspace);
  size_t off = 0;
  float* counts = reinterpret_cast<float*>(ws + off); off += align_up((size_t)n * 4, 256);
  float* keys = reinterpret_cast<float*>(ws + off); off += align_up((size_t)n * 4, 256);
  float* sorted = reinterpret_cast<float*>(ws + off); off += align_up((size_t)n * 4, 256);
  int32_t* excl = reinterpret_cast<int32_t*>(ws + off); off += align_up((size_t)g * 4, 256);
  int32_t* n_pos = reinterpret_cast<int32_t*>(ws + off);
  float* target_dev = reinterpret_cast<float*>(ws + off + 16);
  off += 256;
  void* d_temp = ws + off;
  size_t temp = workspace_bytes - off;
  B2_CHECK_CUDA(cudaMemsetAsync(n_pos, 0, 64, st));
  if (exclude) {
    B2_CHECK_CUDA(cudaMemsetAsync(excl, 0, sizeof(int32_t) * (size_t)g, st));
    norm_flag_kernel<<<grid_blocks(n, 8), 256, 0, st>>>(X, ldx, n, g, max_fraction, excl);
    B2_CHECK_LAUNCH("norm_flag_kernel");
  }
  norm_counts_kernel<<<grid_blocks(n, 8), 256, 0, st>>>(X, ldx, n, g, exclude ? excl : nullptr, counts,
                                                        median ? keys : nullptr, median ? n_pos : nullptr);
  B2_CHECK_LAUNCH("norm_counts_kernel");
  if (median) {
    B2_CHECK_CUDA(cub::DeviceRadixSort::SortKeys(d_temp, temp, keys, sorted, (int)n, 0, 32, st));
    norm_median_kernel<<<1, 1, 0, st>>>(sorted, n_pos, target_dev);
    B2_CHECK_LAUNCH("norm_median_kernel");
  }
  norm_apply_kernel<<<grid_blocks(n, 8), 256, 0, st>>>(X, ldx, n, g, counts, median ? target_dev : nullptr, target_sum,
                                                       do_normalize, do_log1p, log_base);
  B2_CHECK_LAUNCH("norm_apply_kernel");
  return B2_OK;
}
