// NeighborGraph connectivities (reference transforms/graph/neighbor_graph.py:50-57 → scanpy.pp.neighbors(method="umap")
// → umap.umap_.fuzzy_simplicial_set; scanpy 1.10.1 / umap-learn 0.5 are un-vendored third-party code, their published
// algorithm is restated here and in oracle/port.py::umap_connectivities — parity unpinned at that boundary):
//   smooth_knn_dist        : per cell, rho = smallest positive neighbour distance, sigma by 64-step bisection so that
//                            Σ_{j>=1} exp(-max(d_j - rho, 0)/sigma) = log2(k); floors at 1e-3 × mean distance
//   membership strengths   : v_ij = 0 (self) | 1 (d <= rho or sigma = 0) | exp(-(d - rho)/sigma)
//   fuzzy union            : C = A + Aᵀ - A∘Aᵀ, explicit zeros dropped, CSR with ascending columns
// One thread per cell for the bisection when k <= 64 (fp64 bisection state like the numba code), one warp per cell above that
// (the lanes hold the cell's distances and each bisection step's fp64 sum is a warp reduction); the union is a sorted two-list
// merge per row over A and Aᵀ (b2_csr_transpose provides both with ascending columns).
#include "common.cuh"

#include <cub/device/device_scan.cuh>
#include <math_constants.h>

namespace b2 {

constexpr int UM_MAXK = 64;

__global__ void __launch_bounds__(256)
um_mean_kernel(const float* __restrict__ d, int64_t total, double* __restrict__ acc) {
  double s = 0.0;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) s += (double)d[t];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) atomicAdd(acc, s);
}

__global__ void __launch_bounds__(128)
um_smooth_kernel(const int32_t* __restrict__ knn_idx, const float* __restrict__ knn_dist, int32_t n, int32_t k,
                 const double* __restrict__ dist_sum, float* __restrict__ vals, float* __restrict__ sigmas,
                 float* __restrict__ rhos) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float d[UM_MAXK];
  float rho = 0.f, dmax = 0.f, dsum = 0.f;
  float first_pos = -1.f;
  int npos = 0;
  for (int j = 0; j < k; ++j) {
    d[j] = knn_dist[i * k + j];
    dsum += d[j];
    if (d[j] > 0.f) { if (npos == 0) first_pos = d[j]; ++npos; dmax = fmaxf(dmax, d[j]); }
  }
  // local_connectivity = 1: index = 1, interpolation = 0 → rho = non_zero_dists[0] (rows are sorted ascending)
  if (npos >= 1) rho = first_pos;
  else if (npos > 0) rho = dmax;
  const double target = log2((double)k);
  double lo = 0.0, hi = CUDART_INF, mid = 1.0;
  for (int it = 0; it < 64; ++it) {
    double psum = 0.0;
    for (int j = 1; j < k; ++j) {
      const float dd = d[j] - rho;
      psum += dd > 0.f ? exp(-((double)dd / mid)) : 1.0;
    }
    if (fabs(psum - target) < 1e-5) break;
    if (psum > target) { hi = mid; mid = (lo + hi) / 2.0; }
    else { lo = mid; if (hi == CUDART_INF) mid *= 2.0; else mid = (lo + hi) / 2.0; }
  }
  float sigma = (float)mid;
  if (rho > 0.f) {
    const float mean_i = dsum / (float)k;
    if (sigma < 1e-3f * mean_i) sigma = 1e-3f * mean_i;
  } else {
    const float mean_all = (float)(dist_sum[0] / ((double)n * k));
    if (sigma < 1e-3f * mean_all) sigma = 1e-3f * mean_all;
  }
  sigmas[i] = sigma;
  rhos[i] = rho;
  for (int j = 0; j < k; ++j) {
    float v;
    if (knn_idx[i * k + j] == (int32_t)i) v = 0.f;
    else if (d[j] - rho <= 0.f || sigma == 0.f) v = 1.f;
    else v = expf(-((d[j] - rho) / sigma));
    vals[i * k + j] = v;
  }
}

// um_smooth_kernel for k > UM_MAXK, one warp per cell.  rho, the σ floors and the memberships are um_smooth_kernel's
// arithmetic; only the order of each bisection step's fp64 sum differs (lanes, then a warp reduction).
constexpr int UM_WSLOTS = 16;   // distances a lane keeps in registers (k <= 512); longer rows are read again through L1

__global__ void __launch_bounds__(256)
um_smooth_warp_kernel(const int32_t* __restrict__ knn_idx, const float* __restrict__ knn_dist, int32_t n, int32_t k,
                      const double* __restrict__ dist_sum, float* __restrict__ vals, float* __restrict__ sigmas,
                      float* __restrict__ rhos) {
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += nwarps) {
    const float* drow = knn_dist + i * k;
    // in row order, the same in every lane (uniform loads): the fp32 sum, the first positive distance and the largest one
    float rho = 0.f, dmax = 0.f, dsum = 0.f;
    float first_pos = -1.f;
    int npos = 0;
    for (int j = 0; j < k; ++j) {
      const float dj = drow[j];
      dsum += dj;
      if (dj > 0.f) { if (npos == 0) first_pos = dj; ++npos; dmax = fmaxf(dmax, dj); }
    }
    if (npos >= 1) rho = first_pos;
    else if (npos > 0) rho = dmax;
    float dl[UM_WSLOTS];
#pragma unroll
    for (int u = 0; u < UM_WSLOTS; ++u) {
      const int j = lane + 32 * u;
      dl[u] = j < k ? drow[j] : 0.f;
    }
    const double target = log2((double)k);
    double lo = 0.0, hi = CUDART_INF, mid = 1.0;
    for (int it = 0; it < 64; ++it) {
      double psum = 0.0;
#pragma unroll
      for (int u = 0; u < UM_WSLOTS; ++u) {
        const int j = lane + 32 * u;
        const float dd = dl[u] - rho;
        if (j >= 1 && j < k) psum += dd > 0.f ? exp(-((double)dd / mid)) : 1.0;
      }
      for (int j = lane + 32 * UM_WSLOTS; j < k; j += 32) {
        const float dd = drow[j] - rho;
        psum += dd > 0.f ? exp(-((double)dd / mid)) : 1.0;
      }
      psum = warp_sum(psum);                       // xor butterfly: every lane holds the same bits
      if (fabs(psum - target) < 1e-5) break;
      if (psum > target) { hi = mid; mid = (lo + hi) / 2.0; }
      else { lo = mid; if (hi == CUDART_INF) mid *= 2.0; else mid = (lo + hi) / 2.0; }
    }
    float sigma = (float)mid;
    if (rho > 0.f) {
      const float mean_i = dsum / (float)k;
      if (sigma < 1e-3f * mean_i) sigma = 1e-3f * mean_i;
    } else {
      const float mean_all = (float)(dist_sum[0] / ((double)n * k));
      if (sigma < 1e-3f * mean_all) sigma = 1e-3f * mean_all;
    }
    if (lane == 0) { sigmas[i] = sigma; rhos[i] = rho; }
    for (int j = lane; j < k; j += 32) {
      const float dj = drow[j];
      float v;
      if (knn_idx[i * k + j] == (int32_t)i) v = 0.f;
      else if (dj - rho <= 0.f || sigma == 0.f) v = 1.f;
      else v = expf(-((dj - rho) / sigma));
      vals[i * k + j] = v;
    }
  }
}

// merge of row i of A and of Aᵀ (both ascending): value a + b - a·b, zeros dropped
template <bool FILL>
__global__ void __launch_bounds__(256)
um_union_kernel(const int32_t* __restrict__ rpA, const int32_t* __restrict__ ciA, const float* __restrict__ vA,
                const int32_t* __restrict__ rpT, const int32_t* __restrict__ ciT, const float* __restrict__ vT, int32_t n,
                int32_t* __restrict__ counts, const int32_t* __restrict__ rp_out, int32_t* __restrict__ ci_out,
                float* __restrict__ v_out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int32_t pa = rpA[i], ea = rpA[i + 1], pt = rpT[i], et = rpT[i + 1];
  int32_t cnt = 0;
  int32_t wp = FILL ? rp_out[i] : 0;
  while (pa < ea || pt < et) {
    const int32_t ca = pa < ea ? ciA[pa] : INT32_MAX, ct = pt < et ? ciT[pt] : INT32_MAX;
    const int32_t c = ca < ct ? ca : ct;
    float a = 0.f, b = 0.f;
    // duplicate columns inside one list (a cell listed twice among its neighbours) are summed, like coo → csr
    while (pa < ea && ciA[pa] == c) a += vA[pa++];
    while (pt < et && ciT[pt] == c) b += vT[pt++];
    const float v = a + b - a * b;
    if (v != 0.f) {
      if (FILL) { ci_out[wp] = c; v_out[wp] = v; ++wp; }
      else ++cnt;
    }
  }
  if (!FILL) counts[i] = cnt;
}

}  // namespace b2

using namespace b2;

extern "C" int b2_umap_fuzzy_knn_f32(const int32_t* knn_idx, const float* knn_dist, int32_t n, int32_t k, float* vals,
                                     float* sigmas, float* rhos, double* sum_ws, void* stream) {
  B2_REQUIRE(knn_idx && knn_dist && vals && sigmas && rhos && sum_ws && n >= 0 && k >= 2,
             "b2_umap_fuzzy_knn_f32: bad arguments (k >= 2)");
  if (n == 0) return B2_OK;
  cudaStream_t st = as_stream(stream);
  B2_CHECK_CUDA(cudaMemsetAsync(sum_ws, 0, sizeof(double), st));
  um_mean_kernel<<<grid_blocks((int64_t)n * k, 2048, 8), 256, 0, st>>>(knn_dist, (int64_t)n * k, sum_ws);
  B2_CHECK_LAUNCH("um_mean_kernel");
  if (k <= UM_MAXK) {
    um_smooth_kernel<<<ceil_div(n, 128), 128, 0, st>>>(knn_idx, knn_dist, n, k, sum_ws, vals, sigmas, rhos);
    B2_CHECK_LAUNCH("um_smooth_kernel");
  } else {
    um_smooth_warp_kernel<<<grid_blocks((int64_t)n * 32, 256), 256, 0, st>>>(knn_idx, knn_dist, n, k, sum_ws, vals, sigmas, rhos);
    B2_CHECK_LAUNCH("um_smooth_warp_kernel");
  }
  return B2_OK;
}

extern "C" size_t b2_fuzzy_union_workspace_bytes(int32_t n) {
  size_t temp = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, temp, (const int32_t*)nullptr, (int32_t*)nullptr, n + 1);
  return align_up(temp, 256) + align_up(sizeof(int32_t) * ((size_t)n + 1), 256);
}

extern "C" int b2_fuzzy_union_count(const int32_t* rowptr_a, const int32_t* colidx_a, const float* vals_a,
                                    const int32_t* rowptr_t, const int32_t* colidx_t, const float* vals_t, int32_t n,
                                    int32_t* rowptr_out, int64_t* nnz_host, void* workspace, size_t workspace_bytes,
                                    void* stream) {
  B2_REQUIRE(rowptr_a && colidx_a && vals_a && rowptr_t && colidx_t && vals_t && rowptr_out && nnz_host && n >= 0,
             "b2_fuzzy_union_count: bad arguments");
  B2_REQUIRE(workspace && workspace_bytes >= b2_fuzzy_union_workspace_bytes(n), "b2_fuzzy_union_count: workspace too small");
  cudaStream_t st = as_stream(stream);
  size_t temp = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, temp, (const int32_t*)nullptr, (int32_t*)nullptr, n + 1);
  char* base = reinterpret_cast<char*>(workspace);
  int32_t* counts = reinterpret_cast<int32_t*>(base + align_up(temp, 256));
  B2_CHECK_CUDA(cudaMemsetAsync(counts, 0, sizeof(int32_t) * ((size_t)n + 1), st));
  if (n > 0) {
    um_union_kernel<false><<<ceil_div(n, 256), 256, 0, st>>>(rowptr_a, colidx_a, vals_a, rowptr_t, colidx_t, vals_t, n, counts,
                                                            nullptr, nullptr, nullptr);
    B2_CHECK_LAUNCH("um_union_kernel<count>");
  }
  B2_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(base, temp, counts, rowptr_out, n + 1, st));
  int32_t total = 0;
  B2_CHECK_CUDA(cudaMemcpyAsync(&total, rowptr_out + n, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  B2_CHECK_CUDA(cudaStreamSynchronize(st));
  *nnz_host = total;
  return B2_OK;
}

extern "C" int b2_fuzzy_union_fill(const int32_t* rowptr_a, const int32_t* colidx_a, const float* vals_a,
                                   const int32_t* rowptr_t, const int32_t* colidx_t, const float* vals_t, int32_t n,
                                   const int32_t* rowptr_out, int32_t* colidx_out, float* vals_out, void* stream) {
  B2_REQUIRE(rowptr_a && colidx_a && vals_a && rowptr_t && colidx_t && vals_t && rowptr_out && colidx_out && vals_out && n >= 0,
             "b2_fuzzy_union_fill: bad arguments");
  if (n == 0) return B2_OK;
  um_union_kernel<true><<<ceil_div(n, 256), 256, 0, as_stream(stream)>>>(rowptr_a, colidx_a, vals_a, rowptr_t, colidx_t, vals_t, n,
                                                                        nullptr, rowptr_out, colidx_out, vals_out);
  B2_CHECK_LAUNCH("um_union_kernel<fill>");
  return B2_OK;
}
