// dance.utils.matrix.normalize on the device (reference utils/matrix.py:8-67): along `axis`
//   normalize   : x / Σx            standardize : (x - mean) / std (population std)
//   minmax      : (x - min) / (max - min)        l2 : x / sqrt(Σx²)
// with the reference's denominator rule: eps == -1 → zero denominators become 1, eps > 0 → denom + eps.
// Statistics are accumulated in fp64 (numpy's pairwise fp32 sums are not reproducible bit-for-bit by any parallel order;
// fp64 keeps the result within an ulp of the exact value), three passes at most: (sum,min,max) → centred Σ² → apply.
// "vector" = one column (axis 0) or one row (axis 1); stats layout in the workspace: [sum | sumsq] doubles, [min | max] floats.
#include "common.cuh"

#include <math_constants.h>

namespace b2 {

enum { MN_NORMALIZE = 0, MN_STANDARDIZE = 1, MN_MINMAX = 2, MN_L2 = 3 };

__device__ __forceinline__ void atomic_min_f(float* a, float v) {
  // ordered-int trick valid for all finite floats (-0.0 is folded into +0.0 first)
  v += 0.f;
  if (v >= 0.f) atomicMin(reinterpret_cast<int*>(a), __float_as_int(v));
  else atomicMax(reinterpret_cast<unsigned int*>(a), __float_as_uint(v));
}
__device__ __forceinline__ void atomic_max_f(float* a, float v) {
  v += 0.f;
  if (v >= 0.f) atomicMax(reinterpret_cast<int*>(a), __float_as_int(v));
  else atomicMin(reinterpret_cast<unsigned int*>(a), __float_as_uint(v));
}

__global__ void mn_init_kernel(double* sum, double* sq, float* mn, float* mx, int nvec) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += gridDim.x * blockDim.x) {
    sum[i] = 0.0; sq[i] = 0.0; mn[i] = CUDART_INF_F; mx[i] = -CUDART_INF_F;
  }
}

// axis = 1: one warp per row.  pass 0: sum/min/max (+Σx² for l2) ; pass 1: Σ(x-mean)²
__global__ void __launch_bounds__(256)
mn_row_stats_kernel(const float* __restrict__ X, int64_t ldx, int32_t n, int32_t g, int pass, double* __restrict__ sum,
                    double* __restrict__ sq, float* __restrict__ mn, float* __restrict__ mx) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < n; r += nwarps) {
    const float* row = X + r * ldx;
    if (pass == 0) {
      double s = 0.0, q = 0.0;
      float lo = CUDART_INF_F, hi = -CUDART_INF_F;
      for (int c = lane; c < g; c += 32) { const float v = row[c]; s += v; q += (double)v * v; lo = fminf(lo, v); hi = fmaxf(hi, v); }
      s = warp_sum(s); q = warp_sum(q);
      for (int o = 16; o > 0; o >>= 1) { lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o)); hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o)); }
      if (lane == 0) { sum[r] = s; sq[r] = q; mn[r] = lo; mx[r] = hi; }
    } else {
      const double mean = sum[r] / (double)g;
      double q = 0.0;
      for (int c = lane; c < g; c += 32) { const double d = (double)row[c] - mean; q += d * d; }
      q = warp_sum(q);
      if (lane == 0) sq[r] = q;
    }
  }
}

// axis = 0: block = 32 columns × 8 row lanes, grid.y splits the rows; partials combined with atomics
__global__ void __launch_bounds__(256)
mn_col_stats_kernel(const float* __restrict__ X, int64_t ldx, int32_t n, int32_t g, int pass, double* __restrict__ sum,
                    double* __restrict__ sq, float* __restrict__ mn, float* __restrict__ mx) {
  __shared__ double ss[8][33], sqq[8][33];
  __shared__ float slo[8][33], shi[8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + tx;
  const int64_t rows_per = ceil_div<int64_t>(n, gridDim.y);
  const int64_t r0 = (int64_t)blockIdx.y * rows_per;
  const int64_t r1 = (r0 + rows_per < (int64_t)n) ? r0 + rows_per : (int64_t)n;
  double s = 0.0, q = 0.0;
  float lo = CUDART_INF_F, hi = -CUDART_INF_F;
  if (c < g) {
    if (pass == 0) {
      for (int64_t r = r0 + ty; r < r1; r += 8) { const float v = X[r * ldx + c]; s += v; q += (double)v * v; lo = fminf(lo, v); hi = fmaxf(hi, v); }
    } else {
      const double mean = sum[c] / (double)n;
      for (int64_t r = r0 + ty; r < r1; r += 8) { const double d = (double)X[r * ldx + c] - mean; q += d * d; }
    }
  }
  ss[ty][tx] = s; sqq[ty][tx] = q; slo[ty][tx] = lo; shi[ty][tx] = hi;
  __syncthreads();
  if (ty == 0 && c < g) {
    for (int i = 1; i < 8; ++i) { s += ss[i][tx]; q += sqq[i][tx]; lo = fminf(lo, slo[i][tx]); hi = fmaxf(hi, shi[i][tx]); }
    if (pass == 0) {
      atomicAdd(sum + c, s); atomicAdd(sq + c, q);
      if (r1 > r0) { atomic_min_f(mn + c, lo); atomic_max_f(mx + c, hi); }
    } else {
      atomicAdd(sq + c, q);
    }
  }
}

__global__ void mn_zero_sq_kernel(double* sq, int nvec) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += gridDim.x * blockDim.x) sq[i] = 0.0;
}

// shift / denominator per vector, in fp32 as numpy would hold them
__global__ void mn_finalize_kernel(const double* __restrict__ sum, const double* __restrict__ sq, const float* __restrict__ mn,
                                   const float* __restrict__ mx, int nvec, int len, int mode, float eps,
                                   float* __restrict__ shift, float* __restrict__ denom) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += gridDim.x * blockDim.x) {
    float sh = 0.f, d;
    if (mode == MN_NORMALIZE) d = (float)sum[i];
    else if (mode == MN_STANDARDIZE) { sh = -(float)(sum[i] / (double)len); d = (float)sqrt(sq[i] / (double)len); }
    else if (mode == MN_MINMAX) { sh = -mn[i]; d = mx[i] - mn[i]; }
    else d = (float)sqrt(sq[i]);
    if (eps == -1.f) { if (d == 0.f) d = 1.f; }
    else d += eps;
    shift[i] = sh; denom[i] = d;
  }
}

__global__ void __launch_bounds__(256)
mn_apply_kernel(const float* __restrict__ X, int64_t ldx, int32_t n, int32_t g, int axis, const float* __restrict__ shift,
                const float* __restrict__ denom, float* __restrict__ out, int64_t ldo) {
  const int64_t total = (int64_t)n * g;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / g;
    const int c = (int)(t - r * g);
    const int64_t v = axis == 0 ? c : r;
    out[r * ldo + c] = (X[r * ldx + c] + shift[v]) / denom[v];
  }
}

}  // namespace b2

using namespace b2;

static size_t mn_nvec(int32_t n, int32_t g, int axis) { return (size_t)(axis == 0 ? g : n); }

extern "C" size_t b2_matrix_normalize_workspace_bytes(int32_t n_rows, int32_t n_cols, int axis) {
  const size_t nv = mn_nvec(n_rows, n_cols, axis);
  return align_up(nv * 2 * sizeof(double), 256) + align_up(nv * 4 * sizeof(float), 256);
}

extern "C" int b2_matrix_normalize_f32(const float* X, int64_t ldx, int32_t n, int32_t g, int mode, int axis, float eps,
                                       float* out, int64_t ldo, void* workspace, size_t workspace_bytes, void* stream) {
  B2_REQUIRE(X && out && n >= 0 && g >= 0 && ldx >= g && ldo >= g, "b2_matrix_normalize_f32: bad arguments");
  B2_REQUIRE(mode >= 0 && mode <= 3 && (axis == 0 || axis == 1), "b2_matrix_normalize_f32: mode in 0..3, axis in {0,1}");
  B2_REQUIRE(eps == -1.f || eps > 0.f, "b2_matrix_normalize_f32: eps must be positive or -1 (utils/matrix.py:61)");
  if (n == 0 || g == 0) return B2_OK;
  B2_REQUIRE(workspace && workspace_bytes >= b2_matrix_normalize_workspace_bytes(n, g, axis),
             "b2_matrix_normalize_f32: workspace too small");
  cudaStream_t st = as_stream(stream);
  const int nv = (int)mn_nvec(n, g, axis);
  const int len = axis == 0 ? n : g;
  char* base = reinterpret_cast<char*>(workspace);
  double* sum = reinterpret_cast<double*>(base);
  double* sq = sum + nv;
  float* mn = reinterpret_cast<float*>(base + align_up((size_t)nv * 2 * sizeof(double), 256));
  float* mx = mn + nv;
  float* shift = mx + nv;
  float* denom = shift + nv;
  const unsigned small_grid = grid_blocks(nv, 256, 4);
  mn_init_kernel<<<small_grid, 256, 0, st>>>(sum, sq, mn, mx, nv);
  B2_CHECK_LAUNCH("mn_init_kernel");
  const int passes = mode == MN_STANDARDIZE ? 2 : 1;
  for (int pass = 0; pass < passes; ++pass) {
    if (axis == 1) {
      mn_row_stats_kernel<<<grid_blocks(n, 8), 256, 0, st>>>(X, ldx, n, g, pass, sum, sq, mn, mx);
      B2_CHECK_LAUNCH("mn_row_stats_kernel");
    } else {
      if (pass == 1) {
        mn_zero_sq_kernel<<<small_grid, 256, 0, st>>>(sq, nv);
        B2_CHECK_LAUNCH("mn_zero_sq_kernel");
      }
      const int col_tiles = ceil_div(g, 32);
      dim3 grid(col_tiles, row_splits(col_tiles, n, 64, 4));
      mn_col_stats_kernel<<<grid, 256, 0, st>>>(X, ldx, n, g, pass, sum, sq, mn, mx);
      B2_CHECK_LAUNCH("mn_col_stats_kernel");
    }
  }
  mn_finalize_kernel<<<small_grid, 256, 0, st>>>(sum, sq, mn, mx, nv, len, mode, eps, shift, denom);
  B2_CHECK_LAUNCH("mn_finalize_kernel");
  mn_apply_kernel<<<grid_blocks((int64_t)n * g, 1024), 256, 0, st>>>(X, ldx, n, g, axis, shift, denom, out, ldo);
  B2_CHECK_LAUNCH("mn_apply_kernel");
  return B2_OK;
}
