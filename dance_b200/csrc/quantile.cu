// scGNN's `normalizer(X, base)` (scgnn2.py:795-805) on the device: exact numpy quantiles of a whole fp32 matrix plus sklearn's
// minmax_scale of the columns of another one, fused into the concatenation that feeds the next autoencoder
// (feature_AE_handler scgnn2.py:283-294, graph_AE_handler scgnn2.py:543-546, clustering_handler scgnn2.py:155-157).
//   * b2_quantiles_f32  : np.quantile(base, q) (method "linear", q cast to float32) by radix select on the order-preserving
//                         uint32 key.  All order statistics of up to two q share three histogram passes over `base`
//                         (11 / 11 / 10 key bits); pass 1 also collects min, max and the number of non-finite values.  Counts and
//                         ranks are 64-bit (a 1 M × 2 000 base has 2·10⁹ elements).  Nothing leaves the device between passes.
//   * b2_col_minmax_f32 : per-column min / max (NaN ignored, like np.nanmin) — MinMaxScaler.partial_fit's data_min_ / data_max_.
//   * b2_concat_scaled_f32 : out = [left | right·scale_ + min_] (or the raw right), each of sklearn's two operations rounded on
//                         its own (`X *= scale_; X += min_`, never a fused multiply-add), padding columns zeroed.
// -0.0 is keyed as +0.0: numpy's partition does not order the two zeros, so neither does this.
#include "common.cuh"

#include <cmath>
#include <cub/block/block_scan.cuh>

namespace b2 {
namespace {

constexpr int kMaxRanks = 4;          // previous and next order statistic of up to two quantiles
constexpr int kHistThreads = 256;
constexpr int kScanThreads = 256;

__device__ __forceinline__ uint32_t float_key(float x) {
  uint32_t u = __float_as_uint(x);
  if (u == 0x80000000u) u = 0u;                          // -0.0 → +0.0
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float key_float(uint32_t k) {
  const uint32_t u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
#ifdef __CUDA_ARCH__
  return __uint_as_float(u);
#else
  float f;
  memcpy(&f, &u, sizeof f);
  return f;
#endif
}

// Per pass: bits of the key already fixed (prefix), bin bits of this pass, bins.
template <int PASS> struct PassGeom;
template <> struct PassGeom<0> { static constexpr int kShift = 21, kBins = 2048; };
template <> struct PassGeom<1> { static constexpr int kShift = 10, kBins = 2048; };
template <> struct PassGeom<2> { static constexpr int kShift = 0, kBins = 1024; };

// Selection state, device-resident between the passes.
struct SelState {
  uint32_t pref[kMaxRanks];          // key bits fixed so far for each wanted rank
  unsigned long long rem[kMaxRanks]; // rank still to skip inside that prefix
  uint32_t slot_pref[kMaxRanks];     // distinct prefixes histogrammed by the next pass
  int32_t rank_slot[kMaxRanks];
  int32_t nslots;
  uint32_t kmin, kmax;
  unsigned long long nonfinite;
};

// What the host derives from n and q alone (float32 arithmetic of numpy's _get_indexes / _get_gamma).
struct QuantPlan {
  long long rank[kMaxRanks];          // 2j: previous index of q_j, 2j+1: next index
  float gamma[2];
  int nq;
};

constexpr size_t kHistWords = 2048 + kMaxRanks * 2048 + kMaxRanks * 1024;   // u64 bins of the three passes

// Walks every element of a [rows, cols] matrix with row pitch ld: the whole grid strides over it as one flat run when the rows
// are dense, one warp per row otherwise; 16-byte loads where the layout allows.
template <class F>
__device__ __forceinline__ void for_each_element(const float* __restrict__ x, int64_t ld, int64_t rows, int64_t cols, F&& f) {
  const int lane = threadIdx.x & 31;
  const bool aligned = (reinterpret_cast<uintptr_t>(x) & 15) == 0;
  if (ld == cols || rows == 1) {
    const int64_t n = rows * cols;
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (int64_t)gridDim.x * blockDim.x;
    int64_t done = 0;
    if (aligned) {
      const int64_t n4 = n >> 2;
      const float4* x4 = reinterpret_cast<const float4*>(x);
      for (int64_t t = tid; t < n4; t += nth) {
        const float4 v = ldg_stream_f4(x4 + t);
        f(v.x); f(v.y); f(v.z); f(v.w);
      }
      done = n4 << 2;
    }
    for (int64_t t = done + tid; t < n; t += nth) f(__ldg(x + t));
    return;
  }
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const bool vec = aligned && (ld & 3) == 0;
  for (int64_t r = warp; r < rows; r += nwarps) {
    const float* row = x + r * ld;
    int64_t done = 0;
    if (vec) {
      const int64_t c4 = cols >> 2;
      const float4* row4 = reinterpret_cast<const float4*>(row);
      for (int64_t c = lane; c < c4; c += 32) {
        const float4 v = ldg_stream_f4(row4 + c);
        f(v.x); f(v.y); f(v.z); f(v.w);
      }
      done = c4 << 2;
    }
    for (int64_t c = done + lane; c < cols; c += 32) f(__ldg(row + c));
  }
}

// Shared-memory histogram increment, aggregated over the lanes of a warp that hit the same bin (zero-heavy expression data
// sends most of a warp to one bin).
__device__ __forceinline__ void hist_add(uint32_t* h, uint32_t bin) {
  const unsigned peers = __match_any_sync(__activemask(), bin);
  if ((threadIdx.x & 31) == (__ffs(peers) - 1)) atomicAdd(h + bin, (uint32_t)__popc(peers));
}

template <int PASS>
__global__ void __launch_bounds__(kHistThreads)
radix_hist_kernel(const float* __restrict__ x, int64_t ld, int64_t rows, int64_t cols, SelState* __restrict__ st,
                  unsigned long long* __restrict__ hist) {
  constexpr int kBins = PassGeom<PASS>::kBins, kShift = PassGeom<PASS>::kShift;
  __shared__ uint32_t sh[kMaxRanks * 2048];
  const int nslots = PASS == 0 ? 1 : st->nslots;
  uint32_t pref[kMaxRanks];
#pragma unroll
  for (int s = 0; s < kMaxRanks; ++s) pref[s] = PASS == 0 ? 0u : st->slot_pref[s];
  for (int t = threadIdx.x; t < nslots * kBins; t += blockDim.x) sh[t] = 0u;
  __syncthreads();
  uint32_t kmin = 0xffffffffu, kmax = 0u;
  unsigned long long nonfinite = 0;
  for_each_element(x, ld, rows, cols, [&](float v) {
    const uint32_t key = float_key(v);
    if (PASS == 0) {
      kmin = min(kmin, key);
      kmax = max(kmax, key);
      nonfinite += (__float_as_uint(v) & 0x7f800000u) == 0x7f800000u;
      hist_add(sh, key >> kShift);
    } else {
#pragma unroll
      for (int s = 0; s < kMaxRanks; ++s)
        if (s < nslots && (key >> (kShift + (PASS == 1 ? 11 : 10))) == pref[s]) hist_add(sh + s * kBins, (key >> kShift) & (kBins - 1));
    }
  });
  if (PASS == 0) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      kmin = min(kmin, __shfl_xor_sync(0xffffffffu, kmin, o));
      kmax = max(kmax, __shfl_xor_sync(0xffffffffu, kmax, o));
      nonfinite += __shfl_xor_sync(0xffffffffu, nonfinite, o);
    }
    if ((threadIdx.x & 31) == 0) {
      atomicMin(&st->kmin, kmin);
      atomicMax(&st->kmax, kmax);
      if (nonfinite) atomicAdd(&st->nonfinite, nonfinite);
    }
  }
  __syncthreads();
  for (int t = threadIdx.x; t < nslots * kBins; t += blockDim.x)
    if (sh[t]) atomicAdd(hist + t, (unsigned long long)sh[t]);
}

// One block: for every wanted rank, the bin of this pass that holds it (block-wide exclusive scan of the slot's histogram),
// then the distinct prefixes the next pass histograms.
template <int PASS>
__global__ void __launch_bounds__(kScanThreads)
radix_scan_kernel(const unsigned long long* __restrict__ hist, SelState* __restrict__ st, QuantPlan plan) {
  constexpr int kBins = PassGeom<PASS>::kBins, kPer = kBins / kScanThreads, kBits = PASS == 2 ? 10 : 11;
  using Scan = cub::BlockScan<unsigned long long, kScanThreads>;
  __shared__ typename Scan::TempStorage tmp;
  const int nranks = 2 * plan.nq;
#pragma unroll
  for (int r = 0; r < kMaxRanks; ++r) {
    if (r >= nranks) break;
    const int slot = PASS == 0 ? 0 : st->rank_slot[r];
    const unsigned long long rem = PASS == 0 ? (unsigned long long)plan.rank[r] : st->rem[r];
    const uint32_t pref = PASS == 0 ? 0u : st->pref[r];
    const unsigned long long* h = hist + (size_t)slot * kBins;
    unsigned long long c[kPer], tot = 0;
#pragma unroll
    for (int i = 0; i < kPer; ++i) { c[i] = h[threadIdx.x * kPer + i]; tot += c[i]; }
    unsigned long long excl;
    Scan(tmp).ExclusiveSum(tot, excl);
#pragma unroll
    for (int i = 0; i < kPer; ++i) {
      if (excl <= rem && rem < excl + c[i]) {
        st->pref[r] = (pref << kBits) | (uint32_t)(threadIdx.x * kPer + i);
        st->rem[r] = rem - excl;
      }
      excl += c[i];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    int ns = 0;
    for (int r = 0; r < nranks; ++r) {
      int s = 0;
      while (s < ns && st->slot_pref[s] != st->pref[r]) ++s;
      if (s == ns) st->slot_pref[ns++] = st->pref[r];
      st->rank_slot[r] = s;
    }
    st->nslots = ns;
  }
}

// numpy's _lerp in float32, each operation rounded: a + (b−a)·t, or b − (b−a)·(1−t) when t ≥ 0.5.
__device__ __forceinline__ float np_lerp(float a, float b, float t) {
  const float d = __fsub_rn(b, a);
  return t >= 0.5f ? __fsub_rn(b, __fmul_rn(d, __fsub_rn(1.f, t))) : __fadd_rn(a, __fmul_rn(d, t));
}

__global__ void quantile_finish_kernel(const SelState* __restrict__ st, QuantPlan plan, double* __restrict__ out) {
#pragma unroll
  for (int j = 0; j < 2; ++j)
    if (j < plan.nq) out[j] = (double)np_lerp(key_float(st->pref[2 * j]), key_float(st->pref[2 * j + 1]), plan.gamma[j]);
  out[plan.nq] = (double)key_float(st->kmin);
  out[plan.nq + 1] = (double)key_float(st->kmax);
  out[plan.nq + 2] = (double)st->nonfinite;
}

__global__ void sel_init_kernel(SelState* st) {
  st->kmin = 0xffffffffu;
  st->kmax = 0u;
  st->nonfinite = 0;
  st->nslots = 1;
}

// ---- column min / max ---------------------------------------------------------------------------------------------------------
// block = 32 columns × 8 row lanes; blocks stride over the rows, a grid row per 32-column tile.  Keys as above; NaN skipped.
__global__ void __launch_bounds__(256)
col_minmax_kernel(const float* __restrict__ x, int64_t ld, int64_t rows, int32_t cols, uint32_t* __restrict__ kmin,
                  uint32_t* __restrict__ kmax, unsigned long long* __restrict__ nonfinite) {
  __shared__ uint32_t smin[8][32], smax[8][32];
  const int cl = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int64_t c = (int64_t)blockIdx.y * 32 + cl;
  uint32_t lo = 0xffffffffu, hi = 0u;
  unsigned long long bad = 0;
  if (c < cols) {
    for (int64_t r = (int64_t)blockIdx.x * 8 + rl; r < rows; r += (int64_t)gridDim.x * 8) {
      const float v = __ldg(x + r * ld + c);
      const bool fin = (__float_as_uint(v) & 0x7f800000u) != 0x7f800000u;
      bad += !fin;
      if (v == v) { const uint32_t k = float_key(v); lo = min(lo, k); hi = max(hi, k); }
    }
  }
  smin[rl][cl] = lo;
  smax[rl][cl] = hi;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) bad += __shfl_xor_sync(0xffffffffu, bad, o);
  if (cl == 0 && bad) atomicAdd(nonfinite, bad);
  __syncthreads();
  if (rl == 0 && c < cols) {
    for (int i = 1; i < 8; ++i) { lo = min(lo, smin[i][cl]); hi = max(hi, smax[i][cl]); }
    atomicMin(kmin + c, lo);
    atomicMax(kmax + c, hi);
  }
}

__global__ void col_minmax_finish_kernel(const uint32_t* __restrict__ kmin, const uint32_t* __restrict__ kmax, int32_t cols,
                                         const unsigned long long* __restrict__ nonfinite, float* __restrict__ cmin,
                                         float* __restrict__ cmax, double* __restrict__ nonfinite_out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < cols) {
    // a column with no number at all keeps NaN, as np.nanmin of an all-NaN column
    cmin[c] = kmin[c] == 0xffffffffu ? __int_as_float(0x7fc00000) : key_float(kmin[c]);
    cmax[c] = kmax[c] == 0u ? __int_as_float(0x7fc00000) : key_float(kmax[c]);
  }
  if (c == 0 && nonfinite_out) *nonfinite_out = (double)*nonfinite;
}

__global__ void fill_u32_kernel(uint32_t* p, int64_t n, uint32_t v) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) p[i] = v;
}

// ---- widen -----------------------------------------------------------------------------------------------------------------------
// MinMaxScaler.partial_fit in float32 (sklearn/preprocessing/_data.py): scale_ = (hi − lo) / range with near-constant ranges
// (< 10·eps) set to 1, min_ = lo − data_min·scale_; then transform = (x·scale_) + min_, two rounded operations.
__device__ __forceinline__ void minmax_params(float dmin, float dmax, float lo, float hi, float& scale, float& shift) {
  float range = __fsub_rn(dmax, dmin);
  if (range < 10.f * 1.1920928955078125e-7f) range = 1.f;
  scale = __fdiv_rn(__fsub_rn(hi, lo), range);
  shift = __fsub_rn(lo, __fmul_rn(dmin, scale));
}
__device__ __forceinline__ float minmax_apply(float x, float scale, float shift) { return __fadd_rn(__fmul_rn(x, scale), shift); }

// scale_ / min_ of every column of `right` for the feature range (lo, hi); the division is the only rounding step here that
// is not a single IEEE operation in the kernel below, so it stays out of it.
__global__ void minmax_params_kernel(const float* __restrict__ cmin, const float* __restrict__ cmax, int32_t e, float lo, float hi,
                                     float* __restrict__ scale, float* __restrict__ shift) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < e) minmax_params(cmin[c], cmax[c], lo, hi, scale[c], shift[c]);
}

// One block per row group; each thread writes 16 bytes of out: columns [0, a) from left, [a, a+e) from right (scaled when
// SCALE), [a+e, ldo) zero.  ldo is a multiple of 4 and out 16-byte aligned.
template <bool SCALE>
__global__ void __launch_bounds__(256)
concat_kernel(const float* __restrict__ left, int64_t ldl, int32_t a, const float* __restrict__ right, int64_t ldr, int32_t e,
              int64_t rows, const float* __restrict__ scale, const float* __restrict__ shift, float* __restrict__ out, int64_t ldo) {
  const int64_t q4 = ldo >> 2;
  for (int64_t r = blockIdx.x; r < rows; r += gridDim.x) {
    const float* lr = left + r * ldl;
    const float* rr = right + r * ldr;
    float4* o = reinterpret_cast<float4*>(out + r * ldo);
    for (int64_t q = threadIdx.x; q < q4; q += blockDim.x) {
      float v[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int64_t c = q * 4 + i;
        if (c < a) {
          v[i] = __ldg(lr + c);
        } else if (c < (int64_t)a + e) {
          const int j = (int)(c - a);
          v[i] = SCALE ? minmax_apply(__ldg(rr + j), __ldg(scale + j), __ldg(shift + j)) : __ldg(rr + j);
        } else {
          v[i] = 0.f;
        }
      }
      stg_stream_f4(o + q, make_float4(v[0], v[1], v[2], v[3]));
    }
  }
}

}  // namespace
}  // namespace b2

extern "C" size_t b2_quantiles_workspace_bytes(void) {
  return b2::align_up(sizeof(b2::SelState), 256) + b2::kHistWords * sizeof(unsigned long long);
}

extern "C" int b2_quantiles_f32(const float* base, int64_t ldb, int64_t rows, int32_t cols, const float* qs, int32_t nq, double* out,
                                void* workspace, size_t workspace_bytes, void* stream) {
  using namespace b2;
  B2_REQUIRE(base && qs && out, "b2_quantiles_f32: null pointer");
  B2_REQUIRE(rows > 0 && cols > 0 && ldb >= cols, "b2_quantiles_f32: bad shape rows=%lld cols=%d ldb=%lld", (long long)rows, cols,
             (long long)ldb);
  B2_REQUIRE(nq >= 1 && nq <= 2, "b2_quantiles_f32: nq must be 1 or 2, got %d", nq);
  B2_REQUIRE(workspace && workspace_bytes >= b2_quantiles_workspace_bytes(), "b2_quantiles_f32: workspace too small");
  QuantPlan plan{};
  plan.nq = nq;
  const int64_t n = rows * (int64_t)cols;
  const float nm1 = (float)(n - 1);                    // numpy: (n − 1)·q with q float32 and n − 1 rounded to float32
  for (int j = 0; j < nq; ++j) {
    const float q = qs[j];
    B2_REQUIRE(q >= 0.f && q <= 1.f, "b2_quantiles_f32: quantile %g outside [0, 1]", (double)q);
    const float v = nm1 * q;
    if (v >= nm1) {                                     // _get_indexes: at or above the last index → the maximum
      plan.rank[2 * j] = plan.rank[2 * j + 1] = n - 1;
      plan.gamma[j] = 0.f;                              // lerp(a, a, ·) = a + 0 whatever the weight
    } else {
      const int64_t prev = (int64_t)std::floor(v);
      plan.rank[2 * j] = prev;
      plan.rank[2 * j + 1] = prev + 1 < n ? prev + 1 : n - 1;
      plan.gamma[j] = (float)((double)v - (double)prev);   // exact: the fractional part of a float32
    }
  }
  cudaStream_t s = as_stream(stream);
  char* w = reinterpret_cast<char*>(workspace);
  SelState* st = reinterpret_cast<SelState*>(w);
  unsigned long long* h0 = reinterpret_cast<unsigned long long*>(w + align_up(sizeof(SelState), 256));
  unsigned long long* h1 = h0 + 2048;
  unsigned long long* h2 = h1 + kMaxRanks * 2048;
  B2_CHECK_CUDA(cudaMemsetAsync(workspace, 0, b2_quantiles_workspace_bytes(), s));
  sel_init_kernel<<<1, 1, 0, s>>>(st);
  B2_CHECK_LAUNCH("sel_init_kernel");
  const int64_t per_launch = (ldb == cols || rows == 1) ? n / 4 : rows * 32;
  const unsigned g = grid_blocks(per_launch, kHistThreads, 8);
  radix_hist_kernel<0><<<g, kHistThreads, 0, s>>>(base, ldb, rows, cols, st, h0);
  B2_CHECK_LAUNCH("radix_hist_kernel<0>");
  radix_scan_kernel<0><<<1, kScanThreads, 0, s>>>(h0, st, plan);
  B2_CHECK_LAUNCH("radix_scan_kernel<0>");
  radix_hist_kernel<1><<<g, kHistThreads, 0, s>>>(base, ldb, rows, cols, st, h1);
  B2_CHECK_LAUNCH("radix_hist_kernel<1>");
  radix_scan_kernel<1><<<1, kScanThreads, 0, s>>>(h1, st, plan);
  B2_CHECK_LAUNCH("radix_scan_kernel<1>");
  radix_hist_kernel<2><<<g, kHistThreads, 0, s>>>(base, ldb, rows, cols, st, h2);
  B2_CHECK_LAUNCH("radix_hist_kernel<2>");
  radix_scan_kernel<2><<<1, kScanThreads, 0, s>>>(h2, st, plan);
  B2_CHECK_LAUNCH("radix_scan_kernel<2>");
  quantile_finish_kernel<<<1, 1, 0, s>>>(st, plan, out);
  B2_CHECK_LAUNCH("quantile_finish_kernel");
  return B2_OK;
}

extern "C" size_t b2_col_minmax_workspace_bytes(int32_t cols) {
  return b2::align_up(2 * (size_t)(cols > 0 ? cols : 0) * sizeof(uint32_t), 256) + 256;
}

extern "C" int b2_col_minmax_f32(const float* x, int64_t ldx, int64_t rows, int32_t cols, float* cmin, float* cmax, double* nonfinite,
                                 void* workspace, size_t workspace_bytes, void* stream) {
  using namespace b2;
  B2_REQUIRE(x && cmin && cmax, "b2_col_minmax_f32: null pointer");
  B2_REQUIRE(rows > 0 && cols > 0 && ldx >= cols, "b2_col_minmax_f32: bad shape rows=%lld cols=%d ldx=%lld", (long long)rows, cols,
             (long long)ldx);
  B2_REQUIRE(workspace && workspace_bytes >= b2_col_minmax_workspace_bytes(cols), "b2_col_minmax_f32: workspace too small");
  cudaStream_t s = as_stream(stream);
  char* w = reinterpret_cast<char*>(workspace);
  uint32_t* kmin = reinterpret_cast<uint32_t*>(w);
  uint32_t* kmax = kmin + cols;
  unsigned long long* bad = reinterpret_cast<unsigned long long*>(w + align_up(2 * (size_t)cols * sizeof(uint32_t), 256));
  B2_CHECK_CUDA(cudaMemsetAsync(kmax, 0, (size_t)cols * sizeof(uint32_t), s));
  B2_CHECK_CUDA(cudaMemsetAsync(bad, 0, sizeof(unsigned long long), s));
  fill_u32_kernel<<<ceil_div(cols, 256), 256, 0, s>>>(kmin, cols, 0xffffffffu);
  B2_CHECK_LAUNCH("fill_u32_kernel");
  const int tiles = ceil_div(cols, 32);
  int64_t gx = ceil_div<int64_t>(rows, 8 * 64);        // ≥ 64 rows per row lane
  const int64_t cap = ceil_div<int64_t>((int64_t)sm_count() * 16, tiles);
  gx = gx > cap ? cap : (gx < 1 ? 1 : gx);
  col_minmax_kernel<<<dim3((unsigned)gx, (unsigned)tiles), 256, 0, s>>>(x, ldx, rows, cols, kmin, kmax, bad);
  B2_CHECK_LAUNCH("col_minmax_kernel");
  col_minmax_finish_kernel<<<ceil_div(cols, 256), 256, 0, s>>>(kmin, kmax, cols, bad, cmin, cmax, nonfinite);
  B2_CHECK_LAUNCH("col_minmax_finish_kernel");
  return B2_OK;
}

extern "C" size_t b2_concat_scaled_workspace_bytes(int32_t e) { return b2::align_up(2 * (size_t)(e > 0 ? e : 0) * sizeof(float), 256); }

extern "C" int b2_concat_scaled_f32(const float* left, int64_t ldl, int32_t a, const float* right, int64_t ldr, int32_t e, int64_t rows,
                                    const float* cmin, const float* cmax, float lo, float hi, int scale, float* out, int64_t ldo,
                                    void* workspace, size_t workspace_bytes, void* stream) {
  using namespace b2;
  B2_REQUIRE(left && right && out, "b2_concat_scaled_f32: null pointer");
  B2_REQUIRE(rows >= 0 && a > 0 && e > 0 && ldl >= a && ldr >= e, "b2_concat_scaled_f32: bad shape a=%d e=%d", a, e);
  B2_REQUIRE(ldo >= (int64_t)a + e && (ldo & 3) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0,
             "b2_concat_scaled_f32: out needs a row pitch >= a + e that is a multiple of 4 and a 16-byte aligned base (ldo=%lld)",
             (long long)ldo);
  B2_REQUIRE(!scale || (cmin && cmax), "b2_concat_scaled_f32: scaling needs the column min / max");
  B2_REQUIRE(!scale || (workspace && workspace_bytes >= b2_concat_scaled_workspace_bytes(e)), "b2_concat_scaled_f32: workspace too small");
  if (rows == 0) return B2_OK;
  cudaStream_t s = as_stream(stream);
  const unsigned g = grid_blocks(rows, 1, 8);
  if (scale) {
    float* sc = reinterpret_cast<float*>(workspace);
    float* sh = sc + e;
    minmax_params_kernel<<<ceil_div(e, 128), 128, 0, s>>>(cmin, cmax, e, lo, hi, sc, sh);
    B2_CHECK_LAUNCH("minmax_params_kernel");
    concat_kernel<true><<<g, 256, 0, s>>>(left, ldl, a, right, ldr, e, rows, sc, sh, out, ldo);
    B2_CHECK_LAUNCH("concat_kernel<scale>");
  } else {
    concat_kernel<false><<<g, 256, 0, s>>>(left, ldl, a, right, ldr, e, rows, nullptr, nullptr, out, ldo);
    B2_CHECK_LAUNCH("concat_kernel<raw>");
  }
  return B2_OK;
}
