// Shared helpers for the dance_b200 CUDA translation units (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>

#include "../../include/dance_b200.h"

namespace b2 {

// thread-local error message surfaced through b2_last_error()
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);
int sm_count();
const char* last_error();
int path_mode(int which);          // b2_set_path selector value (0 = automatic)
int tuning(int which);             // b2_set_tuning knob value
extern long long g_launch_count;   // kernels launched by this library (process-wide; see b2_launch_count)

#define B2_CHECK_CUDA(expr)                                   \
  do {                                                        \
    cudaError_t _e = (expr);                                  \
    if (_e != cudaSuccess) return b2::cuda_fail(_e, #expr);   \
  } while (0)

#define B2_CHECK_LAUNCH(name)                                 \
  do {                                                        \
    ++b2::g_launch_count;                                     \
    cudaError_t _e = cudaGetLastError();                      \
    if (_e != cudaSuccess) return b2::cuda_fail(_e, name);    \
  } while (0)

#define B2_REQUIRE(cond, ...)                                 \
  do {                                                        \
    if (!(cond)) {                                            \
      b2::set_error(__VA_ARGS__);                             \
      return B2_ERR_INVALID;                                  \
    }                                                         \
  } while (0)

// Dynamic shared memory a CTA may have on sm_90 once its kernel has opted in (227 KB; without the opt-in, 48 KB).
constexpr size_t kMaxDynamicSmem = 227 * 1024;

// Lets `kernel` launch with `bytes` of dynamic shared memory on the current device.  It raises the kernel's maximum-dynamic-
// shared-memory attribute when a (kernel, device) needs more than it has been allowed so far, and does nothing for requests of
// at most 48 KB (none of the opting-in kernels declares static shared memory).  The attribute belongs to the kernel as loaded
// on one device, so each device opts in separately.  It only permits a size; the carve-out, and so the occupancy, is
// unchanged.  Safe to call from several host threads.  Returns B2_OK or B2_ERR_CUDA.
int allow_dynamic_smem(const void* kernel, size_t bytes);

static inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

template <typename T>
__host__ __device__ constexpr T ceil_div(T a, T b) { return (a + b - 1) / b; }

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Grid-stride launch size: ceil(work / per_block) blocks, clamped to [1, sm_count() · blocks_per_sm].
static inline unsigned grid_blocks(int64_t work, int64_t per_block, int blocks_per_sm = 16) {
  const int64_t b = ceil_div(work, per_block), cap = (int64_t)sm_count() * blocks_per_sm;
  return (unsigned)(b < 1 ? 1 : b > cap ? cap : b);
}

// gridDim.y of a column-tiled reduction that splits its rows: ceil(sm_count() · waves / col_tiles), clamped to
// [1, max(rows / min_rows, 1)].
static inline int row_splits(int col_tiles, int64_t rows, int min_rows, int waves) {
  const int64_t s = ceil_div(sm_count() * waves, col_tiles), most = rows / min_rows > 1 ? rows / min_rows : 1;
  return (int)(s < 1 ? 1 : s > most ? most : s);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// streaming (read-once) 128-bit load that does not pollute L1
__device__ __forceinline__ float4 ldg_stream_f4(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ void stg_stream_f4(float4* p, const float4& v) {
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y),
               "f"(v.z), "f"(v.w));
}

// Counter-based uniform draw in (0, 1) of element (row, col) of stream `stream` under `seed`: no state, so a backward pass
// regenerates the forward's draws.  Used by CellwiseMaskData (prep.cu, streams 1 and 2) and by dropout (key = stream).
__device__ __forceinline__ uint32_t hash32(uint32_t x) {
  x ^= x >> 16; x *= 0x7FEB352Du; x ^= x >> 15; x *= 0x846CA68Bu; x ^= x >> 16;
  return x;
}
__device__ __forceinline__ float uniform01(uint32_t seed, uint32_t stream, uint32_t row, uint32_t col) {
  const uint32_t h = hash32(hash32(row + seed * 0x9E3779B1u + stream * 0x85EBCA77u) ^ hash32(col + stream * 0xC2B2AE3Du + 0x27D4EB2Fu));
  return ((float)(h >> 8) + 0.5f) * (1.f / 16777216.f);
}
// Dropout keep bit of element (r, c) under (seed, key): Bernoulli(1 - p); p = 0 keeps everything, p = 1 nothing.
__device__ __forceinline__ bool dropout_keep(uint32_t seed, uint32_t key, uint32_t r, uint32_t c, float p) {
  return uniform01(seed, key, r, c) >= p;
}

__device__ __forceinline__ float apply_act(float v, int act) {
  switch (act) {
    case B2_ACT_RELU: return fmaxf(v, 0.f);
    case B2_ACT_ELU: return v > 0.f ? v : expm1f(v);
    case B2_ACT_TANH: return tanhf(v);
    default: return v;
  }
}

// apply_act extended by leaky_relu and gelu, the codes the GEMM / SpMM / GAT-combine epilogues do not take (their code stays as
// it is).
__device__ __forceinline__ float act_value(float v, int act) {
  switch (act) {
    case B2_ACT_LEAKY_RELU: return v > 0.f ? v : 0.01f * v;
    case B2_ACT_GELU: return 0.5f * v * (1.f + erff(v * 0.70710678118654752f));
    default: return apply_act(v, act);
  }
}

// dy · act'(·) for every B2_ACT_* code: from the output *y for relu, elu, tanh and leaky_relu (y > 0 exactly where x > 0), from
// the pre-activation *x for gelu.  Only the operand the code needs is read, so the other may point anywhere (NONE reads neither).
// relu selects rather than multiplies, as torch's threshold_backward does: 0 wherever y <= 0, whatever dy is.
__device__ __forceinline__ float act_bwd(float dy, const float* y, const float* x, int act) {
  switch (act) {
    case B2_ACT_RELU: return *y > 0.f ? dy : 0.f;
    case B2_ACT_ELU: { const float v = *y; return dy * (v > 0.f ? 1.f : v + 1.f); }
    case B2_ACT_TANH: { const float v = *y; return dy * (1.f - v * v); }
    case B2_ACT_LEAKY_RELU: return dy * (*y > 0.f ? 1.f : 0.01f);
    case B2_ACT_GELU: { const float v = *x; return dy * (normcdff(v) + v * 0.39894228040143268f * __expf(-0.5f * v * v)); }
    default: return dy;
  }
}

}  // namespace b2
