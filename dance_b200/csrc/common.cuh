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

static inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

template <typename T>
__host__ __device__ constexpr T ceil_div(T a, T b) { return (a + b - 1) / b; }

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

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

__device__ __forceinline__ float apply_act(float v, int act) {
  switch (act) {
    case B2_ACT_RELU: return fmaxf(v, 0.f);
    case B2_ACT_ELU: return v > 0.f ? v : expm1f(v);
    case B2_ACT_TANH: return tanhf(v);
    default: return v;
  }
}

}  // namespace b2
