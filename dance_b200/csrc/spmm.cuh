// Shared by the two CSR SpMM kernels (spmm.cu, spmm_stream.cu) and the fp32 → 16-bit conversion: the operand element types and
// the nnz-stream dispatch.
#pragma once
#include "common.cuh"

#include <cuda_bf16.h>
#include <cuda_fp16.h>

namespace b2 {

// Operand element type by type code: 2 = fp32, 0 = bf16, 1 = fp16.  A Vec is 16 bytes = N values; unpack turns one into fp32.
template <int DT> struct Elem {   // bf16 / fp16
  using Vec = uint4;
  static constexpr int N = 8;
  static __device__ __forceinline__ void unpack2(uint32_t u, float& a, float& b) {
    if constexpr (DT == 0) {        // bf16: the fp32 value is the 16 bits shifted into the high half
      a = __uint_as_float(u << 16);
      b = __uint_as_float(u & 0xffff0000u);
    } else {
      const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&u));
      a = f.x;
      b = f.y;
    }
  }
  // round-to-nearest-even
  static __device__ __forceinline__ uint32_t pack2(float a, float b) {
    if constexpr (DT == 0) {
      const __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
      return *reinterpret_cast<const uint32_t*>(&v);
    } else {
      const __half2 v = __floats2half2_rn(a, b);
      return *reinterpret_cast<const uint32_t*>(&v);
    }
  }
  static __device__ __forceinline__ void unpack(const uint4& x, float (&f)[8]) {
    unpack2(x.x, f[0], f[1]);
    unpack2(x.y, f[2], f[3]);
    unpack2(x.z, f[4], f[5]);
    unpack2(x.w, f[6], f[7]);
  }
};
template <> struct Elem<2> {
  using Vec = float4;
  static constexpr int N = 4;
  static __device__ __forceinline__ void unpack(const float4& x, float (&f)[4]) {
    f[0] = x.x;
    f[1] = x.y;
    f[2] = x.z;
    f[3] = x.w;
  }
};

// spmm_stream.cu: the nnz-stream kernel for operand rows of 32 / 64 / 128 bytes.  Returns B2_OK when it took the call, 1 when
// the shape is not one it handles (the caller runs the row-group kernel), < 0 on error.
int spmm_stream_dispatch(int dtype, const int32_t* rowptr, const int32_t* colidx, const float* vals, const void* X, int64_t ldx, float* Y,
                         int64_t ldy, void* Y16, int64_t ldy16, int32_t n_rows, int32_t F, int reduce, int act, const float* bias,
                         cudaStream_t st);

}  // namespace b2
