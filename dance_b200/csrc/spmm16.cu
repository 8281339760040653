// CSR SpMM with a 16-bit dense operand:  Y = act(reduce(A · X16) + bias),  X16 stored as bf16 or fp16, fp32 accumulation.
//
// Same contract as b2_spmm_csr_f32 (spmm.cu) — torch.spmm(adj, support) scgnn2.py:500, DGL update_all(u_mul_e, sum|mean)
// gnn.py:90 / graphsci.py:112-115 — for the reduced-precision configurations (BASELINE config 3 "GraphSCI … bf16", SURVEY
// §8(b)4 `b2_spmm_csr_f32/bf16`).  The aggregate is bound by the gather stream nnz·F·sizeof(x) through L2:
// halving the element size halves the bytes every non-zero pulls, and at 1 M cells × 32 features the operand (64 MB instead
// of 128 MB) comes closer to fitting the 50 MB L2, so fewer gathers spill to HBM.
//
// Layout: a sub-warp group of G lanes owns one output row, lane gl owns features [8·gl, 8·gl+8) (one 16-byte gather per
// non-zero).  The group prefetches up to 32 (col, val) pairs with coalesced loads, then issues the gathers in batches of 8
// independent 16-byte loads per lane before the FMAs consume them.  Accumulation order = CSR order (deterministic).
#include "common.cuh"

#include <cuda_bf16.h>
#include <cuda_fp16.h>

namespace b2 {
int spmm_stream_dispatch(int dtype, const int32_t* rowptr, const int32_t* colidx, const float* vals, const void* X, int64_t ldx, float* Y,
                         int64_t ldy, void* Y16, int64_t ldy16, int32_t n_rows, int32_t F, int reduce, int act, const float* bias,
                         cudaStream_t st);
namespace {

template <int DT> struct X16;
template <> struct X16<0> {   // bf16: the fp32 value is the 16 bits shifted into the high half
  static __device__ __forceinline__ void unpack(uint32_t u, float& a, float& b) {
    a = __uint_as_float(u << 16);
    b = __uint_as_float(u & 0xFFFF0000u);
  }
  static __device__ __forceinline__ uint32_t pack(float a, float b) {
    const __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&v);
  }
};
template <> struct X16<1> {   // fp16
  static __device__ __forceinline__ void unpack(uint32_t u, float& a, float& b) {
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&u));
    a = f.x; b = f.y;
  }
  static __device__ __forceinline__ uint32_t pack(float a, float b) {
    const __half2 v = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&v);
  }
};

__device__ __forceinline__ uint4 ldg_u4(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}

template <int G, int DT>
__global__ void __launch_bounds__(256, 3)
spmm_csr_x16_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx, const float* __restrict__ vals,
                    const uint4* __restrict__ X, int64_t ldx8, float* __restrict__ Y, int64_t ldy, uint4* __restrict__ Y16,
                    int64_t ldy8, int32_t n_rows, int32_t F8, int reduce, int act, const float* __restrict__ bias) {
  constexpr int RPW = 32 / G;                 // rows per warp
  constexpr int WIN = 32;                     // (col, val) pairs prefetched per window
  constexpr int PRE = WIN / G;                // pairs held per lane
  constexpr int TCH = 8;                      // gathers in flight per lane
  const int lane = threadIdx.x & 31;
  const int sub = lane / G, gl = lane % G;
  const unsigned gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (sub * G));
  const bool own = gl < F8;
  const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;

  for (int64_t row = warp0 * RPW + sub; row < n_rows; row += nwarps * RPW) {
    const int32_t start = __ldg(rowptr + row), end = __ldg(rowptr + row + 1);
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    for (int32_t base = start; base < end; base += WIN) {
      int32_t pc[PRE];
      float pw[PRE];
#pragma unroll
      for (int q = 0; q < PRE; ++q) {
        const int32_t e = base + q * G + gl;
        pc[q] = -1;
        pw[q] = 0.f;
        if (e < end) {
          pc[q] = __ldg(colidx + e);
          pw[q] = vals ? __ldg(vals + e) : 1.f;
        }
      }
#pragma unroll
      for (int b = 0; b < WIN / TCH; ++b) {
        if (base + b * TCH >= end) break;     // uniform inside the group
        uint4 x[TCH];
        float w[TCH];
#pragma unroll
        for (int t = 0; t < TCH; ++t) {
          const int idx = b * TCH + t;
          const int32_t cc = __shfl_sync(gmask, pc[idx / G], idx % G, G);
          w[t] = __shfl_sync(gmask, pw[idx / G], idx % G, G);
          x[t] = make_uint4(0u, 0u, 0u, 0u);
          if (cc >= 0 && own) x[t] = ldg_u4(X + (int64_t)cc * ldx8 + gl);
        }
#pragma unroll
        for (int t = 0; t < TCH; ++t) {
          float a, c;
          X16<DT>::unpack(x[t].x, a, c); acc[0] = fmaf(w[t], a, acc[0]); acc[1] = fmaf(w[t], c, acc[1]);
          X16<DT>::unpack(x[t].y, a, c); acc[2] = fmaf(w[t], a, acc[2]); acc[3] = fmaf(w[t], c, acc[3]);
          X16<DT>::unpack(x[t].z, a, c); acc[4] = fmaf(w[t], a, acc[4]); acc[5] = fmaf(w[t], c, acc[5]);
          X16<DT>::unpack(x[t].w, a, c); acc[6] = fmaf(w[t], a, acc[6]); acc[7] = fmaf(w[t], c, acc[7]);
        }
      }
    }
    if (!own) continue;
    const float scale = (reduce == 1 && end > start) ? 1.f / (float)(end - start) : 1.f;   // DGL fn.mean
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float o = acc[i] * scale;
      if (bias) o += __ldg(bias + gl * 8 + i);
      acc[i] = apply_act(o, act);
    }
    if (Y) {
      float4* y = reinterpret_cast<float4*>(Y + row * ldy + gl * 8);
      stg_stream_f4(y, make_float4(acc[0], acc[1], acc[2], acc[3]));
      stg_stream_f4(y + 1, make_float4(acc[4], acc[5], acc[6], acc[7]));
    }
    if (Y16) {
      uint4 o;
      o.x = X16<DT>::pack(acc[0], acc[1]); o.y = X16<DT>::pack(acc[2], acc[3]);
      o.z = X16<DT>::pack(acc[4], acc[5]); o.w = X16<DT>::pack(acc[6], acc[7]);
      Y16[row * ldy8 + gl] = o;
    }
  }
}

template <int G, int DT>
int launch_x16(const int32_t* rowptr, const int32_t* colidx, const float* vals, const void* X, int64_t ldx, float* Y, int64_t ldy,
               void* Y16, int64_t ldy16, int32_t n_rows, int32_t F, int reduce, int act, const float* bias, cudaStream_t st) {
  constexpr int RPW = 32 / G;
  const int threads = 256;
  int64_t blocks = ceil_div<int64_t>(ceil_div<int64_t>(n_rows, RPW), threads / 32);
  const int64_t max_blocks = (int64_t)sm_count() * 64;   // grid-stride beyond this
  if (blocks > max_blocks) blocks = max_blocks;
  if (blocks < 1) blocks = 1;
  spmm_csr_x16_kernel<G, DT><<<(unsigned)blocks, threads, 0, st>>>(rowptr, colidx, vals, reinterpret_cast<const uint4*>(X), ldx / 8, Y,
                                                                  ldy, reinterpret_cast<uint4*>(Y16), ldy16 / 8, n_rows, F / 8, reduce,
                                                                  act, bias);
  B2_CHECK_LAUNCH("spmm_csr_x16_kernel");
  return B2_OK;
}

template <int DT>
int dispatch_x16(const char* name, const int32_t* rowptr, const int32_t* colidx, const float* vals, const void* X, int64_t ldx, float* Y,
                 int64_t ldy, void* Y16, int64_t ldy16, int32_t n_rows, int32_t n_cols, int32_t F, int reduce, int act,
                 const float* bias, void* stream) {
  B2_REQUIRE(rowptr && colidx && X && (Y || Y16), "%s: null pointer", name);
  B2_REQUIRE(n_rows >= 0 && n_cols >= 0, "%s: negative shape", name);
  B2_REQUIRE(F > 0 && F % 8 == 0 && F <= 256, "%s: F=%d must be a multiple of 8 in [8, 256] (slice wider feature blocks)", name, F);
  B2_REQUIRE(ldx % 8 == 0 && ldx >= F && (reinterpret_cast<uintptr_t>(X) & 15) == 0, "%s: X rows must be 16-byte aligned (ldx=%lld)", name,
             (long long)ldx);
  B2_REQUIRE(!Y || (ldy % 4 == 0 && ldy >= F && (reinterpret_cast<uintptr_t>(Y) & 15) == 0), "%s: Y rows must be 16-byte aligned", name);
  B2_REQUIRE(!Y16 || (ldy16 % 8 == 0 && ldy16 >= F && (reinterpret_cast<uintptr_t>(Y16) & 15) == 0), "%s: Y16 rows must be 16-byte aligned",
             name);
  B2_REQUIRE(reduce == 0 || reduce == 1, "%s: reduce must be 0 (sum) or 1 (mean)", name);
  if (n_rows == 0) return B2_OK;
  cudaStream_t st = as_stream(stream);
  {
    const int rc = spmm_stream_dispatch(DT, rowptr, colidx, vals, X, ldx, Y, ldy, Y16, ldy16, n_rows, F, reduce, act, bias, st);
    if (rc != 1) return rc;
  }
  const int F8 = F / 8;
#define B2_X16_CASE(G) return launch_x16<G, DT>(rowptr, colidx, vals, X, ldx, Y, ldy, Y16, ldy16, n_rows, F, reduce, act, bias, st)
  if (F8 <= 1) B2_X16_CASE(1);
  if (F8 <= 2) B2_X16_CASE(2);
  if (F8 <= 4) B2_X16_CASE(4);
  if (F8 <= 8) B2_X16_CASE(8);
  if (F8 <= 16) B2_X16_CASE(16);
  B2_X16_CASE(32);
#undef B2_X16_CASE
}

template <int DT>
__global__ void __launch_bounds__(256)
convert_x16_kernel(const float* __restrict__ src, int64_t lds, uint32_t* __restrict__ dst, int64_t ldd2, int64_t rows, int32_t cols2) {
  const int64_t total = rows * cols2;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / cols2;
    const int c = (int)(t % cols2);
    const float2 v = *reinterpret_cast<const float2*>(src + r * lds + 2 * c);
    dst[r * ldd2 + c] = X16<DT>::pack(v.x, v.y);
  }
}

}  // namespace
}  // namespace b2

extern "C" int b2_spmm_csr_bf16(const int32_t* rowptr, const int32_t* colidx, const float* vals, const void* X, int64_t ldx, float* Y,
                                int64_t ldy, void* Y16, int64_t ldy16, int32_t n_rows, int32_t n_cols, int32_t F, int reduce, int act,
                                const float* bias, void* stream) {
  return b2::dispatch_x16<0>("b2_spmm_csr_bf16", rowptr, colidx, vals, X, ldx, Y, ldy, Y16, ldy16, n_rows, n_cols, F, reduce, act, bias,
                             stream);
}

extern "C" int b2_spmm_csr_f16(const int32_t* rowptr, const int32_t* colidx, const float* vals, const void* X, int64_t ldx, float* Y,
                               int64_t ldy, void* Y16, int64_t ldy16, int32_t n_rows, int32_t n_cols, int32_t F, int reduce, int act,
                               const float* bias, void* stream) {
  return b2::dispatch_x16<1>("b2_spmm_csr_f16", rowptr, colidx, vals, X, ldx, Y, ldy, Y16, ldy16, n_rows, n_cols, F, reduce, act, bias,
                             stream);
}

extern "C" int b2_convert_f32_to_x16(const float* src, int64_t lds, void* dst, int64_t ldd, int64_t rows, int32_t cols, int dtype,
                                     void* stream) {
  using namespace b2;
  B2_REQUIRE(src && dst, "b2_convert_f32_to_x16: null pointer");
  B2_REQUIRE(dtype == 0 || dtype == 1, "b2_convert_f32_to_x16: dtype must be 0 (bf16) or 1 (fp16)");
  B2_REQUIRE(cols > 0 && cols % 2 == 0 && lds % 2 == 0 && ldd % 2 == 0 && lds >= cols && ldd >= cols,
             "b2_convert_f32_to_x16: cols and leading dimensions must be even (cols=%d lds=%lld ldd=%lld)", cols, (long long)lds,
             (long long)ldd);
  B2_REQUIRE((reinterpret_cast<uintptr_t>(src) & 7) == 0 && (reinterpret_cast<uintptr_t>(dst) & 3) == 0, "b2_convert_f32_to_x16: alignment");
  if (rows <= 0) return B2_OK;
  const int64_t total = rows * (cols / 2);
  int64_t blocks = ceil_div<int64_t>(total, 256 * 4);
  const int64_t cap = (int64_t)sm_count() * 32;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  cudaStream_t st = as_stream(stream);
  if (dtype == 0) convert_x16_kernel<0><<<(unsigned)blocks, 256, 0, st>>>(src, lds, reinterpret_cast<uint32_t*>(dst), ldd / 2, rows, cols / 2);
  else convert_x16_kernel<1><<<(unsigned)blocks, 256, 0, st>>>(src, lds, reinterpret_cast<uint32_t*>(dst), ldd / 2, rows, cols / 2);
  B2_CHECK_LAUNCH("convert_x16_kernel");
  return B2_OK;
}
