// CSR SpMM  Y = act(reduce(A · X) + bias)  — the GCN / message-passing aggregate, for fp32, bf16 and fp16 operands.
//
// Replaces torch.spmm(adj, support) (reference scgnn2.py:500, spagcn.py:359,
// scdsc.py:498) and DGL update_all(u_mul_e, sum|mean) (gnn.py:90,
// graphsc.py:463-465); with a 16-bit operand, the reduced-precision configurations (BASELINE config 3 "GraphSCI … bf16",
// graphsci.py:112-115): every non-zero gathers F·2 instead of F·4 bytes.
//
// Operand rows of 32 / 64 / 128 bytes go to the nnz-stream kernel (spmm_stream.cu); every other width runs here.
//
// Layout: one sub-warp group of G lanes owns one output row; each lane owns
// VPL 16-byte vectors of the feature row (4 fp32 or 8 bf16 / fp16 values).  The group streams its (col, val)
// pairs G at a time with one coalesced load, then broadcasts them with
// shuffles while every lane issues G independent 16-byte gathers of X — the
// gathers are the traffic that matters (nnz · F · sizeof(x) bytes through L2), so the
// loop is organised to keep G of them in flight per lane.  Accumulation is in
// fp32 registers in CSR order (deterministic; same order as a sequential CPU
// CSR loop, which is what the oracle does), one fmaf chain per feature whatever the element type, G or VPL.
#include "spmm.cuh"

namespace b2 {

// One chunk of at most G entries of a row: lane t of the group holds the chunk's t-th (col, val) pair.
template <int DT, int G, int VPL, int TCH>
__device__ __forceinline__ void spmm_chunk(float (&acc)[VPL][Elem<DT>::N], int32_t c, float w, int cnt, unsigned gmask, int gl,
                                           const typename Elem<DT>::Vec* __restrict__ X, int64_t ldx, int32_t FV) {
  using E = Elem<DT>;
  using Vec = typename E::Vec;
  if (cnt == G) {
    // full chunk: G independent gathers in flight
    Vec x[TCH][VPL];
#pragma unroll
    for (int t0 = 0; t0 < G; t0 += TCH) {
#pragma unroll
      for (int t = 0; t < TCH; ++t) {
        const int32_t cc = __shfl_sync(gmask, c, t0 + t, G);
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          const int j = gl + v * G;
          x[t][v] = (j < FV) ? __ldg(X + (int64_t)cc * ldx + j) : Vec{};
        }
      }
#pragma unroll
      for (int t = 0; t < TCH; ++t) {
        const float ww = __shfl_sync(gmask, w, t0 + t, G);
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          float f[E::N];
          E::unpack(x[t][v], f);
#pragma unroll
          for (int i = 0; i < E::N; ++i) acc[v][i] = fmaf(ww, f[i], acc[v][i]);
        }
      }
    }
  } else {
    for (int t = 0; t < cnt; ++t) {
      const int32_t cc = __shfl_sync(gmask, c, t, G);
      const float ww = __shfl_sync(gmask, w, t, G);
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        const int j = gl + v * G;
        if (j < FV) {
          float f[E::N];
          E::unpack(__ldg(X + (int64_t)cc * ldx + j), f);
#pragma unroll
          for (int i = 0; i < E::N; ++i) acc[v][i] = fmaf(ww, f[i], acc[v][i]);
        }
      }
    }
  }
}

// X, ldx and FV count 16-byte vectors; Y4 / ldy4 float4s.  Y16 (16-bit types only) receives a copy of the result in the
// operand's type.
template <int DT, int G, int VPL>
__global__ void __launch_bounds__(256)
spmm_csr_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx, const float* __restrict__ vals,
                const typename Elem<DT>::Vec* __restrict__ X, int64_t ldx, float4* __restrict__ Y4, int64_t ldy4, int32_t n_rows,
                int32_t FV, int reduce, int act, const float* __restrict__ bias, uint4* __restrict__ Y16, int64_t ldy16) {
  using E = Elem<DT>;
  constexpr int N = E::N;
  constexpr int RPW = 32 / G;  // rows per warp
  // gathers issued back-to-back before the FMAs consume them (register budget: TCH*VPL vectors)
  constexpr int TCH = VPL >= 4 ? 2 : (VPL == 2 ? 4 : (G < 8 ? G : 8));
  const int lane = threadIdx.x & 31;
  const int sub = lane / G;
  const int gl = lane % G;
  const unsigned gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (sub * G));
  const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;

  for (int64_t row = warp0 * RPW + sub; row < n_rows; row += nwarps * RPW) {
    const int32_t start = __ldg(rowptr + row);
    const int32_t end = __ldg(rowptr + row + 1);
    float acc[VPL][N];
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
#pragma unroll
      for (int i = 0; i < N; ++i) acc[v][i] = 0.f;
    }

    // (col,val) pairs of the first PRE*G entries are fetched in ONE batch of independent loads (most kNN-graph rows
    // are shorter than that), so the dependent chain per row is rowptr → pairs → gathers instead of one round trip
    // per G-entry chunk.
    constexpr int PRE = (G <= 8) ? 4 : ((G == 16) ? 2 : 1);
    int32_t pc[PRE];
    float pw[PRE];
#pragma unroll
    for (int q = 0; q < PRE; ++q) {
      const int32_t e = start + q * G + gl;
      pc[q] = 0;
      pw[q] = 0.f;
      if (e < end) {
        pc[q] = __ldg(colidx + e);
        pw[q] = vals ? __ldg(vals + e) : 1.f;
      }
    }
    int32_t base = start;
#pragma unroll
    for (int q = 0; q < PRE; ++q) {
      if (base >= end) break;
      spmm_chunk<DT, G, VPL, TCH>(acc, pc[q], pw[q], min(G, end - base), gmask, gl, X, ldx, FV);
      base += G;
    }
    for (; base < end; base += G) {
      const int32_t e = base + gl;
      int32_t c = 0;
      float w = 0.f;
      if (e < end) {
        c = __ldg(colidx + e);
        w = vals ? __ldg(vals + e) : 1.f;
      }
      spmm_chunk<DT, G, VPL, TCH>(acc, c, w, min(G, end - base), gmask, gl, X, ldx, FV);
    }

    const float scale = (reduce == 1 && end > start) ? 1.f / (float)(end - start) : 1.f;
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int j = gl + v * G;
      if (j < FV) {
        float* o = acc[v];
        if (reduce == 1) {
          // DGL fn.mean divides the sum by the in-degree
#pragma unroll
          for (int i = 0; i < N; ++i) o[i] = o[i] * scale;
        }
        if (bias) {
          if constexpr (DT == 2) {
            const float4 bb = __ldg(reinterpret_cast<const float4*>(bias) + j);
            o[0] += bb.x; o[1] += bb.y; o[2] += bb.z; o[3] += bb.w;
          } else {
            // the 16-bit entry points take a bias that is only 4-byte aligned
#pragma unroll
            for (int i = 0; i < N; ++i) o[i] += __ldg(bias + j * N + i);
          }
        }
#pragma unroll
        for (int k = 0; k < N; k += 4) {  // written out per quad: as a loop over N, ptxas lays out the fp32 epilogue differently
          o[k] = apply_act(o[k], act); o[k + 1] = apply_act(o[k + 1], act);
          o[k + 2] = apply_act(o[k + 2], act); o[k + 3] = apply_act(o[k + 3], act);
        }
        if (DT == 2 || Y4) {
#pragma unroll
          for (int k = 0; k < N / 4; ++k)
            stg_stream_f4(Y4 + row * ldy4 + j * (N / 4) + k, make_float4(o[4 * k], o[4 * k + 1], o[4 * k + 2], o[4 * k + 3]));
        }
        if constexpr (DT != 2) {
          if (Y16) Y16[row * ldy16 + j] = make_uint4(E::pack2(o[0], o[1]), E::pack2(o[2], o[3]), E::pack2(o[4], o[5]), E::pack2(o[6], o[7]));
        }
      }
    }
  }
}

template <int DT, int G, int VPL>
static int launch_spmm(const int32_t* rowptr, const int32_t* colidx, const float* vals, const void* X, int64_t ldx, float* Y,
                       int64_t ldy, void* Y16, int64_t ldy16, int32_t n_rows, int32_t F, int reduce, int act, const float* bias,
                       cudaStream_t st) {
  using E = Elem<DT>;
  constexpr int RPW = 32 / G;
  const int threads = 256;
  const int64_t warps_needed = ceil_div<int64_t>(n_rows, RPW);
  spmm_csr_kernel<DT, G, VPL><<<grid_blocks(warps_needed, threads / 32, 64), threads, 0, st>>>(
      rowptr, colidx, vals, reinterpret_cast<const typename E::Vec*>(X), ldx / E::N, reinterpret_cast<float4*>(Y), ldy / 4, n_rows,
      F / E::N, reduce, act, bias, reinterpret_cast<uint4*>(Y16), ldy16 / 8);
  B2_CHECK_LAUNCH("spmm_csr_kernel");
  return B2_OK;
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// Validation, then the nnz-stream kernel where it takes the shape, then the row-group kernel.  Y16 is null for fp32.
template <int DT>
static int spmm_dispatch(const char* name, const int32_t* rowptr, const int32_t* colidx, const float* vals, const void* X, int64_t ldx,
                         float* Y, int64_t ldy, void* Y16, int64_t ldy16, int32_t n_rows, int32_t n_cols, int32_t F, int reduce,
                         int act, const float* bias, void* stream) {
  constexpr int N = Elem<DT>::N;
  B2_REQUIRE(rowptr && colidx && X && (Y || Y16), "%s: null pointer", name);
  B2_REQUIRE(n_rows >= 0 && n_cols >= 0, "%s: negative shape", name);
  B2_REQUIRE(F > 0 && F % N == 0, "%s: F=%d must be a positive multiple of %d", name, F, N);
  B2_REQUIRE(DT == 2 || F <= 256, "%s: F=%d > 256 (slice wider feature blocks)", name, F);
  B2_REQUIRE(ldx % N == 0 && ldx >= F && aligned16(X), "%s: X rows must be 16-byte aligned (ldx=%lld)", name, (long long)ldx);
  B2_REQUIRE(!Y || (ldy % 4 == 0 && ldy >= F && aligned16(Y)), "%s: Y rows must be 16-byte aligned (ldy=%lld)", name, (long long)ldy);
  B2_REQUIRE(!Y16 || (ldy16 % 8 == 0 && ldy16 >= F && aligned16(Y16)), "%s: Y16 rows must be 16-byte aligned (ldy16=%lld)", name,
             (long long)ldy16);
  B2_REQUIRE(reduce == 0 || reduce == 1, "%s: reduce must be 0 (sum) or 1 (mean)", name);
  B2_REQUIRE(DT != 2 || !bias || aligned16(bias), "%s: bias must be 16-byte aligned", name);
  if (n_rows == 0) return B2_OK;
  cudaStream_t st = as_stream(stream);
  {
    const int rc = spmm_stream_dispatch(DT, rowptr, colidx, vals, X, ldx, Y, ldy, Y16, ldy16, n_rows, F, reduce, act, bias, st);
    if (rc != 1) return rc;
  }
  const int nv = F / N;  // 16-byte vectors per row
#define B2_SPMM_CASE(G, VPL) \
  return launch_spmm<DT, G, VPL>(rowptr, colidx, vals, X, ldx, Y, ldy, Y16, ldy16, n_rows, F, reduce, act, bias, st)
  // G = 4 for one vector per row as well: a one-vector row at G = 1 or 2 keeps too few gathers in flight (measured on the H100
  // at fp32 F = 4 and bf16 / fp16 F = 8)
  if (nv <= 4) B2_SPMM_CASE(4, 1);
  if (nv <= 8) B2_SPMM_CASE(8, 1);
  if (nv <= 16) B2_SPMM_CASE(16, 1);
  if (nv <= 32) B2_SPMM_CASE(32, 1);
  if constexpr (DT == 2) {
    if (nv <= 64) B2_SPMM_CASE(32, 2);
    if (nv <= 128) B2_SPMM_CASE(32, 4);
  }
#undef B2_SPMM_CASE
  set_error("%s: F=%d > 512 unsupported (split the feature dimension)", name, F);
  return B2_ERR_UNSUPPORTED;
}

template <int DT>
__global__ void __launch_bounds__(256)
convert_x16_kernel(const float* __restrict__ src, int64_t lds, uint32_t* __restrict__ dst, int64_t ldd2, int64_t rows, int32_t cols2) {
  const int64_t total = rows * cols2;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / cols2;
    const int c = (int)(t % cols2);
    const float2 v = *reinterpret_cast<const float2*>(src + r * lds + 2 * c);
    dst[r * ldd2 + c] = Elem<DT>::pack2(v.x, v.y);
  }
}

}  // namespace b2

extern "C" int b2_spmm_csr_f32(const int32_t* rowptr, const int32_t* colidx, const float* vals,
                               const float* X, int64_t ldx, float* Y, int64_t ldy, int32_t n_rows,
                               int32_t n_cols, int32_t F, int reduce, int act, const float* bias, void* stream) {
  return b2::spmm_dispatch<2>("b2_spmm_csr_f32", rowptr, colidx, vals, X, ldx, Y, ldy, nullptr, 0, n_rows, n_cols, F, reduce, act, bias,
                              stream);
}

extern "C" int b2_spmm_csr_bf16(const int32_t* rowptr, const int32_t* colidx, const float* vals, const void* X, int64_t ldx, float* Y,
                                int64_t ldy, void* Y16, int64_t ldy16, int32_t n_rows, int32_t n_cols, int32_t F, int reduce, int act,
                                const float* bias, void* stream) {
  return b2::spmm_dispatch<0>("b2_spmm_csr_bf16", rowptr, colidx, vals, X, ldx, Y, ldy, Y16, ldy16, n_rows, n_cols, F, reduce, act, bias,
                              stream);
}

extern "C" int b2_spmm_csr_f16(const int32_t* rowptr, const int32_t* colidx, const float* vals, const void* X, int64_t ldx, float* Y,
                               int64_t ldy, void* Y16, int64_t ldy16, int32_t n_rows, int32_t n_cols, int32_t F, int reduce, int act,
                               const float* bias, void* stream) {
  return b2::spmm_dispatch<1>("b2_spmm_csr_f16", rowptr, colidx, vals, X, ldx, Y, ldy, Y16, ldy16, n_rows, n_cols, F, reduce, act, bias,
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
  const unsigned blocks = grid_blocks(rows * (cols / 2), 1024, 32);
  cudaStream_t st = as_stream(stream);
  if (dtype == 0) convert_x16_kernel<0><<<blocks, 256, 0, st>>>(src, lds, reinterpret_cast<uint32_t*>(dst), ldd / 2, rows, cols / 2);
  else convert_x16_kernel<1><<<blocks, 256, 0, st>>>(src, lds, reinterpret_cast<uint32_t*>(dst), ldd / 2, rows, cols / 2);
  B2_CHECK_LAUNCH("convert_x16_kernel");
  return B2_OK;
}
