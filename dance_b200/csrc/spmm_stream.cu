// CSR SpMM, nnz-stream form:  Y = act(reduce(A · X) + bias)  for operand rows of 32 / 64 / 128 bytes
// (fp32 F = 8 / 16 / 32, bf16 / fp16 F = 16 / 32 / 64) — the scGNN aggregate Â·support (scgnn2.py:500) and its backward.
//
// Why a second kernel.  The row-per-lane-group kernels (spmm.cu, spmm16.cu) chain rowptr → (col, val) → gathers → FMA per row and
// per 8-entry chunk; partial-mask shuffles in loops of per-row trip count cost them ~65 SASS instructions per four non-zeros and
// low occupancy: latency- and issue-bound, not bandwidth-bound.  Here every warp owns a contiguous range of rows — hence a contiguous stream of non-zeros —
// and runs a software pipeline over 32-entry blocks of that stream:
//
//   block b+NG : its (col, val) pairs are copied to a shared-memory ring with cp.async (4 B per lane)
//   block b    : the 32 operand rows its columns name are gathered into a shared-memory ring with cp.async (16 B per lane)
//   block b-NG+1 (landed): consumed in CSR order — 128 / RB non-zeros per step, lanes across the feature dimension — and every
//                 finished row is written with one coalesced streaming store.
//
// Nothing in the loop waits for a load it has just issued: the (col, val) stream, the gathers and the row pointers (a 32-row
// window, prefetched one window ahead) are all NG blocks deep.  Row boundaries are handled by the consumer (a segmented reduction
// in registers over the variable-degree rows); rows are balanced over the warps by cumulative (non-zeros + rows) with a warp-
// cooperative 32-ary search of rowptr, so skewed degree distributions and empty rows cost nothing extra.  Gathers carry an L2
// evict-last hint, the one-pass streams evict-first.  Accumulation order inside a row = CSR order up to the NPI-way lane split
// (deterministic, independent of the launch geometry).
//
// TMA row copies (tile::gather4, per-row cp.async.bulk) are a poor fit for this pipeline: 64–128-byte rows are too small for the
// TMA unit to pay off.
#include "common.cuh"

#include <cuda_bf16.h>
#include <cuda_fp16.h>

namespace b2 {
namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int SS_WARPS = 8;   // warps per CTA
constexpr int SS_NG = 2;      // 32-entry blocks in flight per warp (more warps beat deeper rings: measured)
constexpr int SS_BLK = 32;

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint64_t policy_evict_last() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ uint64_t policy_evict_first() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ void cp_async_16(uint32_t dst, const void* src, uint64_t pol) {
  asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "l"(pol) : "memory");
}
__device__ __forceinline__ void cp_async_4(uint32_t dst, const void* src, uint64_t pol) {
  asm volatile("cp.async.ca.shared.global.L2::cache_hint [%0], [%1], 4, %2;" ::"r"(dst), "l"(src), "l"(pol) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// smallest r in [0, n_rows] with rowptr[r] + r >= t  (strictly increasing key; key(n_rows) = nnz + n_rows >= t): 32-ary search
__device__ __forceinline__ int warp_partition_point(const int32_t* __restrict__ rowptr, int n_rows, int64_t t, int lane) {
  int lo = 0, hi = n_rows;
  while (hi > lo) {
    const int span = hi - lo;
    const int step = (span + 31) >> 5;
    const int seg_lo = lo + lane * step;
    int q = seg_lo + step - 1;
    if (q > hi - 1) q = hi - 1;
    const bool in = seg_lo < hi;
    const bool pred = in ? ((int64_t)__ldg(rowptr + q) + q >= t) : true;
    const unsigned m = __ballot_sync(FULL, pred);
    const int f = __ffs(m) - 1;
    const int flo = lo + f * step;
    if (f < 0 || flo >= hi) {
      lo = hi;
    } else {
      int fhi = flo + step - 1;
      if (fhi > hi - 1) fhi = hi - 1;
      lo = flo;
      hi = fhi;
    }
  }
  return lo;
}

template <int DT> __device__ __forceinline__ void unpack2(uint32_t u, float& a, float& b) {
  if (DT == 0) {                       // bf16: the fp32 value is the 16 bits shifted into the high half
    a = __uint_as_float(u << 16);
    b = __uint_as_float(u & 0xffff0000u);
  } else {
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&u));
    a = f.x;
    b = f.y;
  }
}
template <int DT> __device__ __forceinline__ uint32_t pack2(float a, float b) {
  if (DT == 0) {
    const __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&v);
  }
  const __half2 v = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&v);
}

struct StreamArgs {
  const int32_t* rowptr;
  const int32_t* colidx;
  const float* vals;          // nullptr: unit weights
  const uint8_t* X;           // operand rows, ldxb bytes apart
  int64_t ldxb;
  float* Y;                   // fp32 result (may be null when Y16 is given)
  int64_t ldy;
  uint8_t* Y16;               // optional 16-bit copy of the result (operand's type), ldy16b bytes apart
  int64_t ldy16b;
  const float* bias;
  int32_t n_rows;
  int reduce, act;
};

// DT: 2 = fp32 operand, 0 = bf16, 1 = fp16.  RB = bytes per operand row (F · element size).  CB = bytes per lane at consumption.
// EPI = false compiles the epilogue away (plain sum, no bias / activation / 16-bit copy): the aggregate's inner loop is issue-bound
// enough (≈ 70 % issue-active) that the extra per-row instructions cost 25 %.
template <int DT, int RB, int CB, bool EPI>
__global__ void __launch_bounds__(SS_WARPS * 32)
spmm_stream_kernel(const StreamArgs a) {
  constexpr int ESZ = DT == 2 ? 4 : 2;
  constexpr int F = RB / ESZ;
  constexpr int NG = SS_NG, BLK = SS_BLK, NC = 2 * NG;
  constexpr int LPR = RB / 16;         // lanes per operand row while gathering (16-byte copies)
  constexpr int RPI = 32 / LPR;        // operand rows per cp.async instruction
  constexpr int LPRC = RB / CB;        // lanes per operand row while consuming
  constexpr int NPI = 32 / LPRC;       // non-zeros per consumption step
  constexpr int NV = CB / ESZ;         // result values per lane
  static_assert(LPR >= 1 && LPRC >= 1 && LPRC <= 32 && NV >= 1 && NV <= 8, "unsupported row width");
  extern __shared__ __align__(128) uint8_t smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint8_t* ring = smem + (size_t)warp * (NG * BLK * RB);
  int32_t* cring = reinterpret_cast<int32_t*>(smem + (size_t)SS_WARPS * NG * BLK * RB) + warp * (NC * BLK);
  float* vring = reinterpret_cast<float*>(smem + (size_t)SS_WARPS * NG * BLK * RB + (size_t)SS_WARPS * NC * BLK * 4) + warp * (NC * BLK);
  const uint32_t ring_s = smem_addr(ring), cring_s = smem_addr(cring), vring_s = smem_addr(vring);
  const int32_t* __restrict__ rowptr = a.rowptr;
  const int n_rows = a.n_rows;
  const int W = gridDim.x * SS_WARPS, w = blockIdx.x * SS_WARPS + warp;
  const int64_t total = (int64_t)__ldg(rowptr + n_rows) + n_rows;
  const int R0 = (w == 0) ? 0 : warp_partition_point(rowptr, n_rows, (int64_t)w * total / W, lane);
  const int R1 = (w == W - 1) ? n_rows : warp_partition_point(rowptr, n_rows, (int64_t)(w + 1) * total / W, lane);
  if (R0 >= R1) return;
  const int E0 = __ldg(rowptr + R0), E1 = __ldg(rowptr + R1);
  const int nblk = (E1 - E0 + BLK - 1) / BLK;
  const uint64_t pol_x = policy_evict_last(), pol_s = policy_evict_first();

  // row-pointer window: lane l holds rowptr[rb + 1 + l]; the next window is prefetched
  int rb = R0;
  int rpv = __ldg(rowptr + min(rb + 1 + lane, n_rows));
  int rpn = __ldg(rowptr + min(rb + 33 + lane, n_rows));
  int r = R0, rbeg = E0, rend = __shfl_sync(FULL, rpv, 0);
  const int subc = lane / LPRC, glc = lane % LPRC;
  float acc[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) acc[i] = 0.f;

  auto issue_pairs = [&](int blk_i, int cs) {     // (col, val) of block blk_i → pair-ring slot cs
    const int e = E0 + blk_i * BLK + lane;
    if (blk_i < nblk && e < E1) {
      cp_async_4(cring_s + (cs * BLK + lane) * 4, a.colidx + e, pol_s);
      if (a.vals) cp_async_4(vring_s + (cs * BLK + lane) * 4, a.vals + e, pol_s);
      else vring[cs * BLK + lane] = 1.f;
    } else {
      cring[cs * BLK + lane] = -1;
    }
  };
  auto emit_row = [&]() {
    // combine the NPI lane groups, then lanes 0 .. LPRC-1 hold features [lane·NV, lane·NV + NV) of row r
#pragma unroll
    for (int o = LPRC; o < 32; o <<= 1) {
#pragma unroll
      for (int i = 0; i < NV; ++i) acc[i] += __shfl_xor_sync(FULL, acc[i], o);
    }
    if (lane < LPRC) {
      float o[NV];
      if (EPI) {
        const float scale = (a.reduce == 1 && rend > rbeg) ? 1.f / (float)(rend - rbeg) : 1.f;   // DGL fn.mean divides by the in-degree
#pragma unroll
        for (int i = 0; i < NV; ++i) {
          float v = acc[i] * scale;
          if (a.bias) v += __ldg(a.bias + lane * NV + i);
          o[i] = apply_act(v, a.act);
        }
      } else {
#pragma unroll
        for (int i = 0; i < NV; ++i) o[i] = acc[i];
      }
      if (a.Y) {
        float* y = a.Y + (int64_t)r * a.ldy + lane * NV;
        if (NV == 1) asm volatile("st.global.cs.f32 [%0], %1;" ::"l"(y), "f"(o[0]) : "memory");
        else if (NV == 2) asm volatile("st.global.cs.v2.f32 [%0], {%1, %2};" ::"l"(y), "f"(o[0]), "f"(o[1 % NV]) : "memory");
        else {
#pragma unroll
          for (int i = 0; i < NV; i += 4)
            asm volatile("st.global.cs.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(y + i), "f"(o[i % NV]), "f"(o[(i + 1) % NV]), "f"(o[(i + 2) % NV]),
                         "f"(o[(i + 3) % NV]) : "memory");
        }
      }
      if (EPI && DT != 2 && a.Y16) {
        uint8_t* y = a.Y16 + (int64_t)r * a.ldy16b + lane * NV * 2;
        if (NV == 2) {
          *reinterpret_cast<uint32_t*>(y) = pack2<DT>(o[0], o[1 % NV]);
        } else if (NV == 4) {
          *reinterpret_cast<uint2*>(y) = make_uint2(pack2<DT>(o[0], o[1 % NV]), pack2<DT>(o[2 % NV], o[3 % NV]));
        } else if (NV == 8) {
          *reinterpret_cast<uint4*>(y) = make_uint4(pack2<DT>(o[0], o[1 % NV]), pack2<DT>(o[2 % NV], o[3 % NV]), pack2<DT>(o[4 % NV], o[5 % NV]),
                                                    pack2<DT>(o[6 % NV], o[7 % NV]));
        }
      }
    }
#pragma unroll
    for (int i = 0; i < NV; ++i) acc[i] = 0.f;
    ++r;
    rbeg = rend;
    int j = r - rb;
    if (j == 32) {
      rb += 32;
      rpv = rpn;
      rpn = __ldg(rowptr + min(rb + 33 + lane, n_rows));
      j = 0;
    }
    rend = __shfl_sync(FULL, rpv, j);
  };

  // prologue: pairs of blocks 0 .. NG-1
#pragma unroll
  for (int j = 0; j < NG; ++j) issue_pairs(j, j);
  cp_async_commit();
  cp_async_wait<0>();
  __syncwarp();

  int st_i = 0, cs_i = 0;      // row-ring stage / pair-ring slot of the block being issued
  int st_c = 0, cs_c = 0;      // … of the block being consumed
  int cs_p = NG;               // pair-ring slot receiving block b + NG
  for (int b = 0; b < nblk + NG - 1; ++b) {
    if (b < nblk) {
      const int c = cring[cs_i * BLK + lane];
#pragma unroll
      for (int i = 0; i < LPR; ++i) {
        const int idx = i * RPI + lane / LPR;
        const int cc = __shfl_sync(FULL, c, idx);
        if (cc >= 0) cp_async_16(ring_s + (st_i * BLK + idx) * RB + (lane % LPR) * 16, a.X + (int64_t)cc * a.ldxb + (lane % LPR) * 16, pol_x);
      }
      issue_pairs(b + NG, cs_p);
      st_i = (st_i + 1 == NG) ? 0 : st_i + 1;
      cs_i = (cs_i + 1 == NC) ? 0 : cs_i + 1;
      cs_p = (cs_p + 1 == NC) ? 0 : cs_p + 1;
    }
    cp_async_commit();
    if (b >= NG - 1) {
      const int bc = b - (NG - 1);
      cp_async_wait<NG - 1>();
      __syncwarp();
      const int eb = E0 + bc * BLK;
      const int eend = min(E1, eb + BLK);
      const uint8_t* blk = ring + (size_t)st_c * BLK * RB;
      const float* vb = vring + cs_c * BLK;
      int e = eb;
      while (true) {
        while (r < R1 && rend <= e) emit_row();
        if (e >= eend || r >= R1) break;
        const int run_end = min(rend, eend);
#pragma unroll 4
        for (int k = e + subc; k < run_end; k += NPI) {
          const int slot = k - eb;
          const float wv = vb[slot];
          const uint8_t* src = blk + slot * RB + glc * CB;
          if (DT == 2) {
            if (NV == 1) {
              acc[0] = fmaf(wv, *reinterpret_cast<const float*>(src), acc[0]);
            } else if (NV == 2) {
              const float2 x = *reinterpret_cast<const float2*>(src);
              acc[0] = fmaf(wv, x.x, acc[0]); acc[1 % NV] = fmaf(wv, x.y, acc[1 % NV]);
            } else {
              const float4 x = *reinterpret_cast<const float4*>(src);
              acc[0] = fmaf(wv, x.x, acc[0]); acc[1 % NV] = fmaf(wv, x.y, acc[1 % NV]);
              acc[2 % NV] = fmaf(wv, x.z, acc[2 % NV]); acc[3 % NV] = fmaf(wv, x.w, acc[3 % NV]);
            }
          } else {
            float p, q;
            if (NV == 2) {
              unpack2<DT>(*reinterpret_cast<const uint32_t*>(src), p, q);
              acc[0] = fmaf(wv, p, acc[0]); acc[1 % NV] = fmaf(wv, q, acc[1 % NV]);
            } else if (NV == 4) {
              const uint2 x = *reinterpret_cast<const uint2*>(src);
              unpack2<DT>(x.x, p, q); acc[0] = fmaf(wv, p, acc[0]); acc[1 % NV] = fmaf(wv, q, acc[1 % NV]);
              unpack2<DT>(x.y, p, q); acc[2 % NV] = fmaf(wv, p, acc[2 % NV]); acc[3 % NV] = fmaf(wv, q, acc[3 % NV]);
            } else {
              const uint4 x = *reinterpret_cast<const uint4*>(src);
              unpack2<DT>(x.x, p, q); acc[0] = fmaf(wv, p, acc[0]); acc[1 % NV] = fmaf(wv, q, acc[1 % NV]);
              unpack2<DT>(x.y, p, q); acc[2 % NV] = fmaf(wv, p, acc[2 % NV]); acc[3 % NV] = fmaf(wv, q, acc[3 % NV]);
              unpack2<DT>(x.z, p, q); acc[4 % NV] = fmaf(wv, p, acc[4 % NV]); acc[5 % NV] = fmaf(wv, q, acc[5 % NV]);
              unpack2<DT>(x.w, p, q); acc[6 % NV] = fmaf(wv, p, acc[6 % NV]); acc[7 % NV] = fmaf(wv, q, acc[7 % NV]);
            }
          }
        }
        e = run_end;
      }
      st_c = (st_c + 1 == NG) ? 0 : st_c + 1;
      cs_c = (cs_c + 1 == NC) ? 0 : cs_c + 1;
    }
  }
  while (r < R1) emit_row();   // rows that end exactly at E1 and trailing empty rows of this warp's range
}

template <int DT, int RB, int CB, bool EPI>
int launch_stream_epi(const StreamArgs& a, cudaStream_t st) {
  const size_t smem = (size_t)SS_WARPS * SS_NG * SS_BLK * RB + (size_t)SS_WARPS * 2 * SS_NG * SS_BLK * 8 + 128;
  auto kern = spmm_stream_kernel<DT, RB, CB, EPI>;
  static bool attr_set = false;
  if (!attr_set) {
    B2_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_set = true;
  }
  int per_sm = (int)((227 * 1024) / (smem + 1024));
  if (per_sm > 2048 / (SS_WARPS * 32)) per_sm = 2048 / (SS_WARPS * 32);
  if (per_sm < 1) per_sm = 1;
  int64_t blocks = (int64_t)sm_count() * per_sm;
  const int64_t useful = ceil_div<int64_t>(a.n_rows, SS_WARPS);      // at least one row per warp
  if (blocks > useful) blocks = useful;
  if (blocks < 1) blocks = 1;
  kern<<<(unsigned)blocks, SS_WARPS * 32, smem, st>>>(a);
  B2_CHECK_LAUNCH("spmm_stream_kernel");
  return B2_OK;
}

template <int DT, int RB, int CB>
int launch_stream(const StreamArgs& a, cudaStream_t st) {
  const bool plain = a.reduce == 0 && a.act == B2_ACT_NONE && !a.bias && !a.Y16 && a.Y;
  return plain ? launch_stream_epi<DT, RB, CB, false>(a, st) : launch_stream_epi<DT, RB, CB, true>(a, st);
}

}  // namespace

// Returns B2_OK when the nnz-stream kernel took the call, 1 when the shape is not one it handles (caller falls back), < 0 on error.
// dtype: 2 fp32, 0 bf16, 1 fp16 operand.
int spmm_stream_dispatch(int dtype, const int32_t* rowptr, const int32_t* colidx, const float* vals, const void* X, int64_t ldx, float* Y,
                         int64_t ldy, void* Y16, int64_t ldy16, int32_t n_rows, int32_t F, int reduce, int act, const float* bias,
                         cudaStream_t st) {
  if (path_mode(B2_PATH_SPMM) == 1) return 1;                       // forced row-per-group kernels (A/B timing, tests of both paths)
  const int esz = dtype == 2 ? 4 : 2;
  const int rbytes = F * esz;
  if (rbytes != 32 && rbytes != 64 && rbytes != 128) return 1;
  if (n_rows < 1) return 1;
  StreamArgs a;
  a.rowptr = rowptr; a.colidx = colidx; a.vals = vals;
  a.X = reinterpret_cast<const uint8_t*>(X); a.ldxb = ldx * esz;
  a.Y = Y; a.ldy = ldy;
  a.Y16 = reinterpret_cast<uint8_t*>(Y16); a.ldy16b = ldy16 * 2;
  a.bias = bias; a.n_rows = n_rows; a.reduce = reduce; a.act = act;
  // CB: fp32 rows of 128 B are consumed 16 B per lane (4 non-zeros per step), everything narrower 4 B per lane
  if (dtype == 2) {
    if (rbytes == 128) return launch_stream<2, 128, 16>(a, st);
    if (rbytes == 64) return launch_stream<2, 64, 4>(a, st);
    return launch_stream<2, 32, 4>(a, st);
  }
  if (dtype == 0) {
    if (rbytes == 128) return launch_stream<0, 128, 8>(a, st);
    if (rbytes == 64) return launch_stream<0, 64, 4>(a, st);
    return launch_stream<0, 32, 4>(a, st);
  }
  if (rbytes == 128) return launch_stream<1, 128, 8>(a, st);
  if (rbytes == 64) return launch_stream<1, 64, 4>(a, st);
  return launch_stream<1, 32, 4>(a, st);
}

}  // namespace b2
