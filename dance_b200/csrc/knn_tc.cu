// Tensor-core candidate filter for the exact kNN search (phase 1 of knn.cu: the N²·d part).
//
// One CTA (one warpgroup) owns 64 queries and streams every 64-reference tile through a TMA ring:
//   S = Q · Rᵀ            wgmma.mma_async m64n64k16 on fp16 (hi, lo) pairs of 2^e·x (22 significant bits; hi·hi + hi·lo + lo·hi),
//                         fp32 accumulation in registers, K = padded feature width (16 per instruction); the accumulators are
//                         written to shared memory so that a thread can read a query's row
//   d̂² = |q|² + |r|² − 2·S/4^e   two threads per query (one per half of the tile's columns) keep the M smallest estimates they
//                         see in an UNSORTED list held in registers (replace-the-maximum: 32 predicated moves + a 32-entry
//                         rescan per insertion); at the end the second half's list is inserted into the first's, which then
//                         holds the M smallest estimates of the query over all references
// The estimates only FILTER: phase 2 (knn_refine_kernel) re-ranks the candidates in fp64 exactly like the reference and
// proves with an error bound that no non-candidate can enter the top-k; unproven queries fall back to fp64 brute force.
// The bound for this filter is documented at `tc_err_rel` below.
//
// Operand layout: Xh / Xl [n, dp] halves (dp = d rounded up to 64 = one 128-byte swizzle atom per 64 features), K-major
// SWIZZLE_128B boxes {64 halves, 64 rows}; an operand tile is dp/64 atoms of 8 KB.
#include "tc_common.cuh"

#include <cuda_fp16.h>
#include <math_constants.h>
#include <stdlib.h>
#include <string.h>

namespace b2 {
namespace ktc {

using namespace tc;

constexpr int BQ = 64;           // queries per CTA (wgmma M)
constexpr int BR = 64;           // references per tile (wgmma N)
constexpr int MC = 32;           // candidates kept per query
constexpr int MAX_ATOMS = 2;     // dp <= 128
constexpr int ATOM_BYTES = 64 * 128;   // 64 rows x 128 B
constexpr int THREADS = 128;
constexpr int STAGES = 2;
constexpr int S_PITCH = BR + 4;  // floats per row of the estimate tile (16-byte rows, conflict-free float4 reads)

struct Params {
  CUtensorMap m_hi, m_lo;        // [n, dp] halves, box {64, 64}, SWIZZLE_128B
  const float* sqn;              // |x|² (fp32, unscaled)
  const float* scale;            // scale[1] = 4^-e
  int32_t* cand_idx;             // [n_q, MC]
  float* cand_thr;               // [n_q]
  int n, n_q, q_begin, atoms;
};
// max |x| → 2^e with max·2^e ∈ [256, 512);  scale[0] = 2^e, scale[1] = 4^-e
__global__ void __launch_bounds__(256)
absmax_kernel(const float* __restrict__ X, int64_t ldx, int32_t n, int32_t d, uint32_t* __restrict__ maxbits) {
  float m = 0.f;
  const int64_t total = (int64_t)n * d;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x)
    m = fmaxf(m, fabsf(X[(t / d) * ldx + t % d]));
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) atomicMax(maxbits, __float_as_uint(m));
}

__global__ void scale_kernel(const uint32_t* __restrict__ maxbits, float* __restrict__ scale) {
  const float m = __uint_as_float(maxbits[0]);
  int e = 0;
  if (m > 0.f && isfinite(m)) { int ex; frexpf(m, &ex); e = 9 - ex; }
  e = e > 40 ? 40 : (e < -40 ? -40 : e);
  scale[0] = ldexpf(1.f, e);
  scale[1] = ldexpf(1.f, -2 * e);
}

__global__ void __launch_bounds__(256)
split_kernel(const float* __restrict__ X, int64_t ldx, int32_t n, int32_t d, int32_t dp, const float* __restrict__ scale,
             __half* __restrict__ xh, __half* __restrict__ xl) {
  const int64_t total = (int64_t)n * dp;
  const float s = scale[0];
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / dp;
    const int c = (int)(t % dp);
    const float v = c < d ? X[i * ldx + c] * s : 0.f;
    const __half h = __float2half_rn(v);
    xh[t] = h;
    xl[t] = __float2half_rn(v - __half2float(h));
  }
}

struct CandList {
  float key[MC];
  int32_t kid[MC];
  int maxslot;                     // slot currently holding the largest kept estimate (= thr)
  float thr;
  __device__ __forceinline__ void init() {
    maxslot = 0;
    thr = CUDART_INF_F;
#pragma unroll
    for (int s = 0; s < MC; ++s) { key[s] = CUDART_INF_F; kid[s] = -1; }
  }
  __device__ __forceinline__ void insert(float e, int32_t id) {
#pragma unroll
    for (int s = 0; s < MC; ++s)
      if (s == maxslot) { key[s] = e; kid[s] = id; }
    float mx = key[0];
    maxslot = 0;
#pragma unroll
    for (int s = 1; s < MC; ++s)
      if (key[s] > mx) { mx = key[s]; maxslot = s; }
    thr = mx;
  }
};

__global__ void __launch_bounds__(THREADS)
knn_candidates_tc_kernel(const __grid_constant__ Params p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int op_bytes = p.atoms * ATOM_BYTES;                 // one operand part (hi or lo) of one tile
  const uint32_t s_q_hi = smem_u32(smem), s_q_lo = s_q_hi + op_bytes;
  const uint32_t s_ring = s_q_lo + op_bytes;                 // [STAGES][hi | lo]
  float* S = reinterpret_cast<float*>(smem + (2 + 2 * STAGES) * op_bytes);   // [BQ][S_PITCH] estimates of the current tile
  const uint32_t q_bar = smem_u32(S + BQ * S_PITCH);
  const uint32_t full_bar = q_bar + 8;              // [STAGES]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int q0 = blockIdx.x * BQ;                   // local query offset
  const int n_tiles = (p.n + BR - 1) / BR;

  if (tid == 0) {
    tma_prefetch_desc(&p.m_hi);
    tma_prefetch_desc(&p.m_lo);
    mbar_init(q_bar, 1);
    for (int s = 0; s < STAGES; ++s) mbar_init(full_bar + 8 * s, 1);
    fence_barrier_init();
  }
  __syncthreads();
  auto issue = [&](int t) {
    const int s = t % STAGES;
    const uint32_t fb = full_bar + 8 * s, st = s_ring + s * 2 * op_bytes;
    mbar_expect_tx(fb, 2 * op_bytes);
    for (int a = 0; a < p.atoms; ++a) {
      tma_load_2d(st + a * ATOM_BYTES, &p.m_hi, fb, a * 64, t * BR);
      tma_load_2d(st + op_bytes + a * ATOM_BYTES, &p.m_lo, fb, a * 64, t * BR);
    }
  };
  if (tid == 0) {
    mbar_expect_tx(q_bar, 2 * op_bytes);
    for (int a = 0; a < p.atoms; ++a) {
      tma_load_2d(s_q_hi + a * ATOM_BYTES, &p.m_hi, q_bar, a * 64, p.q_begin + q0);
      tma_load_2d(s_q_lo + a * ATOM_BYTES, &p.m_lo, q_bar, a * 64, p.q_begin + q0);
    }
    for (int t = 0; t < min(n_tiles, STAGES); ++t) issue(t);
  }

  // selection role: query ql, columns [half·32, half·32 + 32) of every tile (warps 0-1: first half, warps 2-3: second half)
  const int ql = tid & (BQ - 1), half = tid >> 6;
  const int q = q0 + ql;
  const float inv_s2 = p.scale[1];
  const bool live = q < p.n_q;
  const float qn = live ? p.sqn[p.q_begin + q] : 0.f;
  const float m2 = -2.f * inv_s2;
  CandList cl;
  cl.init();
  mbar_wait(q_bar, 0);

  for (int t = 0; t < n_tiles; ++t) {
    const int s = t % STAGES;
    mbar_wait(full_bar + 8 * s, (uint32_t)((t / STAGES) & 1));
    const uint32_t st = s_ring + s * 2 * op_bytes;
    float acc[BR / 2];
    wgmma_fence();
    for (int a = 0; a < p.atoms; ++a) {
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {             // 64 halves per atom = 4 k-steps of 16
        const uint32_t off = (uint32_t)(a * ATOM_BYTES + kk * 32);
        wgmma_f16_ss_n64(acc, wgmma_desc_sw128(s_q_lo + off), wgmma_desc_sw128(st + off), (a | kk) != 0);
        wgmma_f16_ss_n64(acc, wgmma_desc_sw128(s_q_hi + off), wgmma_desc_sw128(st + op_bytes + off), 1);
        wgmma_f16_ss_n64(acc, wgmma_desc_sw128(s_q_hi + off), wgmma_desc_sw128(st + off), 1);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(acc);
    __syncthreads();                               // every thread has finished the previous tile's selection and this tile's MMAs
    if (tid == 0 && t + STAGES < n_tiles) issue(t + STAGES);
    {
      const int r = warp * 16 + (lane >> 2);
#pragma unroll
      for (int v = 0; v < BR / 2; v += 2) {
        const int c = 8 * (v >> 2) + 2 * (lane & 3);
        const int rr = r + 8 * ((v >> 1) & 1);
        *reinterpret_cast<float2*>(S + rr * S_PITCH + c) = make_float2(acc[v], acc[v + 1]);
      }
    }
    __syncthreads();
    const int r0 = t * BR + half * 32;
    // |r|² of the 32 columns: one coalesced load per lane, broadcast by shuffle
    const float rn_l = r0 + lane < p.n ? __ldg(p.sqn + r0 + lane) : CUDART_INF_F;
    float est[32];
#pragma unroll
    for (int c = 0; c < 32; c += 4) {
      const float4 v = *reinterpret_cast<const float4*>(S + ql * S_PITCH + half * 32 + c);
      est[c] = fmaf(m2, v.x, qn + __shfl_sync(0xffffffffu, rn_l, c));
      est[c + 1] = fmaf(m2, v.y, qn + __shfl_sync(0xffffffffu, rn_l, c + 1));
      est[c + 2] = fmaf(m2, v.z, qn + __shfl_sync(0xffffffffu, rn_l, c + 2));
      est[c + 3] = fmaf(m2, v.w, qn + __shfl_sync(0xffffffffu, rn_l, c + 3));
    }
    uint32_t mask = 0;
#pragma unroll
    for (int c = 0; c < 32; ++c) mask |= (est[c] < cl.thr ? 1u : 0u) << c;
    if (live && mask) {
      float es[32];                                // dynamic indexing below → local memory, touched only on this path
#pragma unroll
      for (int c = 0; c < 32; ++c) es[c] = est[c];
      while (mask) {
        const int c = __ffs(mask) - 1;
        mask &= mask - 1;
        const float e = es[c];
        if (e < cl.thr) cl.insert(e, r0 + c);      // thr may have dropped since the mask was built
      }
    }
  }
  // merge: the second half's list goes through shared memory into the first half's
  __syncthreads();
  float* mkey = S;
  int32_t* mid = reinterpret_cast<int32_t*>(S + BQ * MC);
  if (half == 1) {
#pragma unroll
    for (int c = 0; c < MC; ++c) { mkey[ql * MC + c] = cl.key[c]; mid[ql * MC + c] = cl.kid[c]; }
  }
  __syncthreads();
  if (half == 0 && live) {
    for (int c = 0; c < MC; ++c) {
      const float e = mkey[ql * MC + c];
      if (e < cl.thr) cl.insert(e, mid[ql * MC + c]);
    }
#pragma unroll
    for (int c = 0; c < MC; ++c) p.cand_idx[(int64_t)q * MC + c] = cl.kid[c];
    p.cand_thr[q] = cl.thr;
  }
}

static int padded_d(int32_t d) { return (d + 63) / 64 * 64; }

size_t workspace_bytes(int32_t n, int32_t d, int32_t n_q) {
  (void)n_q;
  return 256 + 2 * align_up((size_t)n * padded_d(d) * sizeof(__half), 256);
}

bool eligible(int32_t n, int32_t d, int32_t n_q, int M) {
  if (path_mode(B2_PATH_KNN_FILTER) == 1) return false;      // SIMT filter requested (both filters are bit-exact)
  return M == MC && d >= 8 && padded_d(d) <= 64 * MAX_ATOMS && (int64_t)n * n_q >= (1ll << 24);
}

// Relative error bound of the filter estimate d̂² w.r.t. (|q| + |r|)²:
//   operands carry 22 bits (hi + lo, each rounded to nearest)            → |Δ(q·r)| ≤ 2^-21 |q||r| (+ dropped lo·lo 2^-22)
//   dp/16 · 3 products accumulated in fp32 (bounded as if every add truncated) → ≤ 3·dp/16 · 2^-23 · |q||r|  (≤ 24 adds → 2^-18.4)
//   norms and the final fma in fp32                                       → (d + 8) · 2^-23 (|q|² + |r|²)
// 2·|Δ(q·r)| ≤ 2^-17 |q||r| covers the first two lines with margin.
float tc_err_rel(int32_t d) { return 7.62939453125e-06f + 1.1920928955078125e-07f * (float)(d + 8); }

int launch(const float* X, int64_t ldx, const float* sqn, int32_t n, int32_t d, int32_t q_begin, int32_t n_q, int32_t* cand_idx,
           float* cand_thr, void* ws, size_t ws_bytes, cudaStream_t st) {
  if (ws_bytes < workspace_bytes(n, d, n_q)) return B2_ERR_UNSUPPORTED;
  const int dp = padded_d(d);
  char* w = reinterpret_cast<char*>(ws);
  uint32_t* maxbits = reinterpret_cast<uint32_t*>(w);
  float* scale = reinterpret_cast<float*>(w + 16);
  __half* xh = reinterpret_cast<__half*>(w + 256);
  __half* xl = reinterpret_cast<__half*>(w + 256 + align_up((size_t)n * dp * sizeof(__half), 256));
  B2_CHECK_CUDA(cudaMemsetAsync(maxbits, 0, 4, st));
  int64_t blocks = ceil_div<int64_t>((int64_t)n * d, 256 * 8);
  const int64_t cap = (int64_t)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  absmax_kernel<<<(unsigned)blocks, 256, 0, st>>>(X, ldx, n, d, maxbits);
  B2_CHECK_LAUNCH("knn absmax_kernel");
  scale_kernel<<<1, 1, 0, st>>>(maxbits, scale);
  B2_CHECK_LAUNCH("knn scale_kernel");
  blocks = ceil_div<int64_t>((int64_t)n * dp, 256 * 4);
  const int64_t cap2 = (int64_t)sm_count() * 16;
  if (blocks > cap2) blocks = cap2;
  split_kernel<<<(unsigned)blocks, 256, 0, st>>>(X, ldx, n, d, dp, scale, xh, xl);
  B2_CHECK_LAUNCH("knn split_kernel");

  Params p;
  memset(&p, 0, sizeof(p));
  const int SW128 = (int)CU_TENSOR_MAP_SWIZZLE_128B;
  if (!make_tensor_map_f16_ex(&p.m_hi, xh, (uint64_t)dp, (uint64_t)n, (uint64_t)dp, 64, BR, SW128) ||
      !make_tensor_map_f16_ex(&p.m_lo, xl, (uint64_t)dp, (uint64_t)n, (uint64_t)dp, 64, BR, SW128))
    return B2_ERR_UNSUPPORTED;
  p.sqn = sqn; p.scale = scale; p.cand_idx = cand_idx; p.cand_thr = cand_thr;
  p.n = n; p.n_q = n_q; p.q_begin = q_begin; p.atoms = dp / 64;
  const int op_bytes = p.atoms * ATOM_BYTES;
  const size_t smem = (size_t)(2 + 2 * STAGES) * op_bytes + (size_t)BQ * S_PITCH * 4 + 8 * (1 + STAGES) + 1024;
  static size_t attr_smem = 0;
  if (smem > attr_smem) {
    B2_CHECK_CUDA(cudaFuncSetAttribute(knn_candidates_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_smem = smem;
  }
  knn_candidates_tc_kernel<<<ceil_div(n_q, BQ), THREADS, smem, st>>>(p);
  B2_CHECK_LAUNCH("knn_candidates_tc_kernel");
  return B2_OK;
}

}  // namespace ktc
}  // namespace b2
