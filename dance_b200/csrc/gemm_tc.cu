// Tensor-core GEMM for the dense feature projections (fp32 in / fp32 out):
//   C[M,N] = epilogue( op(A)[M,K] · op(B)[K,N] )
// Hopper structure: one CTA per 128 x BN output tile (and K split), two consumer warpgroups of 64 rows each.  TMA
// (cp.async.bulk.tensor) stages the raw fp32 operand tiles of each 32-wide k-block into a ring; all 256 threads then rewrite the
// stage as K-major, 128B-swizzled tf32 planes (wgmma reads tf32 operands only K-major, so this one pass also serves the
// transposed layouts: nothing is transposed in global memory) and issue wgmma.mma_async m64nBNk8 with fp32 accumulators in
// registers.  The rewrite of k-block i+1 overlaps the asynchronous MMAs of k-block i (two plane buffers); the epilogue applies
// bias / activation / ReLU-mask / accumulate straight from the accumulator registers.
//
// Precision modes
//   TF32   : one wgmma per k-step (tf32 operands: 10-bit mantissa)
//   TF32X3 : fp32-accurate. The rewrite also splits each value into hi = x & 0xFFFFE000 (exactly representable in tf32) and
//            lo = x - hi, and the MMAs accumulate lo·hi + hi·lo into one accumulator and hi·hi into another, summed in the
//            epilogue (error ~2^-21 relative).
//
// Replaces torch.mm / nn.Linear on the reference path (scgnn2.py:352-370, 499).
#include "tc_common.cuh"

#include <stdlib.h>
#include <string.h>

namespace b2 {
namespace tc {

constexpr int BM = 128;            // two warpgroups x 64 rows
constexpr int BK = 32;             // k-block: 32 tf32 = 128 B = one swizzle span
constexpr int UK = 8;              // wgmma K for tf32
constexpr int THREADS = 256;
constexpr int MAX_STAGES = 4;
constexpr int SMEM_LIMIT = 227 * 1024;

struct Params {
  CUtensorMap tmA;
  CUtensorMap tmB;
  float* C;
  const float* bias;
  const float* mask;
  float* partial;          // split-K partial tiles [splits][M][N] (dense) or nullptr
  long long ldc, ldmask;
  int M, N, K;
  int a_mn, b_mn;          // raw tile layout: 0 = K contiguous, 1 = M / N contiguous
  int x3;                  // 3xTF32 split
  int act;
  float beta;
  int tiles_m, tiles_n, splits, kb_per_split, kb_total, stages;
};

// shared memory: [2 plane buffers: A hi | A lo | B hi | B lo] [ring: stages x (A raw | B raw)] [barriers]
struct SmemLayout {
  uint32_t a_plane, b_plane, plane_buf, raw_a, raw_stage, ring, bars, total;
};
__host__ __device__ inline SmemLayout smem_layout(int BN, int x3, int stages) {
  SmemLayout L;
  L.a_plane = BM * BK * 4;
  L.b_plane = (uint32_t)BN * BK * 4;
  L.plane_buf = (x3 ? 2u : 1u) * (L.a_plane + L.b_plane);
  L.raw_a = BM * BK * 4;
  L.raw_stage = L.raw_a + L.b_plane;
  L.ring = 2 * L.plane_buf;
  L.bars = L.ring + (uint32_t)stages * L.raw_stage;
  L.total = L.bars + 8 * MAX_STAGES;
  return L;
}

// raw tile (rows x 32 k, K-contiguous [row][k] or row-contiguous [k][row]) → K-major swizzled tf32 plane(s)
__device__ __forceinline__ void convert_tile(const uint8_t* raw, uint8_t* hi, uint8_t* lo, int rows, int mn, int x3, int tid) {
  for (int c = tid; c < rows * (BK / 4); c += THREADS) {
    int r, kc;
    float4 v;
    if (!mn) {
      r = c >> 3; kc = c & 7;
      v = *reinterpret_cast<const float4*>(raw + r * 128 + kc * 16);
    } else {
      r = c % rows; kc = c / rows;
      const float* col = reinterpret_cast<const float*>(raw) + r;
      v = make_float4(col[(kc * 4 + 0) * rows], col[(kc * 4 + 1) * rows], col[(kc * 4 + 2) * rows], col[(kc * 4 + 3) * rows]);
    }
    const uint32_t off = sw128_offset32((uint32_t)r, (uint32_t)kc * 4);
    if (x3) {
      const float4 h = make_float4(__uint_as_float(__float_as_uint(v.x) & 0xFFFFE000u), __uint_as_float(__float_as_uint(v.y) & 0xFFFFE000u),
                                   __uint_as_float(__float_as_uint(v.z) & 0xFFFFE000u), __uint_as_float(__float_as_uint(v.w) & 0xFFFFE000u));
      *reinterpret_cast<float4*>(hi + off) = h;
      *reinterpret_cast<float4*>(lo + off) = make_float4(v.x - h.x, v.y - h.y, v.z - h.z, v.w - h.w);
    } else {
      *reinterpret_cast<float4*>(hi + off) = v;
    }
  }
}

template <int BN>
__device__ __forceinline__ void mma_ss(float (&d)[BN / 2], uint64_t a, uint64_t b, uint32_t scale_d) {
  if constexpr (BN == 32) wgmma_tf32_ss_n32(d, a, b, scale_d);
  else if constexpr (BN == 64) wgmma_tf32_ss_n64(d, a, b, scale_d);
  else wgmma_tf32_ss_n128(d, a, b, scale_d);
}

template <int BN, bool X3>
__global__ void __launch_bounds__(THREADS, 1)
gemm_tc_kernel(const __grid_constant__ Params p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-byte alignment is required by the 128B swizzle atoms
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const SmemLayout L = smem_layout(BN, p.x3, p.stages);
  const uint32_t full_bar = smem_u32(smem + L.bars);
  const int tid = threadIdx.x, wg = tid >> 7, lt = tid & 127;

  const int u = blockIdx.x;
  const int ks = u % p.splits;
  const int t = u / p.splits;
  const int tn = t % p.tiles_n, tm = t / p.tiles_n;
  const int kb0 = ks * p.kb_per_split;
  const int nk = max(0, min(p.kb_total, kb0 + p.kb_per_split) - kb0);

  if (tid == 0) {
    tma_prefetch_desc(&p.tmA);
    tma_prefetch_desc(&p.tmB);
    for (int s = 0; s < p.stages; ++s) mbar_init(full_bar + 8 * s, 1);
    fence_barrier_init();
  }
  __syncthreads();
  auto issue = [&](int i) {
    const int s = i % p.stages, kb = kb0 + i;
    const uint32_t fb = full_bar + 8 * s;
    const uint32_t ra = smem_u32(smem + L.ring + s * L.raw_stage), rb = ra + L.raw_a;
    mbar_expect_tx(fb, L.raw_stage);
    if (!p.a_mn) tma_load_2d(ra, &p.tmA, fb, kb * BK, tm * BM);
    else tma_load_2d(ra, &p.tmA, fb, tm * BM, kb * BK);
    if (!p.b_mn) tma_load_2d(rb, &p.tmB, fb, kb * BK, tn * BN);
    else tma_load_2d(rb, &p.tmB, fb, tn * BN, kb * BK);
  };
  if (tid == 0)
    for (int i = 0; i < min(nk, p.stages); ++i) issue(i);

  float acc[BN / 2], acc_s[BN / 2];     // hi·hi and the two cross terms (3xTF32)
#pragma unroll
  for (int j = 0; j < BN / 2; ++j) { acc[j] = 0.f; acc_s[j] = 0.f; }

  for (int i = 0; i < nk; ++i) {
    const int s = i % p.stages;
    uint8_t* planes = smem + (i & 1) * L.plane_buf;
    uint8_t* a_hi = planes;
    uint8_t* a_lo = planes + L.a_plane;
    uint8_t* b_hi = planes + (p.x3 ? 2 : 1) * L.a_plane;
    uint8_t* b_lo = b_hi + L.b_plane;
    mbar_wait(full_bar + 8 * s, (uint32_t)((i / p.stages) & 1));
    const uint8_t* raw = smem + L.ring + s * L.raw_stage;
    convert_tile(raw, a_hi, a_lo, BM, p.a_mn, p.x3, tid);
    convert_tile(raw + L.raw_a, b_hi, b_lo, BN, p.b_mn, p.x3, tid);
    fence_proxy_async();                       // generic-proxy plane writes → visible to the tensor core (async proxy)
    __syncthreads();                           // planes complete; the raw stage is free again
    if (tid == 0 && i + p.stages < nk) issue(i + p.stages);
    wgmma_fence();
    const uint32_t ah = smem_u32(a_hi) + wg * 64 * 128, al = smem_u32(a_lo) + wg * 64 * 128;
    const uint32_t bh = smem_u32(b_hi), bl = smem_u32(b_lo);
#pragma unroll
    for (int k = 0; k < BK / UK; ++k) {
      const uint32_t ko = k * UK * 4;
      if (X3) {
        mma_ss<BN>(acc_s, wgmma_desc_sw128(al + ko), wgmma_desc_sw128(bh + ko), 1);
        mma_ss<BN>(acc_s, wgmma_desc_sw128(ah + ko), wgmma_desc_sw128(bl + ko), 1);
      }
      mma_ss<BN>(acc, wgmma_desc_sw128(ah + ko), wgmma_desc_sw128(bh + ko), 1);
    }
    wgmma_commit();
    wgmma_wait<1>();                           // the MMAs of k-block i-1 are done: their plane buffer may be rewritten
    __syncthreads();                           // ... by every warpgroup
  }
  wgmma_wait<0>();
  reg_fence(acc);
  reg_fence(acc_s);

  // ===================== epilogue: straight from the accumulator registers =====================
  const int warp = lt >> 5, lane = lt & 31;
  const int row_base = tm * BM + wg * 64 + warp * 16 + (lane >> 2);
  const bool vec_ok = ((p.ldc & 1) == 0) && ((reinterpret_cast<uintptr_t>(p.C) & 7) == 0);
#pragma unroll
  for (int v = 0; v < BN / 2; v += 2) {
    const int row = row_base + 8 * ((v >> 1) & 1);
    const int col = tn * BN + 8 * (v >> 2) + 2 * (lane & 3);
    if (row >= p.M || col >= p.N) continue;
    float o[2] = {acc[v] + acc_s[v], acc[v + 1] + acc_s[v + 1]};
    const bool two = col + 1 < p.N;
    if (p.partial) {
      float* dst = p.partial + ((size_t)ks * p.M + row) * p.N + col;
      dst[0] = o[0];
      if (two) dst[1] = o[1];
      continue;
    }
    float* dst = p.C + (size_t)row * p.ldc + col;
    const float* mrow = p.mask ? p.mask + (size_t)row * p.ldmask + col : nullptr;
#pragma unroll
    for (int jj = 0; jj < 2; ++jj) {
      if (jj == 1 && !two) break;
      float x = o[jj];
      if (p.bias) x += __ldg(p.bias + col + jj);
      x = apply_act(x, p.act);
      if (mrow && !(__ldg(mrow + jj) > 0.f)) x = 0.f;
      if (p.beta != 0.f) x = fmaf(p.beta, dst[jj], x);
      o[jj] = x;
    }
    if (two && vec_ok) *reinterpret_cast<float2*>(dst) = make_float2(o[0], o[1]);
    else { dst[0] = o[0]; if (two) dst[1] = o[1]; }
  }
}

// deterministic split-K reduction + epilogue
__global__ void __launch_bounds__(256)
splitk_reduce_kernel(const float* __restrict__ partial, int splits, int M, int N, float* __restrict__ C, long long ldc,
                     const float* __restrict__ bias, int act, const float* __restrict__ mask, long long ldmask,
                     float beta) {
  const size_t total = (size_t)M * N;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / N), c = (int)(i % N);
    float s = 0.f;
    for (int k = 0; k < splits; ++k) s += partial[(size_t)k * total + i];
    if (bias) s += bias[c];
    s = apply_act(s, act);
    if (mask && !(mask[(size_t)r * ldmask + c] > 0.f)) s = 0.f;
    float* dst = C + (size_t)r * ldc + c;
    if (beta != 0.f) s = fmaf(beta, *dst, s);
    *dst = s;
  }
}

// ---- host side -----------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

// general 2-D fp32 tensor map: box = {box_inner, box_outer}; swizzle: 0 none, 1 32B, 2 64B, 3 128B, 4 128B_ATOM_32B
bool make_tensor_map_f32_ex(CUtensorMap* map, const float* ptr, uint64_t inner, uint64_t outer, uint64_t ld, uint32_t box_inner,
                            uint32_t box_outer, int swizzle) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {ld * sizeof(float)};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  return enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(ptr), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, (CUtensorMapSwizzle)swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

bool make_tensor_map_f16_ex(CUtensorMap* map, const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld, uint32_t box_inner,
                            uint32_t box_outer, int swizzle) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {ld * 2};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  return enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, (CUtensorMapSwizzle)swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

struct Plan {
  int BN, stages, tiles_m, tiles_n, splits, kb_per_split, kb_total;
  size_t smem;
};

static Plan make_plan(int M, int N, int K, int x3) {
  Plan pl;
  pl.BN = N <= 32 ? 32 : (N <= 64 ? 64 : 128);
  const SmemLayout L0 = smem_layout(pl.BN, x3, 0);
  int stages = (int)((SMEM_LIMIT - 1024 - L0.total) / L0.raw_stage);
  if (stages > MAX_STAGES) stages = MAX_STAGES;
  pl.stages = stages;               // ≥ 2 for every BN (128 KB of planes + 2 x 32 KB raw stages at BN = 128, 3xTF32)
  pl.smem = (size_t)smem_layout(pl.BN, x3, stages).total + 1024 /*align slack*/;
  pl.tiles_m = ceil_div(M, BM);
  pl.tiles_n = ceil_div(N, pl.BN);
  pl.kb_total = ceil_div(K, BK);
  const int tiles = pl.tiles_m * pl.tiles_n;
  const int sms = sm_count();
  int splits = 1;
  if (tiles * 10 < sms * 6 && pl.kb_total >= 8) {
    splits = ceil_div(sms, tiles);
    const int max_splits = pl.kb_total / 4;
    if (splits > max_splits) splits = max_splits;
    if (splits < 1) splits = 1;
  }
  pl.kb_per_split = ceil_div(pl.kb_total, splits);
  pl.splits = ceil_div(pl.kb_total, pl.kb_per_split);
  return pl;
}

template <int BN, bool X3>
static int launch_gemm(const Params& p, const Plan& pl, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    B2_CHECK_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<BN, X3>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT));
    attr_set = true;
  }
  gemm_tc_kernel<BN, X3><<<pl.tiles_m * pl.tiles_n * pl.splits, THREADS, pl.smem, st>>>(p);
  B2_CHECK_LAUNCH("gemm_tc_kernel");
  return B2_OK;
}

}  // namespace tc

size_t gemm_tc_workspace_bytes(int M, int N, int K, int transA, int transB, int precision) {
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  const tc::Plan pl = tc::make_plan(M, N, K, precision == B2_PREC_TF32X3);
  return pl.splits > 1 ? (size_t)pl.splits * M * N * sizeof(float) : 0;
}

int gemm_tc(const float* A, int64_t lda, int transA, const float* B, int64_t ldb, int transB, float* C, int64_t ldc,
            int M, int N, int K, const float* bias, int act, const float* mask, int64_t ldmask, float beta,
            int precision, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  using namespace tc;
  // qualification: TMA needs 16-byte aligned bases and row pitches; tiny problems stay on the CUDA-core kernel
  if (K < 8 || (int64_t)M * N * K < (1ll << 18)) return B2_ERR_UNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(B) & 15) || (lda & 3) || (ldb & 3))
    return B2_ERR_UNSUPPORTED;
  if (!get_encode()) return B2_ERR_UNSUPPORTED;

  const int x3 = precision == B2_PREC_TF32X3;
  const Plan pl = make_plan(M, N, K, x3);
  Params p;
  memset(&p, 0, sizeof(p));
  // raw tiles, unswizzled: A is [M,K] row-major (box 32 k x 128 rows) or stored [K,M] (box 128 rows x 32 k); B likewise
  const int NONE = (int)CU_TENSOR_MAP_SWIZZLE_NONE;
  const bool okA = transA ? make_tensor_map_f32_ex(&p.tmA, A, (uint64_t)M, (uint64_t)K, (uint64_t)lda, BM, BK, NONE)
                          : make_tensor_map_f32_ex(&p.tmA, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda, BK, BM, NONE);
  const bool okB = transB ? make_tensor_map_f32_ex(&p.tmB, B, (uint64_t)K, (uint64_t)N, (uint64_t)ldb, BK, (uint32_t)pl.BN, NONE)
                          : make_tensor_map_f32_ex(&p.tmB, B, (uint64_t)N, (uint64_t)K, (uint64_t)ldb, (uint32_t)pl.BN, BK, NONE);
  if (!okA || !okB) return B2_ERR_UNSUPPORTED;
  p.C = C; p.bias = bias; p.mask = mask; p.ldc = ldc; p.ldmask = ldmask;
  p.M = M; p.N = N; p.K = K;
  p.a_mn = transA ? 1 : 0;
  p.b_mn = transB ? 0 : 1;
  p.x3 = x3; p.act = act; p.beta = beta;
  p.tiles_m = pl.tiles_m; p.tiles_n = pl.tiles_n; p.splits = pl.splits; p.kb_per_split = pl.kb_per_split;
  p.kb_total = pl.kb_total; p.stages = pl.stages;
  p.partial = nullptr;
  if (pl.splits > 1) {
    const size_t need = (size_t)pl.splits * M * N * sizeof(float);
    if (!workspace || workspace_bytes < need) {
      set_error("b2_gemm_f32: split-K workspace too small (%zu < %zu)", workspace_bytes, need);
      return B2_ERR_WORKSPACE;
    }
    p.partial = reinterpret_cast<float*>(workspace);
  }
  const int rc = x3 ? (pl.BN == 32 ? launch_gemm<32, true>(p, pl, st) : (pl.BN == 64 ? launch_gemm<64, true>(p, pl, st) : launch_gemm<128, true>(p, pl, st)))
                    : (pl.BN == 32 ? launch_gemm<32, false>(p, pl, st) : (pl.BN == 64 ? launch_gemm<64, false>(p, pl, st) : launch_gemm<128, false>(p, pl, st)));
  if (rc != B2_OK) return rc;
  if (pl.splits > 1) {
    size_t total = (size_t)M * N;
    int blocks = (int)((total + 255) / 256);
    if (blocks > sm_count() * 8) blocks = sm_count() * 8;
    splitk_reduce_kernel<<<blocks, 256, 0, st>>>(p.partial, pl.splits, M, N, C, ldc, bias, act, mask, ldmask, beta);
    B2_CHECK_LAUNCH("splitk_reduce_kernel");
  }
  return B2_OK;
}

}  // namespace b2
