// Tensor-core GEMM for the dense feature projections (fp32 in / fp32 out):
//   C[M,N] = epilogue( op(A)[M,K] · op(B)[K,N] )
// Hopper structure: one CTA per 128 x BN output tile (and K split), warp-specialised into three warpgroups.  The rewrite
// warpgroup (the last) has one thread stage the raw fp32 operand tiles of each 32-wide k-block into a ring with TMA
// (cp.async.bulk.tensor); the whole warpgroup then rewrites each raw stage into a ring of K-major swizzled plane stages (wgmma
// reads tf32 operands only K-major, so this one pass also serves the transposed layouts: nothing is transposed in global memory).
// The two consumer warpgroups (64 rows each) issue wgmma.mma_async on the plane stages with fp32 accumulators in registers, and
// the epilogue applies bias / activation / ReLU-mask / accumulate straight from the accumulator registers.  The handoffs are
// mbarriers (raw full / empty, plane full / empty), so the rewrite of later k-blocks runs under the MMAs of earlier ones and
// no CTA-wide barrier is left in the k-loop.
//
// Precision modes (a bound on how the operands are rounded; accumulation, inputs, outputs and the epilogue are fp32 in all)
//   TF32   : 128B-swizzled tf32 planes, one m64nBNk8 wgmma per k-step (tf32 operands: 10-bit mantissa, low bits ignored)
//   TF32X3 : fp32-accurate. The rewrite also splits each value into hi = x & 0xFFFFE000 (exactly representable in tf32) and
//            lo = x - hi, and the MMAs accumulate lo·hi + hi·lo into one accumulator and hi·hi into another, summed in the
//            epilogue (error ~2^-21 relative).
//   BF16   : the rewrite rounds each operand to bfloat16 (round-to-nearest-even, cvt.rn.bf16x2.f32: subnormals kept, as
//            torch's .to(torch.bfloat16)) into 64B-swizzled planes (a 32-wide k-block is a 64-byte row), one m64nBNk16
//            .f32.bf16.bf16 wgmma per 16 k.  Same k-block, ring, split-K plan and workspace as TF32.
// Shapes the tensor-core kernel does not take (see gemm_tc's qualification) run on the CUDA-core fp32 kernel in every mode.
//
// Replaces torch.mm / nn.Linear on the reference path (scgnn2.py:352-370, 499).
#include "tc_common.cuh"

#include <cuda_bf16.h>
#include <stdlib.h>
#include <string.h>

namespace b2 {
namespace tc {

constexpr int BM = 128;            // two consumer warpgroups x 64 rows
constexpr int BK = 32;             // k-block: 32 tf32 = 128 B = one 128B swizzle span (32 bf16 = 64 B = one 64B span)
constexpr int CONSUMERS = 256;     // warpgroups 0 and 1
constexpr int REWRITERS = 128;     // warpgroup 2
constexpr int THREADS = CONSUMERS + REWRITERS;
// Register split (setmaxnreg): the consumers hold acc and acc_s (64 + 64 registers at BN = 128 in TF32X3), the rewrite
// warpgroup a batch of up to 8 float4 chunks and their addresses.  128 · 80 + 256 · 208 = 63 488 of the 384 · 168 = 64 512
// the CTA is launched with.
constexpr int REWRITE_REGS = 80, CONSUMER_REGS = 208;
constexpr int MAX_STAGES = 4;      // raw stages and plane stages, each

enum Mode { MODE_TF32 = 0, MODE_TF32X3 = 1, MODE_BF16 = 2 };
__host__ __device__ constexpr int plane_row_bytes(int mode) { return mode == MODE_BF16 ? BK * 2 : BK * 4; }

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
  int mode;                // Mode
  int act;
  float beta;
  int tiles_m, tiles_n, splits, kb_per_split, kb_total, stages, planes;   // stages: raw ring depth; planes: plane ring depth
};

// shared memory: [plane ring: planes x (A hi | A lo | B hi | B lo)] [raw ring: stages x (A raw | B raw)] [barriers]
// (A lo / B lo only in TF32X3; BF16 planes are half the size of tf32 ones, the raw fp32 stage is the same in every mode)
struct SmemLayout {
  uint32_t a_plane, b_plane, plane_buf, raw_a, raw_stage, ring, bars, total;
};
__host__ __device__ inline SmemLayout smem_layout(int BN, int mode, int stages, int planes) {
  SmemLayout L;
  L.a_plane = BM * plane_row_bytes(mode);
  L.b_plane = (uint32_t)BN * plane_row_bytes(mode);
  L.plane_buf = (mode == MODE_TF32X3 ? 2u : 1u) * (L.a_plane + L.b_plane);
  L.raw_a = BM * BK * 4;
  L.raw_stage = L.raw_a + (uint32_t)BN * BK * 4;
  L.ring = (uint32_t)planes * L.plane_buf;
  L.bars = L.ring + (uint32_t)stages * L.raw_stage;
  L.total = L.bars + 8 * 4 * MAX_STAGES;   // raw full / raw empty / plane full / plane empty
  return L;
}

// raw tile (ROWS x 32 k, K-contiguous [row][k] or, MN, row-contiguous [k][row]) → K-major swizzled plane(s): tf32 (128B
// swizzle) or bf16 rounded to nearest even (64B swizzle).  Run by the rewrite warpgroup (lt = thread index within it): each
// thread first loads all of its 16-byte chunks, then converts and stores them, so that a warp has its whole share of shared-
// memory loads in flight at once instead of one chunk's load → convert → store latency per chunk.
template <int MODE, int ROWS, bool MN>
__device__ __forceinline__ void convert_tile(const uint8_t* raw, uint8_t* hi, uint8_t* lo, int lt) {
  constexpr int PER = ROWS * (BK / 4) / REWRITERS;   // chunks per thread: 8 at 128 rows, 2 at 32
  float4 v[PER];
#pragma unroll
  for (int j = 0; j < PER; ++j) {
    const int c = lt + j * REWRITERS;
    if constexpr (!MN) {
      v[j] = *reinterpret_cast<const float4*>(raw + (c >> 3) * 128 + (c & 7) * 16);
    } else {
      const float* col = reinterpret_cast<const float*>(raw) + c % ROWS + (c / ROWS) * 4 * ROWS;
      v[j] = make_float4(col[0], col[ROWS], col[2 * ROWS], col[3 * ROWS]);
    }
  }
#pragma unroll
  for (int j = 0; j < PER; ++j) {
    const int c = lt + j * REWRITERS;
    const uint32_t r = MN ? c % ROWS : c >> 3, kc = MN ? c / ROWS : c & 7;
    if constexpr (MODE == MODE_BF16) {
      const __nv_bfloat162 p0 = __floats2bfloat162_rn(v[j].x, v[j].y), p1 = __floats2bfloat162_rn(v[j].z, v[j].w);   // .x at the lower address
      *reinterpret_cast<uint2*>(hi + sw64_offset16(r, kc * 4)) =
          make_uint2(*reinterpret_cast<const uint32_t*>(&p0), *reinterpret_cast<const uint32_t*>(&p1));
      continue;
    }
    const uint32_t off = sw128_offset32(r, kc * 4);
    if constexpr (MODE == MODE_TF32X3) {
      const float4 x = v[j];
      const float4 h = make_float4(tf32_hi(x.x), tf32_hi(x.y), tf32_hi(x.z), tf32_hi(x.w));
      *reinterpret_cast<float4*>(hi + off) = h;
      *reinterpret_cast<float4*>(lo + off) = make_float4(x.x - h.x, x.y - h.y, x.z - h.z, x.w - h.w);
    } else {
      *reinterpret_cast<float4*>(hi + off) = v[j];
    }
  }
}

template <int BN, int MODE>
__global__ void __launch_bounds__(THREADS, 1)
gemm_tc_kernel(const __grid_constant__ Params p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-byte alignment is required by the 128B swizzle atoms (the 64B ones need 512)
  // (offsetting smem_raw itself, not a rounded integer, keeps the pointer in the shared window: the rewrite then compiles to
  // LDS / STS rather than generic loads and stores)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const SmemLayout L = smem_layout(BN, MODE, p.stages, p.planes);
  // mbarriers: raw_full[s] (TMA bytes landed), raw_empty[s] (every rewrite thread has read stage s), plane_full[b] (every
  // rewrite thread has written plane stage b), plane_empty[b] (every consumer warp has retired the MMAs that read it)
  const uint32_t raw_full = smem_u32(smem + L.bars), raw_empty = raw_full + 8 * MAX_STAGES;
  const uint32_t plane_full = raw_empty + 8 * MAX_STAGES, plane_empty = plane_full + 8 * MAX_STAGES;
  const int tid = threadIdx.x, wg = tid >> 7, lt = tid & 127;

  const int u = blockIdx.x;
  const int ks = u % p.splits;
  const int t = u / p.splits;
  const int tn = t % p.tiles_n, tm = t / p.tiles_n;
  const int kb0 = ks * p.kb_per_split;
  // nk >= 1 for every CTA: make_plan sets splits = ceil(kb_total / kb_per_split), so the last split keeps at least one k-block.
  // The first MMA into each accumulator therefore always runs, and it starts the accumulator (scale-d = 0).
  const int nk = min(p.kb_total, kb0 + p.kb_per_split) - kb0;
  auto plane_ptrs = [&](int b, uint8_t*& a_hi, uint8_t*& a_lo, uint8_t*& b_hi, uint8_t*& b_lo) {
    a_hi = smem + b * L.plane_buf;
    a_lo = a_hi + L.a_plane;
    b_hi = a_hi + (MODE == MODE_TF32X3 ? 2 : 1) * L.a_plane;
    b_lo = b_hi + L.b_plane;
  };

  if (tid == 0) {
    tma_prefetch_desc(&p.tmA);
    tma_prefetch_desc(&p.tmB);
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(raw_full + 8 * s, 1);
      mbar_init(raw_empty + 8 * s, REWRITERS);
    }
    for (int b = 0; b < p.planes; ++b) {
      mbar_init(plane_full + 8 * b, REWRITERS);
      mbar_init(plane_empty + 8 * b, CONSUMERS / 32);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 2) {
    // ===================== rewrite warpgroup: TMA → raw ring → plane ring =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(REWRITE_REGS));
    auto issue = [&](int i) {
      const int s = i % p.stages, kb = kb0 + i;
      const uint32_t fb = raw_full + 8 * s;
      const uint32_t ra = smem_u32(smem + L.ring + s * L.raw_stage), rb = ra + L.raw_a;
      mbar_expect_tx(fb, L.raw_stage);
      if (!p.a_mn) tma_load_2d(ra, &p.tmA, fb, kb * BK, tm * BM);
      else tma_load_2d(ra, &p.tmA, fb, tm * BM, kb * BK);
      if (!p.b_mn) tma_load_2d(rb, &p.tmB, fb, kb * BK, tn * BN);
      else tma_load_2d(rb, &p.tmB, fb, tn * BN, kb * BK);
    };
    if (lt == 0)
      for (int i = 0; i < min(nk, p.stages); ++i) issue(i);
    for (int i = 0; i < nk; ++i) {
      // refill the stage k-block i-1 came from once the whole warpgroup has read it (raw_empty also orders those
      // generic-proxy reads before the TMA's async-proxy writes)
      if (lt == 0 && i >= 1 && i - 1 + p.stages < nk) {
        mbar_wait(raw_empty + 8 * ((i - 1) % p.stages), (uint32_t)(((i - 1) / p.stages) & 1));
        issue(i - 1 + p.stages);
      }
      const int s = i % p.stages, b = i % p.planes;
      if (i >= p.planes) mbar_wait(plane_empty + 8 * b, (uint32_t)(((i / p.planes) - 1) & 1));
      mbar_wait(raw_full + 8 * s, (uint32_t)((i / p.stages) & 1));
      uint8_t *a_hi, *a_lo, *b_hi, *b_lo;
      plane_ptrs(b, a_hi, a_lo, b_hi, b_lo);
      const uint8_t* raw = smem + L.ring + s * L.raw_stage;
      if (p.a_mn) convert_tile<MODE, BM, true>(raw, a_hi, a_lo, lt);
      else convert_tile<MODE, BM, false>(raw, a_hi, a_lo, lt);
      if (p.b_mn) convert_tile<MODE, BN, true>(raw + L.raw_a, b_hi, b_lo, lt);
      else convert_tile<MODE, BN, false>(raw + L.raw_a, b_hi, b_lo, lt);
      mbar_arrive(raw_empty + 8 * s);
      fence_proxy_async();                     // generic-proxy plane writes → visible to the tensor core (async proxy)
      mbar_arrive(plane_full + 8 * b);
    }
    return;
  }

  // ===================== consumer warpgroups: wgmma on the plane ring =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONSUMER_REGS));
  // hi·hi, and the two cross terms (TF32X3 only).  The first MMA into each overwrites it (scale-d = 0) instead of adding to
  // zeros written here: ptxas serialises every wgmma of a kernel (C7515) whose accumulators are also defined by ordinary
  // instructions.
  float acc[BN / 2], acc_s[BN / 2];
  const int lane = lt & 31;
  for (int i = 0; i < nk; ++i) {
    const int b = i % p.planes;
    uint8_t *a_hi, *a_lo, *b_hi, *b_lo;
    plane_ptrs(b, a_hi, a_lo, b_hi, b_lo);
    mbar_wait(plane_full + 8 * b, (uint32_t)((i / p.planes) & 1));
    wgmma_fence();
    const uint32_t ah = smem_u32(a_hi) + wg * 64 * plane_row_bytes(MODE), al = smem_u32(a_lo) + wg * 64 * plane_row_bytes(MODE);
    const uint32_t bh = smem_u32(b_hi), bl = smem_u32(b_lo);
    if constexpr (MODE == MODE_BF16) {
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        const uint32_t ko = k * 16 * 2;
        mma_ss<BF16, BN>(acc, wgmma_desc_sw64(ah + ko), wgmma_desc_sw64(bh + ko), (i | k) != 0);
      }
    } else {
#pragma unroll
      for (int k = 0; k < BK / 8; ++k) {
        const uint32_t ko = k * 8 * 4;
        if constexpr (MODE == MODE_TF32X3) {
          mma_ss<TF32, BN>(acc_s, wgmma_desc_sw128(al + ko), wgmma_desc_sw128(bh + ko), (i | k) != 0);
          mma_ss<TF32, BN>(acc_s, wgmma_desc_sw128(ah + ko), wgmma_desc_sw128(bl + ko), 1);
        }
        mma_ss<TF32, BN>(acc, wgmma_desc_sw128(ah + ko), wgmma_desc_sw128(bh + ko), (i | k) != 0);
      }
    }
    wgmma_commit();
    wgmma_wait<1>();                           // the MMAs of k-block i-1 are done: its plane stage may be rewritten
    if (i >= 1 && lane == 0) mbar_arrive(plane_empty + 8 * ((i - 1) % p.planes));
  }
  wgmma_wait<0>();
  reg_fence(acc);
  if constexpr (MODE == MODE_TF32X3) reg_fence(acc_s);

  // ===================== epilogue: straight from the accumulator registers =====================
  const int warp = lt >> 5;
  const int row_base = tm * BM + wg * 64 + warp * 16 + (lane >> 2);
  const bool vec_ok = ((p.ldc & 1) == 0) && ((reinterpret_cast<uintptr_t>(p.C) & 7) == 0);
#pragma unroll
  for (int v = 0; v < BN / 2; v += 2) {
    const int row = row_base + 8 * ((v >> 1) & 1);
    const int col = tn * BN + 8 * (v >> 2) + 2 * (lane & 3);
    if (row >= p.M || col >= p.N) continue;
    float o[2] = {acc[v], acc[v + 1]};
    if constexpr (MODE == MODE_TF32X3) { o[0] += acc_s[v]; o[1] += acc_s[v + 1]; }
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
  int BN, stages, planes, tiles_m, tiles_n, splits, kb_per_split, kb_total;
  size_t smem;
};

static Plan make_plan(int M, int N, int K, int mode) {
  Plan pl;
  pl.BN = N <= 32 ? 32 : (N <= 64 ? 64 : 128);
  // Two plane stages, then as many raw stages as fit (up to MAX_STAGES), then plane stages with what is left: at BN = 128
  // 2 x 64 KB planes + 3 x 32 KB raw in TF32X3, 3 x 32 KB + 4 x 32 KB in TF32, 4 x 16 KB + 4 x 32 KB in BF16.
  const size_t budget = kMaxDynamicSmem - 1024 /*align slack*/;
  const SmemLayout L0 = smem_layout(pl.BN, mode, 0, 2);
  pl.planes = 2;
  const size_t fit = (budget - L0.total) / L0.raw_stage;                            // ≥ 3 for every BN and mode
  pl.stages = fit < (size_t)MAX_STAGES ? (int)fit : MAX_STAGES;
  while (pl.planes < MAX_STAGES && smem_layout(pl.BN, mode, pl.stages, pl.planes + 1).total <= budget) ++pl.planes;
  pl.smem = (size_t)smem_layout(pl.BN, mode, pl.stages, pl.planes).total + 1024;
  pl.tiles_m = ceil_div(M, BM);
  pl.tiles_n = ceil_div(N, pl.BN);
  pl.kb_total = ceil_div(K, BK);     // the k-block, and so the split-K plan and its workspace, is the same in every mode
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

template <int BN, int MODE>
static int launch_gemm(const Params& p, const Plan& pl, cudaStream_t st) {
  const int rc = allow_dynamic_smem((const void*)gemm_tc_kernel<BN, MODE>, pl.smem);
  if (rc != B2_OK) return rc;
  gemm_tc_kernel<BN, MODE><<<pl.tiles_m * pl.tiles_n * pl.splits, THREADS, pl.smem, st>>>(p);
  B2_CHECK_LAUNCH("gemm_tc_kernel");
  return B2_OK;
}

template <int MODE>
static int launch_gemm_mode(const Params& p, const Plan& pl, cudaStream_t st) {
  return pl.BN == 32 ? launch_gemm<32, MODE>(p, pl, st) : (pl.BN == 64 ? launch_gemm<64, MODE>(p, pl, st) : launch_gemm<128, MODE>(p, pl, st));
}

static int mode_of(int precision) {
  return precision == B2_PREC_TF32X3 ? MODE_TF32X3 : (precision == B2_PREC_BF16 ? MODE_BF16 : MODE_TF32);
}

}  // namespace tc

size_t gemm_tc_workspace_bytes(int M, int N, int K, int transA, int transB, int precision) {
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  const tc::Plan pl = tc::make_plan(M, N, K, tc::mode_of(precision));
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

  const int mode = mode_of(precision);
  const Plan pl = make_plan(M, N, K, mode);
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
  p.mode = mode; p.act = act; p.beta = beta;
  p.tiles_m = pl.tiles_m; p.tiles_n = pl.tiles_n; p.splits = pl.splits; p.kb_per_split = pl.kb_per_split;
  p.kb_total = pl.kb_total; p.stages = pl.stages; p.planes = pl.planes;
  p.partial = nullptr;
  if (pl.splits > 1) {
    const size_t need = (size_t)pl.splits * M * N * sizeof(float);
    if (!workspace || workspace_bytes < need) {
      set_error("b2_gemm_f32: split-K workspace too small (%zu < %zu)", workspace_bytes, need);
      return B2_ERR_WORKSPACE;
    }
    p.partial = reinterpret_cast<float*>(workspace);
  }
  const int rc = mode == MODE_TF32X3 ? launch_gemm_mode<MODE_TF32X3>(p, pl, st)
               : (mode == MODE_BF16 ? launch_gemm_mode<MODE_BF16>(p, pl, st) : launch_gemm_mode<MODE_TF32>(p, pl, st));
  if (rc != B2_OK) return rc;
  if (pl.splits > 1) {
    splitk_reduce_kernel<<<grid_blocks((int64_t)M * N, 256, 8), 256, 0, st>>>(p.partial, pl.splits, M, N, C, ldc, bias, act, mask,
                                                                              ldmask, beta);
    B2_CHECK_LAUNCH("splitk_reduce_kernel");
  }
  return B2_OK;
}

}  // namespace b2
