// Tensor-core version of the all-pairs part of the Graph-AE decoder loss (scgnn2.py:423-426, 603-619):
//   loss += Σ_ij softplus(z_i · z_j),   dZ_i += 2·coef · Σ_j σ(z_i · z_j) · z_j
// Flash-attention-shaped row sweep: a CTA owns 128 rows I (two consumer warpgroups of 64) and streams 128-row tiles J:
//   S  = Z_I · Z_Jᵀ        wgmma m64n128k8 tf32, 3-product split (Z pre-split into hi = x & 0xFFFFE000 and lo = x − hi,
//                          lo·hi + hi·lo + hi·hi), fp32 accumulators in registers
//   G  = σ(S), loss       SFU math on the accumulator registers (e = 2^(−|x|·log2e), r = 1/(1+e), one lg2 per 32 logits)
//   dZ_I += G · Z_J       wgmma m64nDk8 tf32 with A = G taken straight from the registers (hi / lo split of G and Z_J, three
//                          products) and B = Z_Jᵀ from shared memory
// A producer warp copies the pre-split J tiles into a two-stage ring with 1-D bulk copies (the tiles are laid out in global
// memory exactly as wgmma reads them: K-major, 128-byte swizzle).
//
// Register fragment trick: the accumulator of S gives a thread columns (2t, 2t+1) of each 8-column block, the tf32 A fragment
// wants columns (t, t+4).  The sum over j does not care about order, so the 8 columns of each block are fed to the second
// MMA in the order (0, 2, 4, 6, 1, 3, 5, 7) and Z_Jᵀ is stored with its columns permuted the same way.
//
// Work units: row blocks.  The row form covers [row_begin, row_begin + n_rows); the pair-sharded form (multi-GPU) takes
// "super-blocks" s = {block s, block nb−1−s} (a lone middle block when nb is odd), so that super-block ranges split the work
// evenly over ranks.  The J sweep of a unit can be cut into step ranges (grid.y), which then add into dz atomically.
#include "tc_common.cuh"

#include <stdlib.h>
#include <string.h>

namespace b2 {
namespace gtc {

using namespace tc;

constexpr int BT = 128;                 // rows per block / tile
constexpr int CONSUMERS = 256;          // two warpgroups
constexpr int THREADS = CONSUMERS + 32; // + producer warp
constexpr int STAGES = 2;
constexpr int MAX_D = 32;
constexpr uint32_t ZS_BYTES = BT * 128; // one plane of a tile for S (K-major, 128-byte rows)
constexpr int ZS_PLANES = 2;            // hi, lo

static int64_t padded_n(int32_t n) { return ((int64_t)n + BT - 1) / BT * BT; }
template <int DP> constexpr uint32_t zt_bytes() { return (uint32_t)DP * 4 * 128; }   // one plane of Z_Jᵀ: 4 atoms of DP x 128 B

// position of column jj of a tile in the permuted order of the dZ MMA (see header)
__host__ __device__ __forceinline__ int zt_pos(int jj) { const int q = jj & 7; return (jj & ~7) | ((q & 1) ? 4 + (q >> 1) : (q >> 1)); }

__device__ __forceinline__ float tf32_trunc(float x) { return __uint_as_float(__float_as_uint(x) & 0xFFFFE000u); }

// z → hi / lo planes, tile by tile: ZS [tile][128 rows x 32 tf32, swizzled], ZT [tile][4 atoms][DP rows x 32 tf32, swizzled]
template <int DP>
__global__ void __launch_bounds__(256)
gae_split_kernel(const float* __restrict__ z, int64_t ldz, int32_t n, int32_t d, int64_t npad, uint8_t* __restrict__ zs_hi,
                 uint8_t* __restrict__ zs_lo, uint8_t* __restrict__ zt_hi, uint8_t* __restrict__ zt_lo) {
  const int64_t total = npad * DP;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = t / DP;
    const int k = (int)(t % DP);
    const float v = (row < n && k < d) ? z[row * ldz + k] : 0.f;
    const float h = tf32_trunc(v);
    const float l = v - h;
    const int64_t tile = row / BT;
    const int r = (int)(row % BT);
    const size_t so = (size_t)tile * ZS_BYTES + sw128_offset32((uint32_t)r, (uint32_t)k);
    *reinterpret_cast<float*>(zs_hi + so) = h;
    *reinterpret_cast<float*>(zs_lo + so) = l;
    const int p = zt_pos(r);
    const size_t to = (size_t)tile * zt_bytes<DP>() + (size_t)(p >> 5) * (DP * 128) + sw128_offset32((uint32_t)k, (uint32_t)(p & 31));
    *reinterpret_cast<float*>(zt_hi + to) = h;
    *reinterpret_cast<float*>(zt_lo + to) = l;
  }
}

struct Params {
  const float* z;
  int64_t ldz;
  const uint8_t *zs_hi, *zs_lo, *zt_hi, *zt_lo;
  float* dz;
  double* loss_acc;
  float coef;
  int n, d;
  int row_begin, row_end;      // row form: rows [row_begin, row_end), dz row i at dz[(i - row_begin) * d]
  int sb_begin, nb, sym;       // pair-sharded form: grid.x = 2 x super-blocks from sb_begin, dz row i at dz[i * d]
  int n_jt;                    // J tiles
};

template <int N>
__device__ __forceinline__ void mma_rs(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t b, uint32_t scale_d) {
  if constexpr (N == 8) wgmma_tf32_rs_n8(d, a, b, scale_d);
  else if constexpr (N == 16) wgmma_tf32_rs_n16(d, a, b, scale_d);
  else wgmma_tf32_rs_n32(d, a, b, scale_d);
}

__device__ __forceinline__ float ex2_approx(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float lg2_approx(float x) { float y; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float rcp_approx(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

template <int DP>
__global__ void __launch_bounds__(THREADS, 1)
gae_allpairs_tc_kernel(const __grid_constant__ Params p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr uint32_t ZT = zt_bytes<DP>();
  constexpr uint32_t STAGE = ZS_PLANES * ZS_BYTES + 2 * ZT;
  uint8_t* zi_hi = smem;
  uint8_t* zi_lo = smem + ZS_BYTES;
  uint8_t* ring = smem + ZS_PLANES * ZS_BYTES;
  const uint32_t full_bar = smem_u32(ring + STAGES * STAGE), empty_bar = full_bar + 8 * STAGES;

  // ---- work unit ----
  int row0, row_end, dz_row0;
  if (p.sym) {
    const int sb = p.sb_begin + (int)(blockIdx.x >> 1);
    const int blk = (blockIdx.x & 1) ? p.nb - 1 - sb : sb;
    if ((blockIdx.x & 1) && blk == sb) return;           // lone middle block: one unit only
    row0 = blk * BT; row_end = min(p.n, row0 + BT); dz_row0 = 0;
  } else {
    row0 = p.row_begin + (int)blockIdx.x * BT; row_end = min(p.row_end, row0 + BT); dz_row0 = p.row_begin;
  }
  const int per = (p.n_jt + (int)gridDim.y - 1) / (int)gridDim.y;
  const int jt0 = (int)blockIdx.y * per, jt1 = min(p.n_jt, jt0 + per);
  if (jt0 >= jt1) return;
  const int nt = jt1 - jt0;

  const int tid = threadIdx.x;
  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(full_bar + 8 * s, 1); mbar_init(empty_bar + 8 * s, CONSUMERS / 32); }
    fence_barrier_init();
  }
  __syncthreads();

  if (tid >= CONSUMERS) {
    // ===================== producer warp =====================
    if (tid == CONSUMERS) {
      for (int i = 0; i < nt; ++i) {
        const int s = i % STAGES;
        if (i >= STAGES) mbar_wait(empty_bar + 8 * s, (uint32_t)((i / STAGES - 1) & 1));
        const uint32_t fb = full_bar + 8 * s, dst = smem_u32(ring + s * STAGE);
        const size_t t = (size_t)(jt0 + i);
        mbar_expect_tx(fb, STAGE);
        bulk_load(dst, p.zs_hi + t * ZS_BYTES, ZS_BYTES, fb);
        bulk_load(dst + ZS_BYTES, p.zs_lo + t * ZS_BYTES, ZS_BYTES, fb);
        bulk_load(dst + 2 * ZS_BYTES, p.zt_hi + t * ZT, ZT, fb);
        bulk_load(dst + 2 * ZS_BYTES + ZT, p.zt_lo + t * ZT, ZT, fb);
      }
    }
    return;
  }

  // ===================== consumers =====================
  // Z_I planes from z (rows past the range are zero: their logits are masked below)
  for (int e = tid; e < BT * DP; e += CONSUMERS) {
    const int r = e / DP, k = e % DP;
    const int row = row0 + r;
    const float v = (row < row_end && k < p.d) ? p.z[(int64_t)row * p.ldz + k] : 0.f;
    const float h = tf32_trunc(v);
    const uint32_t o = sw128_offset32((uint32_t)r, (uint32_t)k);
    *reinterpret_cast<float*>(zi_hi + o) = h;
    *reinterpret_cast<float*>(zi_lo + o) = v - h;
  }
  fence_proxy_async();
  asm volatile("bar.sync 1, %0;" ::"n"(CONSUMERS) : "memory");

  const int wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
  const int ra = row0 + wg * 64 + warp * 16 + (lane >> 2);       // rows of this thread: ra, ra + 8
  const bool live_a = ra < row_end, live_b = ra + 8 < row_end;
  const uint32_t ai_hi = smem_u32(zi_hi) + wg * 64 * 128, ai_lo = smem_u32(zi_lo) + wg * 64 * 128;
  constexpr float LOG2E = 1.4426950408889634f, LN2 = 0.6931471805599453f;

  // The accumulation inside the tensor core truncates, and the hi·hi product carries almost all of dZ: over a whole J sweep one
  // accumulator would drift by ~1e-5 relative (~6e-5 for |z| ~ 1e5).  So the hi·hi products of a tile go round-robin into NB
  // accumulators (16 / NB adds each), the two cross terms into one more, and the tile's sum joins an fp32 total with
  // round-to-nearest adds.
  constexpr int NB = DP <= 16 ? 4 : 2;
  float dzb[NB][DP / 2], dzs[DP / 2], dzt[DP / 2];
#pragma unroll
  for (int v = 0; v < DP / 2; ++v) dzt[v] = 0.f;
  double loss = 0.0;

  for (int i = 0; i < nt; ++i) {
    const int s = i % STAGES;
    mbar_wait(full_bar + 8 * s, (uint32_t)((i / STAGES) & 1));
    const uint32_t st = smem_u32(ring + s * STAGE);
    const uint32_t bs_hi = st, bs_lo = st + ZS_BYTES, bt_hi = st + 2 * ZS_BYTES, bt_lo = bt_hi + ZT;
    float S[BT / 2];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < DP / 8; ++kk) {
      const uint32_t o = kk * 32;
      wgmma_tf32_ss_n128(S, wgmma_desc_sw128(ai_lo + o), wgmma_desc_sw128(bs_hi + o), kk > 0);
      wgmma_tf32_ss_n128(S, wgmma_desc_sw128(ai_hi + o), wgmma_desc_sw128(bs_lo + o), 1);
      wgmma_tf32_ss_n128(S, wgmma_desc_sw128(ai_hi + o), wgmma_desc_sw128(bs_hi + o), 1);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(S);

    // ---- σ and softplus on the registers ----
    const int jbase = (jt0 + i) * BT + 2 * (lane & 3);
    float relu = 0.f, lg = 0.f, prod = 1.f;
#pragma unroll
    for (int v = 0; v < BT / 2; ++v) {
      if ((v & 31) == 31) { lg += lg2_approx(prod); prod = 1.f; }
      const int j = jbase + 8 * (v >> 2) + (v & 1);
      const bool ok = j < p.n && (((v >> 1) & 1) ? live_b : live_a);
      const float x = S[v];
      const float e = ex2_approx(-fabsf(x) * LOG2E);
      const float inv = rcp_approx(1.f + e);
      const float sg = x >= 0.f ? inv : e * inv;
      relu += ok ? fmaxf(x, 0.f) : 0.f;
      prod *= ok ? 1.f + e : 1.f;
      S[v] = ok ? sg : 0.f;
    }
    loss += (double)(relu + LN2 * (lg + lg2_approx(prod)));

    // ---- dZ_I += G · Z_J ----
    wgmma_fence();
#pragma unroll
    for (int kb = 0; kb < BT / 8; ++kb) {
      const float g[4] = {S[4 * kb], S[4 * kb + 2], S[4 * kb + 1], S[4 * kb + 3]};   // (r, 2t) (r+8, 2t) (r, 2t+1) (r+8, 2t+1)
      uint32_t ahi[4], alo[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        ahi[q] = __float_as_uint(g[q]) & 0xFFFFE000u;
        alo[q] = __float_as_uint(g[q] - __uint_as_float(ahi[q]));
      }
      const uint32_t o = (uint32_t)(kb >> 2) * (DP * 128) + (uint32_t)(kb & 3) * 32;
      mma_rs<DP>(dzs, alo, wgmma_desc_sw128(bt_hi + o), kb > 0);
      mma_rs<DP>(dzs, ahi, wgmma_desc_sw128(bt_lo + o), 1);
      mma_rs<DP>(dzb[kb % NB], ahi, wgmma_desc_sw128(bt_hi + o), kb >= NB);
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int b = 0; b < NB; ++b) reg_fence(dzb[b]);
    reg_fence(dzs);
#pragma unroll
    for (int v = 0; v < DP / 2; ++v) {
      float t = dzs[v];
#pragma unroll
      for (int b = 0; b < NB; ++b) t += dzb[b][v];
      dzt[v] += t;
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(empty_bar + 8 * s);
  }

  // ---- epilogue ----
  const float c2 = 2.f * p.coef;
  const bool atomic = gridDim.y > 1;
#pragma unroll
  for (int v = 0; v < DP / 2; ++v) {
    const int row = ra + 8 * ((v >> 1) & 1);
    const int col = 8 * (v >> 2) + 2 * (lane & 3) + (v & 1);
    if (row >= row_end || col >= p.d) continue;
    float* dst = p.dz + (int64_t)(row - dz_row0) * p.d + col;
    const float val = c2 * dzt[v];
    if (atomic) atomicAdd(dst, val);
    else *dst += val;
  }
  loss = warp_sum(loss);
  if (lane == 0) atomicAdd(p.loss_acc, loss * (double)p.coef);
}

size_t workspace_bytes(int32_t n) { return (size_t)padded_n(n) / BT * (ZS_PLANES * ZS_BYTES + 2 * zt_bytes<MAX_D>()); }

int super_blocks(int32_t n) { return (int)((padded_n(n) / BT + 1) / 2); }

bool eligible(int32_t n, int32_t d, int32_t n_rows) {
  const int mode = path_mode(B2_PATH_GAE_DECODER);           // 0 auto · 1 CUDA cores · 2 this kernel
  if (d < 1 || d > MAX_D || mode == 1) return false;
  return mode == 2 || (int64_t)n * n_rows >= (1ll << 22);
}

template <int DP>
static int launch_dp(const float* z, int64_t ldz, int32_t n, int32_t d, Params p, int units, float* dz, double* loss_acc, void* ws,
                     cudaStream_t st) {
  const int64_t npad = padded_n(n);
  const int nb = (int)(npad / BT);
  uint8_t* w = reinterpret_cast<uint8_t*>(ws);
  uint8_t* zs_hi = w;
  uint8_t* zs_lo = zs_hi + (size_t)nb * ZS_BYTES;
  uint8_t* zt_hi = zs_lo + (size_t)nb * ZS_BYTES;
  uint8_t* zt_lo = zt_hi + (size_t)nb * zt_bytes<DP>();
  int64_t blocks = ceil_div<int64_t>(npad * DP, 256);
  const int64_t cap = (int64_t)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  gae_split_kernel<DP><<<(unsigned)blocks, 256, 0, st>>>(z, ldz, n, d, npad, zs_hi, zs_lo, zt_hi, zt_lo);
  B2_CHECK_LAUNCH("gae_split_kernel");
  if (units <= 0) return B2_OK;
  p.z = z; p.ldz = ldz; p.zs_hi = zs_hi; p.zs_lo = zs_lo; p.zt_hi = zt_hi; p.zt_lo = zt_lo;
  p.dz = dz; p.loss_acc = loss_acc; p.n = n; p.d = d; p.nb = nb; p.n_jt = nb;
  // J step ranges: b2_set_tuning(B2_TUNE_GAE_SPLITS) when set, else enough to fill one wave of SMs
  int splits = tuning(B2_TUNE_GAE_SPLITS);
  if (splits <= 0) splits = ceil_div(sm_count(), units);
  if (splits > nb) splits = nb;
  if (splits < 1) splits = 1;
  const size_t smem = ZS_PLANES * ZS_BYTES + STAGES * (ZS_PLANES * ZS_BYTES + 2 * zt_bytes<DP>()) + 16 * STAGES + 1024;
  static bool attr_set = false;
  if (!attr_set) {
    B2_CHECK_CUDA(cudaFuncSetAttribute(gae_allpairs_tc_kernel<DP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_set = true;
  }
  gae_allpairs_tc_kernel<DP><<<dim3((unsigned)units, (unsigned)splits), THREADS, smem, st>>>(p);
  B2_CHECK_LAUNCH("gae_allpairs_tc_kernel");
  return B2_OK;
}

static int launch_any(const float* z, int64_t ldz, int32_t n, int32_t d, const Params& p, int units, float* dz, double* loss_acc,
                      void* ws, size_t ws_bytes, cudaStream_t st) {
  if (ws_bytes < workspace_bytes(n)) return B2_ERR_UNSUPPORTED;
  if (d <= 8) return launch_dp<8>(z, ldz, n, d, p, units, dz, loss_acc, ws, st);
  if (d <= 16) return launch_dp<16>(z, ldz, n, d, p, units, dz, loss_acc, ws, st);
  return launch_dp<32>(z, ldz, n, d, p, units, dz, loss_acc, ws, st);
}

// rows [row_begin, row_begin + n_rows) against all n columns; adds into dz[n_rows, d] and loss_acc
int launch(const float* z, int64_t ldz, int32_t n, int32_t d, int32_t row_begin, int32_t n_rows, float coef, float* dz,
           double* loss_acc, void* ws, size_t ws_bytes, cudaStream_t st) {
  Params p;
  memset(&p, 0, sizeof(p));
  p.coef = coef; p.row_begin = row_begin; p.row_end = row_begin + n_rows; p.sym = 0;
  return launch_any(z, ldz, n, d, p, ceil_div(n_rows, BT), dz, loss_acc, ws, ws_bytes, st);
}

// super-blocks [sb_begin, sb_end) against all n columns; adds into dz[n, d] (the rows of those blocks) and loss_acc
int launch_super_blocks(const float* z, int64_t ldz, int32_t n, int32_t d, int32_t sb_begin, int32_t sb_end, float coef, float* dz,
                        double* loss_acc, void* ws, size_t ws_bytes, cudaStream_t st) {
  Params p;
  memset(&p, 0, sizeof(p));
  p.coef = coef; p.sym = 1; p.sb_begin = sb_begin;
  return launch_any(z, ldz, n, d, p, 2 * (sb_end - sb_begin), dz, loss_acc, ws, ws_bytes, st);
}

}  // namespace gtc
}  // namespace b2
