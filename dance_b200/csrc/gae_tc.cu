// Tensor-core version of the all-pairs part of the Graph-AE decoder loss (scgnn2.py:423-426, 603-619):
//   loss += Σ_ij softplus(z_i · z_j),   dZ_i += 2·coef · Σ_j σ(z_i · z_j) · z_j
// Flash-attention-shaped row sweep: a CTA owns 128 rows I (two consumer warpgroups of 64) and streams J tiles:
//   S  = Z_I · Z_Jᵀ        wgmma m64nJWk8 tf32, 3-product split (Z pre-split into hi = x & 0xFFFFE000 and lo = x − hi,
//                          lo·hi + hi·lo + hi·hi), fp32 accumulators in registers
//   G  = σ(S), loss       SFU math on the accumulator registers (e = 2^(−|x|·log2e), r = 1/(1+e), one lg2 per 32 logits)
//   dZ_I += G · Z_J       wgmma with A = G taken straight from the registers (split into hi / lo, three products) and
//                          B = Z_Jᵀ from shared memory
// A producer warpgroup (one thread of it) copies the pre-split J tiles into a three-stage ring with 1-D bulk copies (the tiles
// are laid out in global memory exactly as wgmma reads them: K-major, 128-byte swizzle).
//
// Two kernels share that sweep:
//   gae_allpairs_tc_kernel  J tiles of 128 columns over every column: row subsets (row shards) and the pair-sharded form.
//                          dZ_I in tf32 m64nDPk8: the hi / lo split of G and of Z_J, lo·hi + hi·lo + hi·hi.
//   gae_tri_tc_kernel       the full-row call.  S is symmetric, so block I only sweeps J ≥ I in tiles of 64 columns.  The
//                          128 x 128 diagonal block is evaluated as in the full sweep (it holds both orders of each pair); every
//                          tile above it counts its loss twice and also yields dZ_J += Gᵀ · Z_I: G goes to shared memory as
//                          hi / lo planes of Gᵀ (K-major in i, the A operand) and Z_Iᵀ is the B operand.  Both dZ products run
//                          in fp16 m64nNk16 (half the wgmmas of tf32 k8 at the same cost each): G·2^14 and each 64-row tile of
//                          z scaled by 2^e_t into fp16's range, split into fp16 hi / lo (22 significant bits like the tf32
//                          split); the tile sums are unscaled exactly in fp32.  Each issues its three products as two: hi·hi
//                          and hi·lo as one m64n(2·DP)k16 against a B operand laid out [hi | lo], and lo·hi.  dZ_J runs on a
//                          fourth warpgroup of its own (below).
//
// Schedule: each product is issued as one batch of wgmmas with one commit and one wait, which needs S, both halves of G and
// the dZ accumulators live in registers at once; the producer warpgroup gives its registers to the consumers (setmaxnreg) to
// make room.  The two consumer warpgroups run out of phase ("ping-pong"): while one does σ / softplus on the SFU, the other's
// products run on the tensor cores.  Tiles with no masked logit take an elementwise loop without the per-logit mask.
// Triangle: the consumers' turns hold S and dZ_I only.  A dZ_J warpgroup takes each consumer warpgroup's Gᵀ through an
// mbarrier pair (Gᵀ full / Gᵀ empty), issues both halves of a tile's dZ_J (K = warpgroup 0's rows, then warpgroup 1's) into
// the same accumulators in turn, adds the halves in fp32 and sends the tile's sum to dz with one set of red.global.add.
//
// Register fragments: the accumulator of S gives a thread columns (2t, 2t+1) of each 8-column block.  That is the triangle's
// fp16 A fragment (two columns packed per register), so its dZ_I takes G in the natural column order.  The full sweep's tf32
// A fragment wants columns (t, t+4); the sum over j does not care about order, so the 8 columns of each block are fed to its
// dZ MMA in the order (0, 2, 4, 6, 1, 3, 5, 7) and Z_Jᵀ is stored with its columns permuted the same way (zt_pos).  The
// triangle's packed fp16 G is also the fragment stmatrix takes: each 8 x 8 block goes to the Gᵀ planes transposed
// (stmatrix .trans, four blocks per instruction), so Gᵀ and Z_Iᵀ are K-major in the natural order of i.
//
// Work units: row blocks.  The row form covers [row_begin, row_begin + n_rows); the pair-sharded form (multi-GPU) takes
// "super-blocks" s = {block s, block nb−1−s} (a lone middle block when nb is odd), so that super-block ranges split the work
// evenly over ranks; the triangle's block I carries nb − I blocks of work and blocks are launched in order, longest first.
// The J sweep of a unit can be cut into step ranges (grid.y), which then add into dz atomically.
#include "tc_common.cuh"

#include <cuda_fp16.h>
#include <stdlib.h>
#include <string.h>

namespace b2 {
namespace gtc {

using namespace tc;

constexpr int BT = 128;                 // rows per block / workspace tile
constexpr int CONSUMERS = 256;          // two warpgroups
constexpr int THREADS = CONSUMERS + 128; // + producer warpgroup
constexpr int TRI_THREADS = THREADS + 128; // triangle: + dZ_J warpgroup
// Register split (setmaxnreg): the consumers hold S, both halves of G and the dZ accumulators while a dZ batch is in flight.
// Full sweep: 128 · 40 + 256 · 232 = 64 512 of the 65 536 registers of an SM.
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;
// Triangle: producer 24, dZ_J warpgroup DJ (its accumulators and the tile's fp32 sum), consumers (no dZ_J accumulators).
template <int DP>
struct TriRegs {
  static constexpr int PRODUCER = 24, DJ = DP <= 16 ? 80 : 96, CONSUMER = DP <= 16 ? 200 : 192;
};
static_assert(128 * (TriRegs<16>::PRODUCER + TriRegs<16>::DJ + 2 * TriRegs<16>::CONSUMER) <= 65536 &&
              128 * (TriRegs<32>::PRODUCER + TriRegs<32>::DJ + 2 * TriRegs<32>::CONSUMER) <= 65536, "triangle registers");
constexpr int STAGES = 3;
constexpr int MAX_D = 32;
constexpr uint32_t ZS_BYTES = BT * 128; // one plane of a tile for S (K-major, 128-byte rows)
constexpr int ZS_PLANES = 2;            // hi, lo

static int64_t padded_n(int32_t n) { return ((int64_t)n + BT - 1) / BT * BT; }
template <int DP> constexpr uint32_t zt_bytes() { return (uint32_t)DP * 4 * 128; }   // one plane of Z_Jᵀ: 4 atoms of DP x 128 B

// Shared memory of a sweep.  Full sweep (DP = 32): Z_I 32 KB + 3 x 64 KB stages.  Triangle: a J tile's Z_Jᵀ is one fp16
// [hi | lo] block of 2·DP rows x 64 j, Z_Iᵀ the same per warpgroup, Gᵀ planes of 64 j x 64 i fp16; the 64-column J tiles of S
// are the halves of a 128-row workspace tile (contiguous in both planes).  DP = 32: Z_I 32 KB, Z_Iᵀ 16 KB, Gᵀ 32 KB,
// 3 x 24 KB stages.
template <int DP, bool TRI>
struct Tiles {
  static constexpr int JW = TRI ? 64 : BT;                        // J tile width
  static constexpr uint32_t JS = JW * 128;                        // one plane of a J tile for S
  static constexpr uint32_t JT = TRI ? 2 * DP * 128 : zt_bytes<DP>();   // a J tile's Z_Jᵀ: one plane (triangle: [hi | lo])
  static constexpr uint32_t STAGE = ZS_PLANES * JS + (TRI ? 1 : 2) * JT;
  static constexpr uint32_t ZIT = TRI ? 2 * DP * 128 : 0;         // triangle: one warpgroup's Z_Iᵀ, [hi | lo]
  static constexpr uint32_t GT = TRI ? 64 * 128 : 0;              // triangle: one plane of a warpgroup's Gᵀ, 64 j x 64 i
  static constexpr uint32_t RING = ZS_PLANES * ZS_BYTES + 2 * ZIT + 4 * GT;
  static constexpr size_t SMEM = RING + STAGES * STAGE + 16 * STAGES + (TRI ? 32 : 0) + 1024;   // + Gᵀ full / empty x 2
};

// position of column jj of a tile in the permuted order of the dZ MMA (see header)
__host__ __device__ __forceinline__ int zt_pos(int jj) { const int q = jj & 7; return (jj & ~7) | ((q & 1) ? 4 + (q >> 1) : (q >> 1)); }

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
    const float h = tf32_hi(v);
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

// Triangle: z → the tf32 hi / lo planes for S as above, and per 64-row tile t the fp16 [hi | lo] block of Z_Jᵀ
// (2·DP rows x 64 j, K-major, 128-byte swizzle) of z·2^e_t, with e_t (exps[t]) chosen from the tile's largest |z| so that the
// scaled values stay ≤ 2^14: hi = rn(x·2^e), lo = rn(x·2^e − hi), 22 significant bits like the tf32 split.  A zero tile
// gets e = 0.  One block per 64-row tile.
template <int DP>
__global__ void __launch_bounds__(256)
gae_split_f16_kernel(const float* __restrict__ z, int64_t ldz, int32_t n, int32_t d, uint8_t* __restrict__ zs_hi,
                     uint8_t* __restrict__ zs_lo, uint8_t* __restrict__ zt, int* __restrict__ exps) {
  __shared__ float wmax[8];
  const int64_t row0 = (int64_t)blockIdx.x * 64;
  auto load = [&](int e) {
    const int64_t row = row0 + e / DP;
    const int k = e % DP;
    return (row < n && k < d) ? z[row * ldz + k] : 0.f;
  };
  float m = 0.f;
  for (int e = threadIdx.x; e < 64 * DP; e += 256) m = fmaxf(m, fabsf(load(e)));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = m;
  __syncthreads();
  m = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) m = fmaxf(m, wmax[w]);
  int ex = 0;
  if (m > 0.f) { int e2; frexpf(m, &e2); ex = min(100, max(-100, 14 - e2)); }   // m < 2^e2
  if (threadIdx.x == 0) exps[blockIdx.x] = ex;
  const float sc = ldexpf(1.f, ex);
  uint8_t* zt_t = zt + (size_t)blockIdx.x * (2 * DP * 128);
  for (int e = threadIdx.x; e < 64 * DP; e += 256) {
    const int r = e / DP, k = e % DP;
    const int64_t row = row0 + r;
    const float v = load(e);
    const float h = tf32_hi(v);
    const size_t so = (size_t)(row / BT) * ZS_BYTES + sw128_offset32((uint32_t)(row % BT), (uint32_t)k);
    *reinterpret_cast<float*>(zs_hi + so) = h;
    *reinterpret_cast<float*>(zs_lo + so) = v - h;
    const float x = v * sc;
    const __half xh = __float2half_rn(x);
    *reinterpret_cast<__half*>(zt_t + sw128_offset16((uint32_t)k, (uint32_t)r)) = xh;
    *reinterpret_cast<__half*>(zt_t + sw128_offset16((uint32_t)(DP + k), (uint32_t)r)) = __float2half_rn(x - __half2float(xh));
  }
}

// 2^(−14−e): undoes the scale of a product of G·2^14 and a tile scaled by 2^e, exactly (e ∈ [−100, 100])
__device__ __forceinline__ float unscale(int e) { return __int_as_float((127 - 14 - e) << 23); }

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
  const int* exps;             // triangle: scale exponent of each 64-row tile (zt_hi holds the fp16 blocks)
};

__device__ __forceinline__ float ex2_approx(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float lg2_approx(float x) { float y; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float rcp_approx(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
// Four 8 x 8 b16 matrices in the mma fragment layout (register q of lane l: row l/4, columns 2·(l%4), +1 of matrix q) stored
// transposed: lane l gives the address of row l % 8 of stored matrix l / 8, i.e. of column l % 8 of fragment matrix l / 8.
__device__ __forceinline__ void stsm_x4_trans(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c),
               "r"(d) : "memory");
}

// σ and softplus of one thread's logits S (the m64nJW accumulator), in place: S becomes the hi part of G = σ(S) and L its lo
// part, ready to be the register A operand of the dZ product.  Returns the thread's share of Σ softplus.  MASKED zeroes G and
// drops the loss of columns j ≥ n and of rows past the range (the last J tile, a partial I block); interior tiles skip the
// per-logit mask and its selects.  F16 (the triangle): G·2^14 is split into fp16 hi / lo, packed two columns per register
// (the f16 A fragment) into S[0 .. V/2) and L[0 .. V/2).  The 2^14 rides in the reciprocal's argument, rcp(2^-14·(1+e)) =
// 2^14 / (1+e) (power-of-two scaling is exact, so G·2^14 is what σ · 2^14 gave), and the product of the (1+e) is formed as
// prod·e + prod in one FFMA; with the mask, a dropped logit multiplies by 1 + 0.  Both save an instruction per logit in the
// consumers' serial σ / softplus phase; the MUFU count (ex2, rcp, one lg2 per 32) is the same.
template <bool MASKED, int V, bool F16>
__device__ __forceinline__ float sigmoid_softplus(float (&S)[V], float (&L)[V], int jbase, int n, bool live_a, bool live_b) {
  constexpr float LOG2E = 1.4426950408889634f, LN2 = 0.6931471805599453f, INV_G_SCALE = 1.f / 16384.f;
  float relu = 0.f, lg = 0.f, prod = 1.f;
#pragma unroll
  for (int v = 0; v < V; ++v) {
    if ((v & 31) == 31) { lg += lg2_approx(prod); prod = 1.f; }
    const float x = S[v];
    const float e = ex2_approx(-fabsf(x) * LOG2E);
    const float inv = F16 ? rcp_approx(fmaf(e, INV_G_SCALE, INV_G_SCALE)) : rcp_approx(1.f + e);
    float sg = x >= 0.f ? inv : e * inv;
    if constexpr (MASKED) {
      const int j = jbase + 8 * (v >> 2) + (v & 1);
      const bool ok = j < n && (((v >> 1) & 1) ? live_b : live_a);
      relu += ok ? fmaxf(x, 0.f) : 0.f;
      if constexpr (F16) prod = fmaf(prod, ok ? e : 0.f, prod);
      else prod *= ok ? 1.f + e : 1.f;
      sg = ok ? sg : 0.f;
    } else {
      relu += fmaxf(x, 0.f);
      if constexpr (F16) prod = fmaf(prod, e, prod);
      else prod *= 1.f + e;
    }
    if constexpr (F16) {
      S[v] = sg;
    } else {
      const float hi = tf32_hi(sg);
      S[v] = hi;
      L[v] = sg - hi;
    }
  }
  if constexpr (F16) {
#pragma unroll
    for (int q = 0; q < V / 2; ++q) {
      const __half2 h = __floats2half2_rn(S[2 * q], S[2 * q + 1]);
      const float2 hf = __half22float2(h);
      const __half2 l = __floats2half2_rn(S[2 * q] - hf.x, S[2 * q + 1] - hf.y);
      S[q] = __uint_as_float(*reinterpret_cast<const uint32_t*>(&h));
      L[q] = __uint_as_float(*reinterpret_cast<const uint32_t*>(&l));
    }
  }
  return relu + LN2 * (lg + lg2_approx(prod));
}

// Triangle: sum of a tile's merged dZ accumulators for output element v: columns c (hi·hi) and c + DP (hi·lo) sit DP / 2
// elements apart, s holds lo·hi
template <int NBM, int DP>
__device__ __forceinline__ float merged(const float (&acc)[NBM][DP], const float (&s)[DP / 2], int v) {
  float t = s[v];
#pragma unroll
  for (int b = 0; b < NBM; ++b) t += acc[b][v] + acc[b][v + DP / 2];
  return t;
}

// The sweep of one work unit; TRI selects the triangle (see header).
template <int DP, bool TRI>
__device__ __forceinline__ void decoder_sweep(const Params& p) {
  using T = Tiles<DP, TRI>;
  constexpr int JW = T::JW;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* zi_hi = smem;
  uint8_t* zi_lo = smem + ZS_BYTES;
  uint8_t* zit = smem + ZS_PLANES * ZS_BYTES;      // triangle: Z_Iᵀ [warpgroup]; then Gᵀ [warpgroup][hi, lo]
  uint8_t* ring = smem + T::RING;
  constexpr uint32_t ATOM = DP * 128;              // full sweep: DP rows of 32 tf32 along K
  constexpr int NB = DP <= 16 ? 4 : 2;             // full sweep: hi·hi accumulators
  constexpr int NBM = DP <= 16 ? 2 : 1;            // triangle: [hi·hi | hi·lo] accumulators
  const uint32_t full_bar = smem_u32(ring + STAGES * T::STAGE), empty_bar = full_bar + 8 * STAGES;
  // triangle: per consumer warpgroup, "its Gᵀ is written" (4 warp arrivals) and "its Gᵀ may be overwritten" (4 dZ_J warps)
  const uint32_t gt_full = empty_bar + 8 * STAGES, gt_empty = gt_full + 16;

  // ---- work unit ----
  int row0, row_end, dz_row0, jt0, jt1;
  if constexpr (TRI) {
    row0 = (int)blockIdx.x * BT; row_end = min(p.n, row0 + BT); dz_row0 = 0;
    const int first = row0 / JW;                         // J tiles from the diagonal block on
    const int per = (p.n_jt - first + (int)gridDim.y - 1) / (int)gridDim.y;
    jt0 = first + (int)blockIdx.y * per; jt1 = min(p.n_jt, jt0 + per);
  } else {
    if (p.sym) {
      const int sb = p.sb_begin + (int)(blockIdx.x >> 1);
      const int blk = (blockIdx.x & 1) ? p.nb - 1 - sb : sb;
      if ((blockIdx.x & 1) && blk == sb) return;         // lone middle block: one unit only
      row0 = blk * BT; row_end = min(p.n, row0 + BT); dz_row0 = 0;
    } else {
      row0 = p.row_begin + (int)blockIdx.x * BT; row_end = min(p.row_end, row0 + BT); dz_row0 = p.row_begin;
    }
    const int per = (p.n_jt + (int)gridDim.y - 1) / (int)gridDim.y;
    jt0 = (int)blockIdx.y * per; jt1 = min(p.n_jt, jt0 + per);
  }
  if (jt0 >= jt1) return;
  const int nt = jt1 - jt0;
  const int diag_end = (row0 + BT) / JW;                 // triangle: tiles below this one are the diagonal block's
  const int handed0 = max(jt0, diag_end) - jt0;          // triangle: tiles handed0 .. nt − 1 yield dZ_J

  const int tid = threadIdx.x;
  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(full_bar + 8 * s, 1); mbar_init(empty_bar + 8 * s, CONSUMERS / 32); }
    if constexpr (TRI) {
      for (int w = 0; w < 2; ++w) { mbar_init(gt_full + 8 * w, 4); mbar_init(gt_empty + 8 * w, 4); }
    }
    fence_barrier_init();
  }
  __syncthreads();

  if constexpr (TRI) {
    if (tid >= THREADS) {
      // ===================== dZ_J warpgroup =====================
      // dZ_J += Gᵀ · Z_I of every tile above the diagonal block, both consumer warpgroups' halves (K = their 64 rows i) in
      // turn into the same accumulators as one warpgroup's used to, each half summed into an fp32 total; the tile's total
      // then goes to dz with one set of reductions.  A consumer's Gᵀ planes are handed over through gt_full / gt_empty.
      asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(TriRegs<DP>::DJ));
      if (handed0 >= nt) return;
      const int t = tid - THREADS, warp = t >> 5, lane = t & 31;
      // each warpgroup half of Z_I in its 64-row tile's scale; the half's sum is unscaled before the two are added
      const int e0 = p.exps[2 * blockIdx.x], e1 = p.exps[2 * blockIdx.x + 1];
      const float sc_i[2] = {unscale(e0), unscale(e1)};
      // Z_Iᵀ (B of dZ_J) per consumer warpgroup: [DP hi rows | DP lo rows] x 64 i (fp16), scaled by 2^e; rows past the range
      // are zero
      for (int e = t; e < BT * DP; e += 128) {
        const int r = e / DP, k = e % DP;
        const int row = row0 + r;
        const float v = (row < row_end && k < p.d) ? p.z[(int64_t)row * p.ldz + k] : 0.f;
        const float x = ldexpf(v, (r >> 6) ? e1 : e0);
        const __half xh = __float2half_rn(x);
        const uint32_t q = (uint32_t)(r & 63);
        uint8_t* b = zit + (r >> 6) * T::ZIT;
        *reinterpret_cast<__half*>(b + sw128_offset16((uint32_t)k, q)) = xh;
        *reinterpret_cast<__half*>(b + sw128_offset16((uint32_t)(DP + k), q)) = __float2half_rn(x - __half2float(xh));
      }
      fence_proxy_async();
      asm volatile("bar.sync 4, 128;" ::: "memory");
      const bool vec = (p.d & 1) == 0 && (reinterpret_cast<uintptr_t>(p.dz) & 7) == 0;
      const float c2 = 2.f * p.coef;
      float djm[NBM][DP], djs[DP / 2], djt[DP / 2];
      for (int i = handed0; i < nt; ++i) {
        const uint32_t parity = (uint32_t)((i - handed0) & 1);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          mbar_wait(gt_full + 8 * h, parity);
          const uint32_t ag_hi = smem_u32(zit + 2 * T::ZIT + h * 2 * T::GT), ag_lo = ag_hi + T::GT;
          const uint32_t bi = smem_u32(zit) + h * T::ZIT;
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < 64 / 16; ++kk) {
            const uint32_t o = (uint32_t)kk * 32;
            mma_ss<F16, DP>(djs, wgmma_desc_sw128(ag_lo + o), wgmma_desc_sw128(bi + o), kk > 0);
            mma_ss<F16, 2 * DP>(djm[kk % NBM], wgmma_desc_sw128(ag_hi + o), wgmma_desc_sw128(bi + o), kk >= NBM);
          }
          wgmma_commit();
          wgmma_wait<0>();
          reg_fence(djs);
#pragma unroll
          for (int b = 0; b < NBM; ++b) reg_fence(djm[b]);
          __syncwarp();
          if (lane == 0) mbar_arrive(gt_empty + 8 * h);     // this warpgroup's Gᵀ is read
#pragma unroll
          for (int v = 0; v < DP / 2; ++v) djt[v] = (h ? djt[v] : 0.f) + merged(djm, djs, v) * sc_i[h];
        }
        const int ja = (jt0 + i) * JW + warp * 16 + (lane >> 2);
#pragma unroll
        for (int v = 0; v < DP / 2; v += 2) {
          const int row = ja + 8 * ((v >> 1) & 1);
          const int col = 8 * (v >> 2) + 2 * (lane & 3);
          if (row >= p.n || col >= p.d) continue;
          float* dst = p.dz + (int64_t)row * p.d + col;
          if (vec) {
            atomicAdd(reinterpret_cast<float2*>(dst), make_float2(c2 * djt[v], c2 * djt[v + 1]));
          } else {
            atomicAdd(dst, c2 * djt[v]);
            if (col + 1 < p.d) atomicAdd(dst + 1, c2 * djt[v + 1]);
          }
        }
      }
      return;
    }
  }

  if (tid >= CONSUMERS) {
    // ===================== producer warpgroup =====================
    // One thread issues the copies; the warpgroup exists so that it can hand its registers to the consumers.
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(TRI ? TriRegs<DP>::PRODUCER : PRODUCER_REGS));
    if (tid == CONSUMERS) {
      for (int i = 0; i < nt; ++i) {
        const int s = i % STAGES;
        if (i >= STAGES) mbar_wait(empty_bar + 8 * s, (uint32_t)((i / STAGES - 1) & 1));
        const uint32_t fb = full_bar + 8 * s, dst = smem_u32(ring + s * T::STAGE);
        const size_t t = (size_t)(jt0 + i);
        mbar_expect_tx(fb, T::STAGE);
        bulk_load(dst, p.zs_hi + t * T::JS, T::JS, fb);
        bulk_load(dst + T::JS, p.zs_lo + t * T::JS, T::JS, fb);
        if constexpr (TRI) {
          bulk_load(dst + 2 * T::JS, p.zt_hi + t * T::JT, T::JT, fb);   // [hi | lo], as the split kernel wrote it
        } else {
          bulk_load(dst + 2 * T::JS, p.zt_hi + t * T::JT, T::JT, fb);
          bulk_load(dst + 2 * T::JS + T::JT, p.zt_lo + t * T::JT, T::JT, fb);
        }
      }
    }
    return;
  }

  // ===================== consumers =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(TRI ? TriRegs<DP>::CONSUMER : CONSUMER_REGS));
  // Z_I planes from z (rows past the range are zero: their logits are masked below)
  for (int e = tid; e < BT * DP; e += CONSUMERS) {
    const int r = e / DP, k = e % DP;
    const int row = row0 + r;
    const float v = (row < row_end && k < p.d) ? p.z[(int64_t)row * p.ldz + k] : 0.f;
    const float h = tf32_hi(v);
    const uint32_t o = sw128_offset32((uint32_t)r, (uint32_t)k);
    *reinterpret_cast<float*>(zi_hi + o) = h;
    *reinterpret_cast<float*>(zi_lo + o) = v - h;
  }
  fence_proxy_async();
  asm volatile("bar.sync 1, %0;" ::"n"(CONSUMERS) : "memory");

  // The triangle broadcasts wg from lane 0 so that ptxas knows it is warp-uniform: the shared-memory descriptors of the
  // warpgroup's Gᵀ and Z_Iᵀ then live in uniform registers instead of taking consumer registers and an R2UR per wgmma.  The
  // full sweep has no per-warpgroup operand but Z_I and already issues few R2UR (26 for 108 HGMMAs at DP = 16).
  const int wg = TRI ? __shfl_sync(0xffffffffu, tid >> 7, 0) : tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
  const int ra = row0 + wg * 64 + warp * 16 + (lane >> 2);       // rows of this thread: ra, ra + 8
  const bool live_a = ra < row_end, live_b = ra + 8 < row_end;
  const uint32_t ai_hi = smem_u32(zi_hi) + wg * 64 * 128, ai_lo = smem_u32(zi_lo) + wg * 64 * 128;
  const bool full_rows = row0 + BT <= row_end;                   // no dead rows in this block: only the last J tile is masked
  // triangle: this warpgroup's Gᵀ planes (A of dZ_J); the address this lane gives stmatrix in the hi plane is column
  // 16·m + 8·(lane / 16) + lane % 8 of G (row j of Gᵀ, m = 0 .. 3 below), rows i from 16·warp + 8·((lane / 8) % 2) (the
  // 16-byte chunk of 8 i in the 128-byte swizzle)
  const uint32_t gt_hi = smem_u32(zit + 2 * T::ZIT + wg * 2 * T::GT) +
                         sw128_offset16((uint32_t)(8 * (lane >> 4) + (lane & 7)), (uint32_t)(16 * warp + 8 * ((lane >> 3) & 1)));
  const uint32_t gt_lo = gt_hi + T::GT;
  const float c2 = 2.f * p.coef;

  // The accumulation inside the tensor core truncates, and the hi·hi product carries almost all of dZ: over a whole J sweep one
  // accumulator would drift by ~1e-5 relative (~6e-5 for |z| ~ 1e5).  So the hi·hi products of a tile go round-robin into
  // several accumulators (at most 4 k-steps each for DP ≤ 16, 8 at DP = 32), the cross terms into one more, and the tile's sum
  // joins an fp32 total with round-to-nearest adds.  The full sweep issues the three products at N = DP (NB accumulators for
  // hi·hi).  The triangle has twice the dZ products per logit and issues fewer, wider ones: hi·hi and hi·lo as one N = 2·DP
  // product against [hi | lo] of the B operand (NBM accumulators), lo·hi alone; the same for dZ_J (dZ_J warpgroup).
  float dzb[TRI ? 1 : NB][DP / 2], dzs[DP / 2], dzt[DP / 2];
  float dzm[TRI ? NBM : 1][DP];
#pragma unroll
  for (int v = 0; v < DP / 2; ++v) dzt[v] = 0.f;
  double loss = 0.0;

  // Ping-pong: the two warpgroups take turns on the tensor cores.  A turn is the dZ product of the previous tile followed by the
  // S product of the next one, each issued as one batch with one commit (named barrier 2 + wg means "wg may issue"), and the
  // warpgroup works through σ / softplus of its S while the other one's products run.  Warpgroup 0 takes the first turn.  Each
  // warpgroup takes nt + 1 turns and passes nt of them on; warpgroup 0 passes its last one as well, so that every bar.arrive
  // meets one bar.sync.  In the triangle a turn holds dZ_I only: dZ_J of the tile runs on the dZ_J warpgroup, which takes each
  // warpgroup's Gᵀ through gt_full and gives it back through gt_empty once its wgmmas have retired.
  //   Full sweep: the dZ batch is waited for before S is issued into the same registers, and the turn passes on once S is done.
  //   Triangle (OVERLAP): S alternates between two accumulators, so the dZ_I batch of tile i − 1 (A = the previous S and L) and
  //     the S batch of tile i go out back to back and the turn passes on once both are committed; the tensor pipe does not
  //     drain within a turn, and the other warpgroup's batches queue behind them.  wait<1> then retires dZ_I while S still
  //     runs.  With dZ_J on its own warpgroup the second accumulator fits at every DP without spills, and it measured faster
  //     than one S accumulator at DP = 16 and 32 as well (DESIGN §4.1).
  constexpr bool OVERLAP = TRI;
  float S[JW / 2], L[JW / 2];   // S: accumulator of S, then the hi part of G; L: the lo part of G
  auto take_turn = [&]() { asm volatile("bar.sync %0, %1;" ::"r"(2 + wg), "n"(CONSUMERS) : "memory"); };
  auto pass_turn = [&]() { asm volatile("bar.arrive %0, %1;" ::"r"(3 - wg), "n"(CONSUMERS) : "memory"); };

  // S = Z_I · Z_Jᵀ of tile i into the accumulator S: one batch of 3·DP/8 products, committed (the caller waits)
  auto issue_s = [&](int i, float (&S)[JW / 2]) {
    const int s = i % STAGES;
    mbar_wait(full_bar + 8 * s, (uint32_t)((i / STAGES) & 1));
    const uint32_t bs_hi = smem_u32(ring + s * T::STAGE), bs_lo = bs_hi + T::JS;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < DP / 8; ++kk) {
      const uint32_t o = kk * 32;
      mma_ss<TF32, JW>(S, wgmma_desc_sw128(ai_lo + o), wgmma_desc_sw128(bs_hi + o), kk > 0);
      mma_ss<TF32, JW>(S, wgmma_desc_sw128(ai_hi + o), wgmma_desc_sw128(bs_lo + o), 1);
      mma_ss<TF32, JW>(S, wgmma_desc_sw128(ai_hi + o), wgmma_desc_sw128(bs_hi + o), 1);
    }
    wgmma_commit();
  };
  // dZ_I += G · Z_J of tile i with A = (S, L) from the registers; one batch, committed (the caller waits, then dz_fence).
  // Full sweep: 3·16 products; triangle: 2·4.
  auto issue_dz = [&](int i, float (&S)[JW / 2]) {
    const uint32_t bt_hi = smem_u32(ring + (i % STAGES) * T::STAGE) + 2 * T::JS, bt_lo = bt_hi + T::JT;
    wgmma_fence();
    if constexpr (TRI) {
      // A = G·2^14 as packed fp16 (sigmoid_softplus), in the natural column order; B = [Z_Jᵀ hi | Z_Jᵀ lo] rows, K = j
#pragma unroll
      for (int kb = 0; kb < JW / 16; ++kb) {
        const uint32_t ahi[4] = {__float_as_uint(S[4 * kb]), __float_as_uint(S[4 * kb + 1]), __float_as_uint(S[4 * kb + 2]),
                                 __float_as_uint(S[4 * kb + 3])};
        const uint32_t alo[4] = {__float_as_uint(L[4 * kb]), __float_as_uint(L[4 * kb + 1]), __float_as_uint(L[4 * kb + 2]),
                                 __float_as_uint(L[4 * kb + 3])};
        mma_rs<F16, DP>(dzs, alo, wgmma_desc_sw128(bt_hi + kb * 32), kb > 0);
        mma_rs<F16, 2 * DP>(dzm[kb % NBM], ahi, wgmma_desc_sw128(bt_hi + kb * 32), kb >= NBM);
      }
    } else {
#pragma unroll
      for (int kb = 0; kb < JW / 8; ++kb) {
        // A fragment (r, t) (r+8, t) (r, t+4) (r+8, t+4) in the permuted column order: (r, 2t) (r+8, 2t) (r, 2t+1) (r+8, 2t+1)
        const uint32_t ahi[4] = {__float_as_uint(S[4 * kb]), __float_as_uint(S[4 * kb + 2]), __float_as_uint(S[4 * kb + 1]),
                                 __float_as_uint(S[4 * kb + 3])};
        const uint32_t alo[4] = {__float_as_uint(L[4 * kb]), __float_as_uint(L[4 * kb + 2]), __float_as_uint(L[4 * kb + 1]),
                                 __float_as_uint(L[4 * kb + 3])};
        const uint32_t o = (uint32_t)(kb >> 2) * ATOM + (uint32_t)(kb & 3) * 32;
        mma_rs<TF32, DP>(dzs, alo, wgmma_desc_sw128(bt_hi + o), kb > 0);
        mma_rs<TF32, DP>(dzs, ahi, wgmma_desc_sw128(bt_lo + o), 1);
        mma_rs<TF32, DP>(dzb[kb % NB], ahi, wgmma_desc_sw128(bt_hi + o), kb >= NB);
      }
    }
    wgmma_commit();
  };
  auto dz_fence = [&]() {
    reg_fence(dzs);
    if constexpr (TRI) {
#pragma unroll
      for (int b = 0; b < NBM; ++b) reg_fence(dzm[b]);
    } else {
#pragma unroll
      for (int b = 0; b < NB; ++b) reg_fence(dzb[b]);
    }
  };
  // the tile's dZ_I joins the fp32 total and its stage goes back to the producer
  auto retire_dz = [&](int i, float sc) {
#pragma unroll
    for (int v = 0; v < DP / 2; ++v) {
      if constexpr (TRI) {
        dzt[v] += merged(dzm, dzs, v) * sc;
      } else {
        float t = dzs[v];
#pragma unroll
        for (int b = 0; b < NB; ++b) t += dzb[b][v];
        dzt[v] += t;
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(empty_bar + 8 * (i % STAGES));
  };
  // σ / softplus of tile i on the registers once its S is done; above the diagonal block the triangle then writes Gᵀ for the
  // dZ_J warpgroup, once that warpgroup has read the previous one
  auto elementwise = [&](int i, float (&S)[JW / 2]) {
    const int jbase = (jt0 + i) * JW + 2 * (lane & 3);
    const float l = full_rows && (jt0 + i + 1) * JW <= p.n ? sigmoid_softplus<false, JW / 2, TRI>(S, L, jbase, p.n, live_a, live_b)
                                                           : sigmoid_softplus<true, JW / 2, TRI>(S, L, jbase, p.n, live_a, live_b);
    if constexpr (TRI) {
      if (i >= handed0) {
        loss += 2.0 * (double)l;   // a tile above the diagonal block stands for its mirror too
        mbar_wait(gt_empty + 8 * wg, (uint32_t)(((i - handed0) & 1) ^ 1));
        // column j of G is row j of Gᵀ.  The packed registers S[2c], S[2c + 1] (and L) are the fragments of the 8 x 8 blocks
        // (rows r .. r + 7 and r + 8 .. r + 15 of the warp, columns 8c .. 8c + 7); stmatrix .trans writes four of them as rows
        // of Gᵀ, K-major in the natural i order.
#pragma unroll
        for (int m = 0; m < JW / 16; ++m) {
          stsm_x4_trans(gt_hi + m * 16 * 128, __float_as_uint(S[4 * m]), __float_as_uint(S[4 * m + 1]),
                        __float_as_uint(S[4 * m + 2]), __float_as_uint(S[4 * m + 3]));
          stsm_x4_trans(gt_lo + m * 16 * 128, __float_as_uint(L[4 * m]), __float_as_uint(L[4 * m + 1]),
                        __float_as_uint(L[4 * m + 2]), __float_as_uint(L[4 * m + 3]));
        }
        fence_proxy_async();
        __syncwarp();
        if (lane == 0) mbar_arrive(gt_full + 8 * wg);
      } else {
        loss += (double)l;
      }
    } else {
      loss += (double)l;
    }
  };

  if constexpr (OVERLAP) {
    float S2[JW / 2];
    // the turn of tile i ≥ 1: dZ of tile i − 1 from (Sp, L), then S of tile i into Sn
    // the scale of tile i − 1 is loaded before the waits
    auto tile_unscale = [&](int i) { return unscale(__ldg(p.exps + jt0 + i)); };
    auto turn = [&](int i, float (&Sp)[JW / 2], float (&Sn)[JW / 2]) {
      take_turn();
      issue_dz(i - 1, Sp);
      issue_s(i, Sn);
      pass_turn();
      const float sc = tile_unscale(i - 1);
      wgmma_wait<1>();     // dZ is done, S may still run
      dz_fence();
      retire_dz(i - 1, sc);
      wgmma_wait<0>();
      reg_fence(Sn);
      elementwise(i, Sn);
    };
    // the last turn: dZ of tile nt − 1 from (Sp, L)
    auto last = [&](float (&Sp)[JW / 2]) {
      take_turn();
      issue_dz(nt - 1, Sp);
      if (wg == 0) pass_turn();
      const float sc = tile_unscale(nt - 1);
      wgmma_wait<0>();
      dz_fence();
      retire_dz(nt - 1, sc);
    };
    if (wg == 1) take_turn();
    issue_s(0, S);
    pass_turn();
    wgmma_wait<0>();
    reg_fence(S);
    elementwise(0, S);
    // unrolled by two, so that which accumulator each batch reads and writes is known at compile time (ptxas serialises
    // wgmmas whose register operands it cannot tell apart)
    for (int i = 1;; i += 2) {
      if (i == nt) { last(S); break; }
      turn(i, S, S2);
      if (i + 1 == nt) { last(S2); break; }
      turn(i + 1, S2, S);
    }
  } else {
    auto run_dz = [&](int i) {
      issue_dz(i, S);
      wgmma_wait<0>();
      dz_fence();
    };
    // wait for S of tile i, pass the turn on, then σ / softplus
    auto finish_s = [&](int i) {
      wgmma_wait<0>();
      reg_fence(S);
      pass_turn();
      elementwise(i, S);
    };
    if (wg == 1) take_turn();
    issue_s(0, S);
    finish_s(0);
    for (int i = 1; i < nt; ++i) {
      take_turn();
      run_dz(i - 1);
      issue_s(i, S);       // S runs while the previous tile's dZ is summed
      retire_dz(i - 1, 1.f);
      finish_s(i);
    }
    take_turn();
    run_dz(nt - 1);
    retire_dz(nt - 1, 1.f);
    if (wg == 0) pass_turn();
  }

  // ---- epilogue ----
  // The triangle's rows also receive dZ_J from the CTAs of the blocks above, so it always adds atomically.
  const bool atomic = TRI || gridDim.y > 1;
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

template <int DP>
__global__ void __launch_bounds__(THREADS, 1)
gae_allpairs_tc_kernel(const __grid_constant__ Params p) {
  decoder_sweep<DP, false>(p);
}

template <int DP>
__global__ void __launch_bounds__(TRI_THREADS, 1)
gae_tri_tc_kernel(const __grid_constant__ Params p) {
  decoder_sweep<DP, true>(p);
}

size_t workspace_bytes(int32_t n) { return (size_t)padded_n(n) / BT * (ZS_PLANES * ZS_BYTES + 2 * zt_bytes<MAX_D>()); }

int super_blocks(int32_t n) { return (int)((padded_n(n) / BT + 1) / 2); }

bool eligible(int32_t n, int32_t d, int32_t n_rows, size_t ws_bytes) {
  const int mode = path_mode(B2_PATH_GAE_DECODER);           // 0 auto · 1 CUDA cores · 2 these kernels
  if (d < 1 || d > MAX_D || mode == 1 || ws_bytes < workspace_bytes(n)) return false;
  return mode == 2 || (int64_t)n * n_rows >= (1ll << 22);
}

template <int DP, bool TRI>
static int launch_sweep(const Params& p, int units, cudaStream_t st) {
  // J step ranges: b2_set_tuning(B2_TUNE_GAE_SPLITS) when set, else enough to fill one wave of SMs
  int splits = tuning(B2_TUNE_GAE_SPLITS);
  if (splits <= 0) splits = ceil_div(sm_count(), units);
  if (splits > p.n_jt) splits = p.n_jt;
  if (splits < 1) splits = 1;
  auto kernel = TRI ? gae_tri_tc_kernel<DP> : gae_allpairs_tc_kernel<DP>;
  constexpr size_t smem = Tiles<DP, TRI>::SMEM;
  static_assert(smem <= kMaxDynamicSmem, "decoder shared memory");
  const int rc = allow_dynamic_smem((const void*)kernel, smem);
  if (rc != B2_OK) return rc;
  kernel<<<dim3((unsigned)units, (unsigned)splits), TRI ? TRI_THREADS : THREADS, smem, st>>>(p);
  B2_CHECK_LAUNCH(TRI ? "gae_tri_tc_kernel" : "gae_allpairs_tc_kernel");
  return B2_OK;
}

// Splits z into the workspace planes, then sweeps `units` work units (none: the split only).  tri: every row against every
// column by the triangle (units must be the nb row blocks), which takes the fp16 split.
template <int DP>
static int launch_dp(Params p, int units, bool tri, void* ws, cudaStream_t st) {
  const int64_t npad = padded_n(p.n);
  p.nb = (int)(npad / BT);
  uint8_t* zs_hi = reinterpret_cast<uint8_t*>(ws);
  uint8_t* zs_lo = zs_hi + (size_t)p.nb * ZS_BYTES;
  uint8_t* zt_hi = zs_lo + (size_t)p.nb * ZS_BYTES;
  if (tri && units > 0) {
    // the fp16 Z_Jᵀ blocks (2·nb of 2·DP·128 bytes) and the tile exponents take the place of the tf32 Z_Jᵀ planes
    static_assert(2 * 2 * DP * 128 + 2 * sizeof(int) <= 2 * zt_bytes<MAX_D>(), "triangle workspace");
    int* exps = reinterpret_cast<int*>(zt_hi + (size_t)(2 * p.nb) * (2 * DP * 128));
    gae_split_f16_kernel<DP><<<(unsigned)(2 * p.nb), 256, 0, st>>>(p.z, p.ldz, p.n, p.d, zs_hi, zs_lo, zt_hi, exps);
    B2_CHECK_LAUNCH("gae_split_f16_kernel");
    p.zs_hi = zs_hi; p.zs_lo = zs_lo; p.zt_hi = zt_hi; p.exps = exps;
    p.n_jt = ceil_div(p.n, Tiles<DP, true>::JW);   // 64-column tiles holding at least one column j < n
    return launch_sweep<DP, true>(p, units, st);
  }
  uint8_t* zt_lo = zt_hi + (size_t)p.nb * zt_bytes<DP>();
  gae_split_kernel<DP><<<grid_blocks(npad * DP, 256), 256, 0, st>>>(p.z, p.ldz, p.n, p.d, npad, zs_hi, zs_lo, zt_hi, zt_lo);
  B2_CHECK_LAUNCH("gae_split_kernel");
  if (units <= 0) return B2_OK;
  p.zs_hi = zs_hi; p.zs_lo = zs_lo; p.zt_hi = zt_hi; p.zt_lo = zt_lo;
  p.n_jt = p.nb;
  return launch_sweep<DP, false>(p, units, st);
}

// Adds the all-pairs part into dz and loss_acc; ws holds workspace_bytes(n) bytes.  Row form (sym = false): rows [begin, end)
// against all n columns, dz[end - begin, d]; the call over all rows uses the symmetry of S (triangle), a row subset sweeps every
// column.  Pair-sharded form (sym = true): super-blocks [begin, end) against all n columns, dz[n, d] (the rows of those blocks).
int launch(const float* z, int64_t ldz, int32_t n, int32_t d, bool sym, int32_t begin, int32_t end, float coef, float* dz,
           double* loss_acc, void* ws, cudaStream_t st) {
  Params p;
  memset(&p, 0, sizeof(p));
  p.z = z; p.ldz = ldz; p.n = n; p.d = d; p.coef = coef; p.dz = dz; p.loss_acc = loss_acc; p.sym = sym;
  int units;
  if (sym) {
    p.sb_begin = begin;
    units = 2 * (end - begin);
  } else {
    p.row_begin = begin; p.row_end = end;
    units = ceil_div(end - begin, BT);
  }
  const bool tri = !sym && begin == 0 && end == n;
  if (d <= 8) return launch_dp<8>(p, units, tri, ws, st);
  if (d <= 16) return launch_dp<16>(p, units, tri, ws, st);
  return launch_dp<32>(p, units, tri, ws, st);
}

}  // namespace gtc
}  // namespace b2
