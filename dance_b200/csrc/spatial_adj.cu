// SpaGCN's spot graph from the spot coordinates, without the N × N matrices (reference spagcn.py:249-287 calculate_p / search_l,
// :290-334 refine, :337-366 GraphConvolution on adj_exp, :807-809 calc_adj_exp; spatial_graph.py:13-76 and utils/matrix.py
// pairwise_distance build the dense matrices this replaces).  Every pair's distance and weight come from spatial_pair.cuh, the
// functions the dense kernels use, so each one is the same bits as the dense path's entry.
//
//   spatial_exp_adj_mm_kernel<N>   AX[r, :] = Σ_c W(rows[r], cols[c]) · X[c, :] on the tensor cores.  A CTA owns 128 rows (two
//       consumer warpgroups of 64) and sweeps the columns in tiles of 32.  The consumers compute the tile's weights straight in
//       the register A fragment of wgmma m64nNk8 tf32 and split them into hi = w & 0xFFFFE000 and lo = w − hi; X comes as
//       pre-split hi / lo tf32 planes of X_Jᵀ (K-major in j, 128-byte swizzle), which one producer thread copies into a
//       four-stage mbarrier ring.  Per k-step: hi·hi into one accumulator, hi·lo + lo·hi into another (tf32 keeps fp32's
//       exponent range, so weights over many decades need no scaling).  The tensor core's accumulate truncates, so each tile
//       starts its accumulators afresh and their sum joins an fp32 total with round-to-nearest adds.  The weights of the next
//       tile are computed while the current tile's products run (two register buffers).
//   spatial_exp_adj_sum_kernel     Σ_{r,c} W in fp64 (CUDA cores; bound by the fp64 distance and MUFU, not by the sum).
//   spatial_nearest_kernel         per row the m ≤ 8 columns of smallest fp32 distance, ties to the lower column index and NaN
//       distances last: what torch.sort(dis, stable=True)[:, :m] returns on the materialised matrix.
#include "tc_common.cuh"
#include "spatial_pair.cuh"

#include <math_constants.h>

namespace b2 {
namespace sadj {

constexpr int MAXD = 4;                   // coordinates per spot; fewer are padded with zeros (adds +0.0, see pair_l2)
constexpr int BJ = 32;                    // columns per tile: 32 tf32 = one 128-byte swizzle row of the planes
constexpr int BM = 128;                   // rows per CTA
constexpr int CONSUMERS = 256;            // two warpgroups
constexpr int THREADS = CONSUMERS + 128;  // and a producer warpgroup, one thread of which issues the copies
// setmaxnreg split: at N = 64 a consumer holds acc, acc_x and tot (3 x 32) and two buffers of weight fragments (2 x 32);
// 128 · 40 + 256 · 232 = 64 512 of the 65 536 registers
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;
constexpr int STAGES = 4;
constexpr int MAX_N = 64;                 // widest feature chunk of one launch; wider X is swept in chunks
constexpr int NEAR_MAX = 8;               // nearest columns per row

__host__ __device__ constexpr uint32_t tile_bytes(int n) { return 2u * (uint32_t)n * 128u; }   // hi plane, then lo plane
static int chunk_width(int fc) { return fc <= 8 ? 8 : fc <= 16 ? 16 : fc <= 32 ? 32 : 64; }

__device__ __forceinline__ void load_point(const float* __restrict__ p, int64_t i, int d, float (&x)[MAXD]) {
#pragma unroll
  for (int c = 0; c < MAXD; ++c) x[c] = c < d ? __ldg(p + i * d + c) : 0.f;
}

// X[:, 0:fc] → tile t of the planes holds columns j = 32t … 32t+31 as N feature rows of 32 tf32 (K-major in j), hi then lo;
// features f ≥ fc and columns j ≥ n_cols are zero.
__global__ void __launch_bounds__(256)
spatial_planes_kernel(const float* __restrict__ X, int64_t ldx, int32_t n_cols, int32_t fc, int32_t N, int32_t tiles,
                      uint8_t* __restrict__ planes) {
  const int64_t total = (int64_t)tiles * BJ * N;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int f = (int)(e % N);
    const int64_t j = e / N;
    const float x = (j < n_cols && f < fc) ? X[j * ldx + f] : 0.f;
    const float hi = tc::tf32_hi(x);
    uint8_t* tile = planes + (j / BJ) * tile_bytes(N);
    const uint32_t off = tc::sw128_offset32((uint32_t)f, (uint32_t)(j % BJ));
    *reinterpret_cast<float*>(tile + off) = hi;
    *reinterpret_cast<float*>(tile + N * 128 + off) = x - hi;
  }
}

template <int N>
__global__ void __launch_bounds__(THREADS, 1)
spatial_exp_adj_mm_kernel(const float* __restrict__ rows, int32_t n_rows, const float* __restrict__ cols, int32_t n_cols, int32_t d,
                          float two_l2, const uint8_t* __restrict__ planes, int32_t tiles, int32_t fc, float* __restrict__ AX,
                          int64_t ldax) {
  using namespace tc;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // 128B-swizzle atoms: 1024-byte aligned
  constexpr uint32_t TB = tile_bytes(N);
  // full[s]: the stage's bytes landed; empty[s]: every consumer warp has retired the products that read it
  const uint32_t full = smem_u32(smem + STAGES * TB), empty = full + 8 * STAGES;
  const int tid = threadIdx.x;
  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full + 8 * s, 1);
      mbar_init(empty + 8 * s, CONSUMERS / 32);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (tid >= CONSUMERS) {
    // ===================== producer: one thread copies plane tiles into the ring =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PRODUCER_REGS));
    if (tid == CONSUMERS) {
      for (int t = 0; t < tiles; ++t) {
        const int s = t % STAGES;
        if (t >= STAGES) mbar_wait(empty + 8 * s, (uint32_t)(((t / STAGES) - 1) & 1));
        mbar_expect_tx(full + 8 * s, TB);
        bulk_load(smem_u32(smem + s * TB), planes + (size_t)t * TB, TB, full + 8 * s);
      }
    }
    return;
  }

  // ===================== consumers: weights in registers → wgmma =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONSUMER_REGS));
  const int wg = tid >> 7, lt = tid & 127, lane = lt & 31, kq = lane & 3;
  const int r0 = blockIdx.x * BM + wg * 64 + (lt >> 5) * 16 + (lane >> 2);   // this thread's rows: r0 and r0 + 8
  float p0[MAXD], p1[MAXD];
  load_point(rows, min(r0, n_rows - 1), d, p0);
  load_point(rows, min(r0 + 8, n_rows - 1), d, p1);

  // A fragment of k-step ks: a[0] = (r0, k), a[1] = (r0 + 8, k), a[2] = (r0, k + 4), a[3] = (r0 + 8, k + 4), k = lane % 4
  auto weights = [&](int t, uint32_t (&hi)[4][4], uint32_t (&lo)[4][4]) {
#pragma unroll
    for (int ks = 0; ks < 4; ++ks)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int j = t * BJ + ks * 8 + kq + 4 * h;
        float w0 = 0.f, w1 = 0.f;        // columns past n_cols weigh 0
        if (j < n_cols) {
          float q[MAXD];
          load_point(cols, j, d, q);
          w0 = exp_adj_weight(pair_l2(p0, q, MAXD), two_l2);
          w1 = exp_adj_weight(pair_l2(p1, q, MAXD), two_l2);
        }
        const float h0 = tf32_hi(w0), h1 = tf32_hi(w1);
        hi[ks][2 * h] = __float_as_uint(h0);
        lo[ks][2 * h] = __float_as_uint(w0 - h0);
        hi[ks][2 * h + 1] = __float_as_uint(h1);
        lo[ks][2 * h + 1] = __float_as_uint(w1 - h1);
      }
  };
  // hi·hi into acc, the cross terms into acc_x; the first product of a tile overwrites (scale-d = 0), so no ordinary
  // instruction defines an accumulator (ptxas would serialise every wgmma, C7515)
  float acc[N / 2], acc_x[N / 2], tot[N / 2];
#pragma unroll
  for (int v = 0; v < N / 2; ++v) tot[v] = 0.f;
  auto issue = [&](int t, const uint32_t (&hi)[4][4], const uint32_t (&lo)[4][4]) {
    const int s = t % STAGES;
    mbar_wait(full + 8 * s, (uint32_t)((t / STAGES) & 1));
    wgmma_fence();
    const uint32_t bh = smem_u32(smem + s * TB), bl = bh + N * 128;
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      mma_rs<TF32, N>(acc, hi[ks], wgmma_desc_sw128(bh + ks * 32), ks != 0);
      mma_rs<TF32, N>(acc_x, hi[ks], wgmma_desc_sw128(bl + ks * 32), ks != 0);
      mma_rs<TF32, N>(acc_x, lo[ks], wgmma_desc_sw128(bh + ks * 32), 1);
    }
    wgmma_commit();
  };
  auto retire = [&](int t) {
    wgmma_wait<0>();
    reg_fence(acc);
    reg_fence(acc_x);
#pragma unroll
    for (int v = 0; v < N / 2; ++v) tot[v] += acc[v] + acc_x[v];
    __syncwarp();
    if (lane == 0) mbar_arrive(empty + 8 * (t % STAGES));
  };
  uint32_t ha[4][4], la[4][4], hb[4][4], lb[4][4];
  weights(0, ha, la);
  for (int t = 0; t < tiles; t += 2) {
    issue(t, ha, la);
    if (t + 1 < tiles) weights(t + 1, hb, lb);     // under tile t's products
    retire(t);
    if (t + 1 < tiles) {
      issue(t + 1, hb, lb);
      if (t + 2 < tiles) weights(t + 2, ha, la);
      retire(t + 1);
    }
  }

  // accumulator element v: row r0 + 8·((v >> 1) & 1), column 8·(v >> 2) + 2·(lane % 4) + (v & 1)
#pragma unroll
  for (int v = 0; v < N / 2; ++v) {
    const int row = r0 + 8 * ((v >> 1) & 1), col = 8 * (v >> 2) + 2 * kq + (v & 1);
    if (row < n_rows && col < fc) AX[(int64_t)row * ldax + col] = tot[v];
  }
}

constexpr int SUM_ROWS = 64;   // rows per block of the weight total; each thread sweeps its columns against all of them

__global__ void __launch_bounds__(256)
spatial_exp_adj_sum_kernel(const float* __restrict__ rows, int32_t n_rows, const float* __restrict__ cols, int32_t n_cols, int32_t d,
                           float two_l2, double* __restrict__ acc) {
  __shared__ float rp[SUM_ROWS][MAXD];
  const int64_t rb = (int64_t)blockIdx.x * SUM_ROWS;
  const int nr = (int)min((int64_t)SUM_ROWS, n_rows - rb);
  for (int t = threadIdx.x; t < SUM_ROWS * MAXD; t += blockDim.x) {
    const int r = t / MAXD, c = t % MAXD;
    rp[r][c] = (r < nr && c < d) ? rows[(rb + r) * d + c] : 0.f;
  }
  __syncthreads();
  double local = 0.0;
  for (int64_t j = (int64_t)blockIdx.y * blockDim.x + threadIdx.x; j < n_cols; j += (int64_t)gridDim.y * blockDim.x) {
    float q[MAXD];
    load_point(cols, j, d, q);
    for (int r = 0; r < nr; ++r) local += (double)exp_adj_weight(pair_l2(rp[r], q, MAXD), two_l2);
  }
  local = warp_sum(local);
  if ((threadIdx.x & 31) == 0 && local != 0.0) atomicAdd(acc, local);
}

// the order of torch.sort(stable=True): by distance, NaN after every number (+inf included), equal keys by column index
__device__ __forceinline__ bool near_less(float da, int ia, float db, int ib) {
  const bool na = isnan(da), nb = isnan(db);
  if (na != nb) return nb;
  return (na || da == db) ? ia < ib : da < db;
}

// one warp per row: each lane keeps the 8 smallest (distance, column) of its columns sorted, then m rounds of a warp arg-min
// over the lanes' heads.  An empty slot is (NaN, INT_MAX), after every real column, so with m <= n_cols every index written
// is a real column even where distances are NaN.
__global__ void __launch_bounds__(256)
spatial_nearest_kernel(const float* __restrict__ rows, int32_t n_rows, const float* __restrict__ cols, int32_t n_cols, int32_t d,
                       int32_t m, int32_t* __restrict__ idx_out) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < n_rows; r += nwarps) {
    float p[MAXD];
    load_point(rows, r, d, p);
    float bd[NEAR_MAX];
    int bi[NEAR_MAX];
#pragma unroll
    for (int s = 0; s < NEAR_MAX; ++s) { bd[s] = CUDART_NAN_F; bi[s] = 0x7fffffff; }
    for (int j = lane; j < n_cols; j += 32) {
      float q[MAXD];
      load_point(cols, j, d, q);
      const float dist = pair_l2(p, q, MAXD);
      if (near_less(dist, j, bd[NEAR_MAX - 1], bi[NEAR_MAX - 1])) {
        bd[NEAR_MAX - 1] = dist;
        bi[NEAR_MAX - 1] = j;
#pragma unroll
        for (int s = NEAR_MAX - 1; s > 0; --s)
          if (near_less(bd[s], bi[s], bd[s - 1], bi[s - 1])) {
            const float td = bd[s]; bd[s] = bd[s - 1]; bd[s - 1] = td;
            const int ti = bi[s]; bi[s] = bi[s - 1]; bi[s - 1] = ti;
          }
      }
    }
    for (int k = 0; k < m; ++k) {
      float wd = bd[0];
      int wi = bi[0];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float od = __shfl_xor_sync(0xffffffffu, wd, o);
        const int oi = __shfl_xor_sync(0xffffffffu, wi, o);
        if (near_less(od, oi, wd, wi)) { wd = od; wi = oi; }
      }
      if (bi[0] == wi) {   // column indices are distinct across lanes: exactly one lane pops its head
#pragma unroll
        for (int s = 0; s < NEAR_MAX - 1; ++s) { bd[s] = bd[s + 1]; bi[s] = bi[s + 1]; }
        bd[NEAR_MAX - 1] = CUDART_NAN_F;
        bi[NEAR_MAX - 1] = 0x7fffffff;
      }
      if (lane == 0) idx_out[r * m + k] = wi;
    }
  }
}

template <int N>
static int launch_mm(const float* rows, int32_t n_rows, const float* cols, int32_t n_cols, int32_t d, float two_l2,
                     const uint8_t* planes, int32_t tiles, int32_t fc, float* AX, int64_t ldax, cudaStream_t st) {
  const size_t smem = STAGES * tile_bytes(N) + 16 * STAGES + 1024;
  const int rc = allow_dynamic_smem((const void*)spatial_exp_adj_mm_kernel<N>, smem);
  if (rc != B2_OK) return rc;
  spatial_exp_adj_mm_kernel<N><<<(unsigned)ceil_div(n_rows, BM), THREADS, smem, st>>>(rows, n_rows, cols, n_cols, d, two_l2, planes,
                                                                                       tiles, fc, AX, ldax);
  B2_CHECK_LAUNCH("spatial_exp_adj_mm_kernel");
  return B2_OK;
}

}  // namespace sadj
}  // namespace b2

using namespace b2;
using namespace b2::sadj;

extern "C" size_t b2_spatial_exp_adj_mm_workspace_bytes(int32_t n_cols, int32_t F) {
  if (n_cols <= 0 || F <= 0) return 0;
  return (size_t)ceil_div(n_cols, BJ) * tile_bytes(chunk_width(F < MAX_N ? F : MAX_N));
}

extern "C" int b2_spatial_exp_adj_mm_f32(const float* rows, int32_t n_rows, const float* cols, int32_t n_cols, int32_t d, double l,
                                         const float* X, int64_t ldx, int32_t F, float* AX, int64_t ldax, void* workspace,
                                         size_t workspace_bytes, void* stream) {
  B2_REQUIRE(rows && cols && X && AX, "b2_spatial_exp_adj_mm_f32: null pointer");
  B2_REQUIRE(d >= 1 && d <= MAXD, "b2_spatial_exp_adj_mm_f32: d=%d outside 1..%d", d, MAXD);
  B2_REQUIRE(l > 0.0 && isfinite(l), "b2_spatial_exp_adj_mm_f32: l must be positive and finite");
  B2_REQUIRE(n_rows >= 1 && n_cols >= 1 && F >= 1 && ldx >= F && ldax >= F, "b2_spatial_exp_adj_mm_f32: bad shape");
  const size_t need = b2_spatial_exp_adj_mm_workspace_bytes(n_cols, F);
  B2_REQUIRE(workspace && workspace_bytes >= need && (reinterpret_cast<uintptr_t>(workspace) & 15) == 0,
             "b2_spatial_exp_adj_mm_f32: workspace must be 16-byte aligned and hold %zu bytes", need);
  cudaStream_t st = as_stream(stream);
  const float two_l2 = exp_adj_two_l2(l);
  const int32_t tiles = ceil_div(n_cols, BJ);
  uint8_t* planes = reinterpret_cast<uint8_t*>(workspace);
  for (int32_t f0 = 0; f0 < F; f0 += MAX_N) {
    const int32_t fc = F - f0 < MAX_N ? F - f0 : MAX_N;
    const int N = chunk_width(fc);
    spatial_planes_kernel<<<grid_blocks((int64_t)tiles * BJ * N, 256), 256, 0, st>>>(X + f0, ldx, n_cols, fc, N, tiles, planes);
    B2_CHECK_LAUNCH("spatial_planes_kernel");
    int rc;
    if (N == 8) rc = launch_mm<8>(rows, n_rows, cols, n_cols, d, two_l2, planes, tiles, fc, AX + f0, ldax, st);
    else if (N == 16) rc = launch_mm<16>(rows, n_rows, cols, n_cols, d, two_l2, planes, tiles, fc, AX + f0, ldax, st);
    else if (N == 32) rc = launch_mm<32>(rows, n_rows, cols, n_cols, d, two_l2, planes, tiles, fc, AX + f0, ldax, st);
    else rc = launch_mm<64>(rows, n_rows, cols, n_cols, d, two_l2, planes, tiles, fc, AX + f0, ldax, st);
    if (rc != B2_OK) return rc;
  }
  return B2_OK;
}

extern "C" int b2_spatial_exp_adj_sum_f32(const float* rows, int32_t n_rows, const float* cols, int32_t n_cols, int32_t d, double l,
                                          double* sum_out_dev, void* stream) {
  B2_REQUIRE(rows && cols && sum_out_dev, "b2_spatial_exp_adj_sum_f32: null pointer");
  B2_REQUIRE(d >= 1 && d <= MAXD, "b2_spatial_exp_adj_sum_f32: d=%d outside 1..%d", d, MAXD);
  B2_REQUIRE(l > 0.0 && isfinite(l), "b2_spatial_exp_adj_sum_f32: l must be positive and finite");
  B2_REQUIRE(n_rows >= 0 && n_cols >= 0, "b2_spatial_exp_adj_sum_f32: bad shape");
  cudaStream_t st = as_stream(stream);
  B2_CHECK_CUDA(cudaMemsetAsync(sum_out_dev, 0, sizeof(double), st));
  if (n_rows == 0 || n_cols == 0) return B2_OK;
  const dim3 grid((unsigned)ceil_div(n_rows, SUM_ROWS), (unsigned)std::min<int64_t>(ceil_div(n_cols, 256), 65535));
  spatial_exp_adj_sum_kernel<<<grid, 256, 0, st>>>(rows, n_rows, cols, n_cols, d, exp_adj_two_l2(l), sum_out_dev);
  B2_CHECK_LAUNCH("spatial_exp_adj_sum_kernel");
  return B2_OK;
}

extern "C" int b2_spatial_nearest_f32(const float* rows, int32_t n_rows, const float* cols, int32_t n_cols, int32_t d, int32_t m,
                                      int32_t* idx_out, void* stream) {
  B2_REQUIRE(rows && cols && idx_out, "b2_spatial_nearest_f32: null pointer");
  B2_REQUIRE(d >= 1 && d <= MAXD, "b2_spatial_nearest_f32: d=%d outside 1..%d", d, MAXD);
  B2_REQUIRE(m >= 1 && m <= NEAR_MAX && m <= n_cols && n_rows >= 0, "b2_spatial_nearest_f32: need 1 <= m <= min(%d, n_cols)",
             NEAR_MAX);
  if (n_rows == 0) return B2_OK;
  spatial_nearest_kernel<<<grid_blocks(n_rows, 8), 256, 0, as_stream(stream)>>>(rows, n_rows, cols, n_cols, d, m, idx_out);
  B2_CHECK_LAUNCH("spatial_nearest_kernel");
  return B2_OK;
}
