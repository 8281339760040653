// Exact euclidean k-nearest-neighbour search: filter (fp32 tile distances, per-query
// candidate lists) → refine (fp64 re-rank exactly like the reference) → verify
// (error-bound proof that no non-candidate can enter the top-k) → rare fallback
// (fp64 brute force for unproven queries).  That path keeps at most KMAXC candidates per
// query; larger k (k + r0 + 8 > KMAXC) runs the batched estimate / select / collect /
// refine path at the end of this file, which has no such limit.
//
// Reference being replaced: calculateKNNgraphDistanceMatrixStatsSingleThread
// (scgnn2.py:675-689): per row scipy `cdist(..., "euclidean")` in fp64 on the fp32
// features, `argsort`, take sorted ranks 1..k.  Also the kNN inside NeighborGraph
// (neighbor_graph.py:50-57) and StagateGraph (spatial_graph.py:147-149).
#include "common.cuh"
#include "spatial_pair.cuh"

#include <cub/block/block_scan.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_sort.cuh>
#include <math_constants.h>

#include <vector>

namespace b2 {

constexpr int KQ = 64;    // queries per CTA
constexpr int KR = 128;   // reference points per tile
constexpr int KK = 16;    // feature chunk
constexpr int KTHREADS = 256;
constexpr int KMAXC = 64; // max candidates kept per query

__global__ void __launch_bounds__(256)
row_sqnorm_kernel(const float* __restrict__ X, int64_t ldx, int32_t n, int32_t d, float* __restrict__ out,
                  float* __restrict__ max_out) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  float local_max = 0.f;
  for (int64_t r = warp; r < n; r += nwarps) {
    float s = 0.f;
    for (int c = lane; c < d; c += 32) { const float v = X[r * ldx + c]; s = fmaf(v, v, s); }
    s = warp_sum(s);
    if (lane == 0) out[r] = s;
    local_max = fmaxf(local_max, s);
  }
  if (lane == 0) atomicMax(reinterpret_cast<int*>(max_out), __float_as_int(local_max));  // non-negative floats order as ints
}

// ---- phase 1: candidate generation ------------------------------------------
template <int M>
__global__ void __launch_bounds__(KTHREADS)
knn_candidates_kernel(const float* __restrict__ X, int64_t ldx, const float* __restrict__ sqn, int32_t n, int32_t d,
                      int32_t q_begin, int32_t n_q, int32_t* __restrict__ cand_idx, float* __restrict__ cand_thr) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float (*Qs)[KQ + 4] = reinterpret_cast<float (*)[KQ + 4]>(smem_raw);
  float (*Rs)[KR + 4] = reinterpret_cast<float (*)[KR + 4]>(smem_raw + sizeof(float) * KK * (KQ + 4));
  float (*Ds)[KR + 1] = reinterpret_cast<float (*)[KR + 1]>(smem_raw + sizeof(float) * KK * (KQ + 4 + KR + 4));
  float (*Lk)[M] = reinterpret_cast<float (*)[M]>(smem_raw + sizeof(float) * (KK * (KQ + 4 + KR + 4) + KQ * (KR + 1)));
  int32_t (*Li)[M] = reinterpret_cast<int32_t (*)[M]>(reinterpret_cast<unsigned char*>(Lk) + sizeof(float) * KQ * M);

  const int tid = threadIdx.x;
  const int tq = tid >> 4, tr = tid & 15;   // 16 x 16 thread grid: 4 queries x 8 refs each
  const int q0 = blockIdx.x * KQ;            // local query offset

  for (int t = tid; t < KQ * M; t += KTHREADS) { (&Lk[0][0])[t] = CUDART_INF_F; (&Li[0][0])[t] = -1; }

  float qn[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int q = q0 + tq * 4 + i;
    qn[i] = (q < n_q) ? sqn[q_begin + q] : 0.f;
  }

  for (int r0 = 0; r0 < n; r0 += KR) {
    float acc[4][8];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

    for (int k0 = 0; k0 < d; k0 += KK) {
      __syncthreads();
      // Q tile: 64 x 16, R tile: 128 x 16 ; consecutive threads read consecutive features (64 B segments)
#pragma unroll
      for (int i = 0; i < (KQ * KK) / KTHREADS; ++i) {
        const int idx = tid + i * KTHREADS;
        const int k = idx & (KK - 1), q = idx >> 4;
        const int gq = q0 + q, gk = k0 + k;
        Qs[k][q] = (gq < n_q && gk < d) ? X[(int64_t)(q_begin + gq) * ldx + gk] : 0.f;
      }
#pragma unroll
      for (int i = 0; i < (KR * KK) / KTHREADS; ++i) {
        const int idx = tid + i * KTHREADS;
        const int k = idx & (KK - 1), r = idx >> 4;
        const int gr = r0 + r, gk = k0 + k;
        Rs[k][r] = (gr < n && gk < d) ? X[(int64_t)gr * ldx + gk] : 0.f;
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < KK; ++k) {
        const float4 a = *reinterpret_cast<const float4*>(&Qs[k][tq * 4]);
        const float4 b0 = *reinterpret_cast<const float4*>(&Rs[k][tr * 4]);
        const float4 b1 = *reinterpret_cast<const float4*>(&Rs[k][64 + tr * 4]);
        const float av[4] = {a.x, a.y, a.z, a.w};
        const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
      }
    }
    // d² = |q|² + |r|² - 2 q·r  → shared tile
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int rl = (j < 4) ? tr * 4 + j : 64 + tr * 4 + (j - 4);
      const int gr = r0 + rl;
      const float rn = (gr < n) ? sqn[gr] : CUDART_INF_F;
#pragma unroll
      for (int i = 0; i < 4; ++i) Ds[tq * 4 + i][rl] = fmaf(-2.f, acc[i][j], qn[i] + rn);
    }
    __syncthreads();
    // selection: thread t owns query t
    if (tid < KQ) {
      float thr = Lk[tid][M - 1];
      for (int j = 0; j < KR; ++j) {
        const float v = Ds[tid][j];
        if (v < thr) {
          int p = M - 1;
          while (p > 0 && Lk[tid][p - 1] > v) { Lk[tid][p] = Lk[tid][p - 1]; Li[tid][p] = Li[tid][p - 1]; --p; }
          Lk[tid][p] = v;
          Li[tid][p] = r0 + j;
          thr = Lk[tid][M - 1];
        }
      }
    }
  }
  __syncthreads();
  for (int t = tid; t < KQ * M; t += KTHREADS) {
    const int q = t / M, c = t % M;
    if (q0 + q < n_q) cand_idx[(int64_t)(q0 + q) * M + c] = Li[q][c];
  }
  if (tid < KQ && q0 + tid < n_q) cand_thr[q0 + tid] = Lk[tid][M - 1];
}

// fp64 squared distance evaluated exactly like the reference's scipy cdist on doubles:
// sequential over features, no fused multiply-add.
__device__ __forceinline__ double exact_sqdist(const float* __restrict__ a, const float* __restrict__ b, int d) {
  double s = 0.0;
  for (int c = 0; c < d; ++c) {
    const double diff = __dsub_rn((double)a[c], (double)b[c]);
    s = __dadd_rn(s, __dmul_rn(diff, diff));
  }
  return s;
}

__device__ __forceinline__ bool lex_less(double da, int ia, double db, int ib) {
  return da < db || (da == db && ia < ib);
}

// ---- phase 2: refine + verify (one warp per query) ----------------------------
template <int M>
__global__ void __launch_bounds__(256)
knn_refine_kernel(const float* __restrict__ X, int64_t ldx, const float* __restrict__ sqn,
                  const float* __restrict__ max_sqn, int32_t n, int32_t d, int32_t k, int32_t q_begin, int32_t n_q,
                  int r0, const int32_t* __restrict__ cand_idx, const float* __restrict__ cand_thr, float err_rel,
                  int32_t* __restrict__ idx_out, double* __restrict__ dist_out, int32_t* __restrict__ fail_list,
                  int32_t* __restrict__ fail_count) {
  constexpr int PER = M / 32;
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t q = warp; q < n_q; q += nwarps) {
    const float* xq = X + (int64_t)(q_begin + q) * ldx;
    double dist[PER];
    int cidx[PER];
#pragma unroll
    for (int u = 0; u < PER; ++u) {
      cidx[u] = cand_idx[q * M + lane + 32 * u];
      dist[u] = (cidx[u] >= 0) ? sqrt(exact_sqdist(xq, X + (int64_t)cidx[u] * ldx, d)) : CUDART_INF;
      if (cidx[u] < 0) cidx[u] = 0x7fffffff;
    }
    // rank of each candidate under (distance, index)
    int rank[PER];
#pragma unroll
    for (int u = 0; u < PER; ++u) rank[u] = 0;
#pragma unroll
    for (int v = 0; v < PER; ++v) {
      for (int src = 0; src < 32; ++src) {
        const double od = __shfl_sync(0xffffffffu, dist[v], src);
        const int oi = __shfl_sync(0xffffffffu, cidx[v], src);
#pragma unroll
        for (int u = 0; u < PER; ++u) rank[u] += lex_less(od, oi, dist[u], cidx[u]) ? 1 : 0;
      }
    }
    double worst = 0.0;  // exact distance of the last returned rank
#pragma unroll
    for (int u = 0; u < PER; ++u) {
      const int pos = rank[u] - r0;
      if (pos >= 0 && pos < k) {
        idx_out[q * k + pos] = cidx[u];
        if (dist_out) dist_out[q * k + pos] = dist[u];
      }
      if (rank[u] == r0 + k - 1) worst = dist[u];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) worst = fmax(worst, __shfl_xor_sync(0xffffffffu, worst, o));
    if (lane == 0) {
      bool proven = (n <= M);
      if (!proven) {
        // every non-candidate has fp32 estimate >= thr; |estimate - true d²| <= err
        const double qn = (double)sqn[q_begin + q], rmax = (double)max_sqn[0];
        const double err = (double)err_rel * (qn + rmax + 2.0 * sqrt(qn * rmax));   // err_rel: bound of the filter that produced thr
        const double thr = (double)cand_thr[q];
        proven = isfinite(worst) && (thr - err) > worst * worst * (1.0 + 1e-12);
      }
      if (!proven) fail_list[atomicAdd(fail_count, 1)] = (int32_t)q;
    }
  }
}

// ---- phase 3: fp64 brute force for unproven queries ----------------------------
__global__ void __launch_bounds__(256)
knn_fallback_kernel(const float* __restrict__ X, int64_t ldx, int32_t n, int32_t d, int32_t k, int32_t q_begin, int r0,
                    const int32_t* __restrict__ fail_list, const int32_t* __restrict__ fail_count,
                    int32_t* __restrict__ idx_out, double* __restrict__ dist_out) {
  __shared__ double s_d[256];
  __shared__ int s_i[256];
  __shared__ double prev_d;
  __shared__ int prev_i;
  const int nfail = *fail_count;
  for (int f = blockIdx.x; f < nfail; f += gridDim.x) {
    const int q = fail_list[f];
    const float* xq = X + (int64_t)(q_begin + q) * ldx;
    if (threadIdx.x == 0) { prev_d = -1.0; prev_i = -1; }
    __syncthreads();
    for (int round = 0; round < r0 + k; ++round) {
      const double pd = prev_d;
      const int pi = prev_i;
      double bd = CUDART_INF;
      int bi = 0x7fffffff;
      for (int r = threadIdx.x; r < n; r += blockDim.x) {
        const double dd = sqrt(exact_sqdist(xq, X + (int64_t)r * ldx, d));
        if (lex_less(pd, pi, dd, r) && lex_less(dd, r, bd, bi)) { bd = dd; bi = r; }
      }
      s_d[threadIdx.x] = bd;
      s_i[threadIdx.x] = bi;
      __syncthreads();
      for (int s = 128; s > 0; s >>= 1) {
        if (threadIdx.x < s && lex_less(s_d[threadIdx.x + s], s_i[threadIdx.x + s], s_d[threadIdx.x], s_i[threadIdx.x])) {
          s_d[threadIdx.x] = s_d[threadIdx.x + s];
          s_i[threadIdx.x] = s_i[threadIdx.x + s];
        }
        __syncthreads();
      }
      if (threadIdx.x == 0) {
        prev_d = s_d[0];
        prev_i = s_i[0];
        const int pos = round - r0;
        if (pos >= 0) {
          idx_out[(int64_t)q * k + pos] = s_i[0];
          if (dist_out) dist_out[(int64_t)q * k + pos] = s_d[0];
        }
      }
      __syncthreads();
    }
  }
}

// dense fp32 euclidean matrix, each entry pair_l2 (spatial_pair.cuh)
__global__ void __launch_bounds__(256)
pairwise_dense_kernel(const float* __restrict__ X, int64_t ldx, int32_t n, int32_t d, float* __restrict__ D,
                      int64_t ldd) {
  const int64_t total = (int64_t)n * n;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / n, j = t % n;
    D[i * ldd + j] = pair_l2(X + i * ldx, X + j * ldx, d);
  }
}

// ---- large k: batched estimate → radix select → collect → fp64 refine -------------------------------------------
// Per batch of bq queries: S = X_q · Xᵀ by b2_gemm_f32 in tf32x3 into a [bq, n] fp32 block of at most LK_BLOCK_BYTES; the
// estimate d̂² = fmaf(−2, S, |q|² + |r|²); e_K, its K-th smallest value per query (K = k + r0), by a three-pass radix select
// over the float bits; every reference with d̂² ≤ thr_q = e_K + 2·err_q (plus a relative margin) collected in ascending index
// order; their fp64 distances (exact_sqdist, then sqrt) stable-sorted per query, so index order breaks ties; ranks r0 … r0+k−1.
//
// Exactness: |d̂² − D| ≤ err_q for every reference of query q, D = exact_sqdist.  The K references with the smallest estimates
// all have D ≤ e_K + err_q, so the K-th smallest D is at most e_K + err_q, and every reference of the top K, or tied with the
// K-th, has d̂² ≤ D + err_q ≤ e_K + 2·err_q: it is collected.  The margin |e_K + err_q|·1e-12 (as the SIMT proof's 1 + 1e-12)
// also keeps references whose sqrt rounds equal to the K-th distance's.  No query is left unproven.
//
// err_q = lk_err_rel(d, dp) · (|q|² + R² + 2|q|R), R² = max |r|², dp = d rounded up to 4 (zero columns add nothing):
//   tf32x3 operands: hi = x & 0xFFFFE000, lo = x − hi with |lo| < 2^-10 |x|; the MMA truncates lo to tf32 (|Δlo| < 2^-10 |lo|),
//     lo·lo is dropped: per product |Δ(q_i r_i)| < (2^-20 + 2^-20 + 2^-20) |q_i||r_i|, summed ≤ 3·2^-20 |q||r|
//   fp32 accumulation of the 3·dp products, of the two accumulators and of at most dp/128 split-K partials, every add bounded
//     as if it truncated: ≤ (3.1·dp + 4)·2^-23 Σ|terms|, Σ|terms| ≤ (1 + 2^-9)|q||r|, so ≤ (3.2·dp + 5)·2^-23 |q||r| (the
//     CUDA-core fallback of b2_gemm_f32, dp fused products, is inside the same bound)
//   2|ΔS| ≤ (3·2^-20 + (3.2·dp + 5)·2^-23) · 2|q||r|, and 2|q||r| ≤ |q|² + R² + 2|q|R
//   fp32 norms, |q|² + |r|² and the fma: (d + 8)·2^-23 (|q|² + |r|²) as for the SIMT filter; D's own fp64 rounding
//     (≤ d·2^-52 (|q| + |r|)²) fits in the spare 2^-23.
constexpr int LK_THREADS = 512;
constexpr size_t LK_BLOCK_BYTES = size_t(1) << 31;   // the [bq, n] estimate block

static double lk_err_rel(int32_t d, int32_t dp) {
  return 3.0 * 0x1p-20 + (3.2 * dp + (double)d + 14.0) * 0x1p-23;
}

__device__ __forceinline__ uint32_t lk_key(float f) {     // float order → unsigned order
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float lk_unkey(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// the estimate of reference j for the query whose S row is `s`: one expression for every pass
__device__ __forceinline__ float lk_est(const float* __restrict__ s, const float* __restrict__ sqn, float qn, int j) {
  return fmaf(-2.f, s[j], qn + sqn[j]);
}

__global__ void __launch_bounds__(256)
knn_lk_pad_kernel(const float* __restrict__ X, int64_t ldx, int32_t n, int32_t d, int32_t dp, float* __restrict__ Xp) {
  const int64_t total = (int64_t)n * dp;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / dp;
    const int c = (int)(t % dp);
    Xp[t] = c < d ? X[i * ldx + c] : 0.f;
  }
}

// one CTA per query row of the batch: e_K by radix select (11 + 11 + 10 bits, shared-memory histograms), then thr_q and the
// number of references with d̂² ≤ thr_q
__global__ void __launch_bounds__(LK_THREADS)
knn_lk_select_kernel(const float* __restrict__ S, int64_t lds, const float* __restrict__ sqn, const float* __restrict__ max_sqn,
                     int32_t n, int32_t q0, int32_t K, double err_rel, double* __restrict__ thr_out, int32_t* __restrict__ count_out) {
  using Scan = cub::BlockScan<int, LK_THREADS>;
  __shared__ typename Scan::TempStorage scan_tmp;
  __shared__ int hist[2048];
  __shared__ uint32_t s_bin;
  __shared__ int s_rem;
  const int tid = threadIdx.x;
  const int64_t row = blockIdx.x;
  const float* s = S + row * lds;
  const float qn = sqn[q0 + row];
  uint32_t prefix = 0;
  int rem = K;                                      // rank (1-based) of e_K among the keys that share `prefix`
#pragma unroll 1
  for (int pass = 0; pass < 3; ++pass) {
    const int shift = pass == 0 ? 21 : (pass == 1 ? 10 : 0);
    const uint32_t bin_mask = pass == 2 ? 1023u : 2047u;
    const uint32_t hi_mask = pass == 0 ? 0u : ~0u << (pass == 1 ? 21 : 10);
    for (int b = tid; b < 2048; b += LK_THREADS) hist[b] = 0;
    __syncthreads();
    for (int j = tid; j < n; j += LK_THREADS) {
      const uint32_t key = lk_key(lk_est(s, sqn, qn, j));
      if ((key & hi_mask) == prefix) atomicAdd(&hist[(key >> shift) & bin_mask], 1);
    }
    __syncthreads();
    int h[4], local = 0, before;
#pragma unroll
    for (int u = 0; u < 4; ++u) { h[u] = hist[tid * 4 + u]; local += h[u]; }
    Scan(scan_tmp).ExclusiveSum(local, before);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (before < rem && rem <= before + h[u]) { s_bin = (uint32_t)(tid * 4 + u); s_rem = rem - before; }
      before += h[u];
    }
    __syncthreads();
    prefix |= s_bin << shift;
    rem = s_rem;
    __syncthreads();
  }
  const double qd = (double)qn, rmax = (double)max_sqn[0];
  const double err = err_rel * (qd + rmax + 2.0 * sqrt(qd * rmax));
  const double base = (double)lk_unkey(prefix) + err;
  const double thr = base + fabs(base) * 1e-12 + err;
  int c = 0;
  for (int j = tid; j < n; j += LK_THREADS) c += (double)lk_est(s, sqn, qn, j) <= thr ? 1 : 0;
  int unused, total;
  Scan(scan_tmp).ExclusiveSum(c, unused, total);
  if (tid == 0) { thr_out[row] = thr; count_out[row] = total; }
}

// one CTA per query row of a chunk [row0, row0 + gridDim.x) of the batch: the references with d̂² ≤ thr_q in ascending index
// order, then their fp64 distances.  offs: the batch's exclusive scan of the counts; seg: the chunk's segment offsets.
__global__ void __launch_bounds__(LK_THREADS)
knn_lk_collect_kernel(const float* __restrict__ S, int64_t lds, const float* __restrict__ sqn, const float* __restrict__ X, int64_t ldx,
                      int32_t n, int32_t d, int32_t q0, int32_t row0, const double* __restrict__ thr, const int32_t* __restrict__ offs,
                      int32_t* __restrict__ seg, int32_t* __restrict__ cand, double* __restrict__ cdist) {
  constexpr int ITEMS = 4;
  using Scan = cub::BlockScan<int, LK_THREADS>;
  __shared__ typename Scan::TempStorage scan_tmp;
  const int tid = threadIdx.x;
  const int64_t row = row0 + blockIdx.x;
  const int32_t base = offs[row0], off = offs[row] - base, end = offs[row + 1] - base;
  if (tid == 0) {
    seg[blockIdx.x] = off;
    if (blockIdx.x == gridDim.x - 1) seg[gridDim.x] = end;
  }
  const float* s = S + row * lds;
  const float qn = sqn[q0 + row];
  const double t = thr[row];
  int32_t w = off;
  for (int j0 = 0; j0 < n; j0 += LK_THREADS * ITEMS) {
    int flag[ITEMS], pos[ITEMS], total;
#pragma unroll
    for (int u = 0; u < ITEMS; ++u) {
      const int j = j0 + tid * ITEMS + u;
      flag[u] = (j < n && (double)lk_est(s, sqn, qn, j) <= t) ? 1 : 0;
    }
    Scan(scan_tmp).ExclusiveSum(flag, pos, total);
#pragma unroll
    for (int u = 0; u < ITEMS; ++u)
      if (flag[u]) cand[w + pos[u]] = j0 + tid * ITEMS + u;
    w += total;
    __syncthreads();
  }
  const float* xq = X + (q0 + row) * ldx;
  for (int32_t c = off + tid; c < end; c += LK_THREADS) cdist[c] = sqrt(exact_sqdist(xq, X + (int64_t)cand[c] * ldx, d));
}

// ranks r0 … r0+k−1 of each sorted segment of the chunk → rows out_row0 … of the result
__global__ void __launch_bounds__(256)
knn_lk_emit_kernel(const int32_t* __restrict__ seg, const int32_t* __restrict__ sidx, const double* __restrict__ sdist, int32_t rows,
                   int32_t k, int32_t r0, int64_t out_row0, int32_t* __restrict__ idx_out, double* __restrict__ dist_out) {
  const int64_t total = (int64_t)rows * k;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / k;
    const int p = (int)(t % k);
    const int32_t src = seg[i] + r0 + p;
    idx_out[(out_row0 + i) * k + p] = sidx[src];
    if (dist_out) dist_out[(out_row0 + i) * k + p] = sdist[src];
  }
}

// Sizes of the large-k path.  K is sized as k + 1 whatever include_rank0 is, so that the workspace query needs no r0.
struct LkPlan {
  int32_t dp, bq;
  int64_t lds, cap;               // S pitch; candidates one sort holds (≥ n, so that any one query fits)
  size_t gemm_ws, scan_ws, sort_ws;
  size_t off_xp, off_s, off_gemm, off_thr, off_counts, off_offs, off_seg, off_scan, off_cand, off_cdist, off_sidx, off_sdist,
      off_sort, bytes;
};

static size_t lk_sort_bytes(int64_t items, int32_t segments) {
  size_t b = 0;
  cub::DeviceSegmentedSort::StableSortPairs(nullptr, b, (const double*)nullptr, (double*)nullptr, (const int32_t*)nullptr,
                                            (int32_t*)nullptr, (int)items, segments, (const int32_t*)nullptr,
                                            (const int32_t*)nullptr);
  return b;
}

static LkPlan lk_plan(int32_t n, int32_t d, int32_t k, int32_t n_q) {
  LkPlan p;
  p.dp = (d + 3) / 4 * 4;
  p.lds = ((int64_t)n + 3) / 4 * 4;
  const int64_t bq = (int64_t)(LK_BLOCK_BYTES / (4 * (size_t)p.lds));
  p.bq = (int32_t)(bq < 1 ? 1 : (bq > n_q ? n_q : bq));
  const int64_t want = 4ll * p.bq * (k + 1), all = (int64_t)p.bq * n;
  p.cap = want < all ? want : all;
  if (p.cap > (1ll << 30)) p.cap = 1ll << 30;
  if (p.cap < n) p.cap = n;
  const int32_t last = n_q % p.bq;
  p.gemm_ws = b2_gemm_workspace_bytes(p.bq, n, p.dp, 0, 1, B2_PREC_TF32X3);
  if (last) {
    const size_t g = b2_gemm_workspace_bytes(last, n, p.dp, 0, 1, B2_PREC_TF32X3);
    if (g > p.gemm_ws) p.gemm_ws = g;
  }
  p.scan_ws = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, p.scan_ws, (const int32_t*)nullptr, (int32_t*)nullptr, p.bq + 1);
  p.sort_ws = lk_sort_bytes(p.cap, p.bq);
  size_t o = align_up((size_t)n * 4, 256) + 256;   // |x|² and max |x|², laid out as in the SIMT path
  auto take = [&](size_t bytes) { const size_t at = o; o += align_up(bytes, 256); return at; };
  p.off_xp = take((size_t)n * p.dp * 4);
  p.off_s = take((size_t)p.bq * p.lds * 4);
  p.off_gemm = take(p.gemm_ws);
  p.off_thr = take((size_t)p.bq * 8);
  p.off_counts = take(((size_t)p.bq + 1) * 4);
  p.off_offs = take(((size_t)p.bq + 1) * 4);
  p.off_seg = take(((size_t)p.bq + 1) * 4);
  p.off_scan = take(p.scan_ws);
  p.off_cand = take((size_t)p.cap * 4);
  p.off_cdist = take((size_t)p.cap * 8);
  p.off_sidx = take((size_t)p.cap * 4);
  p.off_sdist = take((size_t)p.cap * 8);
  p.off_sort = take(p.sort_ws);
  p.bytes = o;
  return p;
}

static int knn_large_k(const float* X, int64_t ldx, int32_t n, int32_t d, int32_t k, int32_t q_begin, int32_t n_q, int r0,
                       int32_t* idx_out, double* dist_out, char* ws, cudaStream_t st) {
  const LkPlan p = lk_plan(n, d, k, n_q);
  float* sqn = reinterpret_cast<float*>(ws);
  float* max_sqn = reinterpret_cast<float*>(ws + align_up((size_t)n * 4, 256));
  float* Xp = reinterpret_cast<float*>(ws + p.off_xp);
  float* S = reinterpret_cast<float*>(ws + p.off_s);
  double* thr = reinterpret_cast<double*>(ws + p.off_thr);
  int32_t* counts = reinterpret_cast<int32_t*>(ws + p.off_counts);
  int32_t* offs = reinterpret_cast<int32_t*>(ws + p.off_offs);
  int32_t* seg = reinterpret_cast<int32_t*>(ws + p.off_seg);
  int32_t* cand = reinterpret_cast<int32_t*>(ws + p.off_cand);
  double* cdist = reinterpret_cast<double*>(ws + p.off_cdist);
  int32_t* sidx = reinterpret_cast<int32_t*>(ws + p.off_sidx);
  double* sdist = reinterpret_cast<double*>(ws + p.off_sdist);
  const int K = k + r0;
  const double err_rel = lk_err_rel(d, p.dp);

  B2_CHECK_CUDA(cudaMemsetAsync(max_sqn, 0, 4, st));
  row_sqnorm_kernel<<<grid_blocks(n, 8), 256, 0, st>>>(X, ldx, n, d, sqn, max_sqn);
  B2_CHECK_LAUNCH("row_sqnorm_kernel");
  knn_lk_pad_kernel<<<grid_blocks((int64_t)n * p.dp, 1024), 256, 0, st>>>(X, ldx, n, d, p.dp, Xp);
  B2_CHECK_LAUNCH("knn_lk_pad_kernel");

  std::vector<int32_t> h_offs((size_t)p.bq + 1);
  for (int32_t b0 = 0; b0 < n_q; b0 += p.bq) {
    const int32_t m = n_q - b0 < p.bq ? n_q - b0 : p.bq;
    const int32_t q0 = q_begin + b0;
    const int rc = b2_gemm_f32(Xp + (int64_t)q0 * p.dp, p.dp, 0, Xp, p.dp, 1, S, p.lds, m, n, p.dp, nullptr, B2_ACT_NONE, nullptr, 0,
                               0.f, B2_PREC_TF32X3, p.gemm_ws ? ws + p.off_gemm : nullptr, p.gemm_ws, st);
    if (rc != B2_OK) return rc;
    knn_lk_select_kernel<<<m, LK_THREADS, 0, st>>>(S, p.lds, sqn, max_sqn, n, q0, K, err_rel, thr, counts);
    B2_CHECK_LAUNCH("knn_lk_select_kernel");
    B2_CHECK_CUDA(cudaMemsetAsync(counts + m, 0, 4, st));
    size_t scan_ws = p.scan_ws;
    B2_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(ws + p.off_scan, scan_ws, counts, offs, m + 1, st));
    B2_CHECK_CUDA(cudaMemcpyAsync(h_offs.data(), offs, ((size_t)m + 1) * 4, cudaMemcpyDeviceToHost, st));
    B2_CHECK_CUDA(cudaStreamSynchronize(st));
    // rows [a, b) whose candidates fit in one sort; one row always fits (at most n ≤ cap candidates)
    for (int32_t a = 0; a < m;) {
      int32_t b = a + 1;
      while (b < m && (int64_t)h_offs[b + 1] - h_offs[a] <= p.cap) ++b;
      const int32_t rows = b - a, items = h_offs[b] - h_offs[a];
      knn_lk_collect_kernel<<<rows, LK_THREADS, 0, st>>>(S, p.lds, sqn, X, ldx, n, d, q0, a, thr, offs, seg, cand, cdist);
      B2_CHECK_LAUNCH("knn_lk_collect_kernel");
      size_t sort_ws = lk_sort_bytes(items, rows);
      B2_REQUIRE(sort_ws <= p.sort_ws, "b2_knn_l2_f32: segmented sort needs %zu bytes, %zu reserved", sort_ws, p.sort_ws);
      B2_CHECK_CUDA(cub::DeviceSegmentedSort::StableSortPairs(ws + p.off_sort, sort_ws, cdist, sdist, cand, sidx, items, rows, seg,
                                                              seg + 1, st));
      knn_lk_emit_kernel<<<grid_blocks((int64_t)rows * k, 256), 256, 0, st>>>(seg, sidx, sdist, rows, k, r0, (int64_t)b0 + a, idx_out,
                                                                             dist_out);
      B2_CHECK_LAUNCH("knn_lk_emit_kernel");
      a = b;
    }
  }
  return B2_OK;
}

static size_t cand_smem_bytes(int M) {
  return sizeof(float) * (KK * (KQ + 4 + KR + 4) + KQ * (KR + 1)) + (sizeof(float) + sizeof(int32_t)) * KQ * M;
}

// `need` = number of sorted ranks that must be recovered (k, +1 when rank 0 is dropped); 8 spare candidates
static int choose_M(int need) { return (need + 8 <= 32) ? 32 : 64; }

namespace ktc {   // knn_tc.cu: tensor-core candidate filter
size_t workspace_bytes(int32_t n, int32_t d, int32_t n_q);
bool eligible(int32_t n, int32_t d, int32_t n_q, int M);
float tc_err_rel(int32_t d);
int launch(const float* X, int64_t ldx, const float* sqn, int32_t n, int32_t d, int32_t q_begin, int32_t n_q, int32_t* cand_idx,
           float* cand_thr, void* ws, size_t ws_bytes, cudaStream_t st);
}  // namespace ktc

}  // namespace b2

using namespace b2;

// k + 8 <= KMAXC: the candidate-list path; k + 9 > KMAXC: the large-k path (both at k = KMAXC - 8, where include_rank0 decides)
extern "C" size_t b2_knn_workspace_bytes(int32_t n, int32_t d, int32_t k, int32_t n_queries) {
  size_t bytes = 0;
  if (k + 8 <= KMAXC) {
    const int M = choose_M(k + 1);
    bytes = align_up((size_t)n * 4, 256) + align_up((size_t)n_queries * M * 4, 256) + 2 * align_up((size_t)n_queries * 4, 256) +
            1024 + (ktc::eligible(n, d, n_queries, M) ? ktc::workspace_bytes(n, d, n_queries) : 0);
  }
  if (k + 9 > KMAXC && n > 0 && d > 0 && n_queries > 0) {
    const size_t large = lk_plan(n, d, k, n_queries).bytes;
    if (large > bytes) bytes = large;
  }
  return bytes;
}

extern "C" int b2_knn_l2_f32(const float* X, int64_t ldx, int32_t n, int32_t d, int32_t k, int32_t q_begin,
                             int32_t q_end, int include_rank0, int32_t* idx_out, double* dist_out, void* workspace,
                             size_t workspace_bytes, void* stream) {
  B2_REQUIRE(X && idx_out, "b2_knn_l2_f32: null pointer");
  B2_REQUIRE(n > 0 && d > 0 && ldx >= d, "b2_knn_l2_f32: bad shape");
  B2_REQUIRE(0 <= q_begin && q_begin <= q_end && q_end <= n, "b2_knn_l2_f32: bad query range");
  const int r0 = include_rank0 ? 0 : 1;
  B2_REQUIRE(k >= 1 && k + r0 <= n, "b2_knn_l2_f32: k=%d needs at least k+%d points, have %d", k, r0, n);
  const int32_t n_q = q_end - q_begin;
  if (n_q == 0) return B2_OK;
  B2_REQUIRE(workspace && workspace_bytes >= b2_knn_workspace_bytes(n, d, k, n_q), "b2_knn_l2_f32: workspace too small");
  cudaStream_t st = as_stream(stream);
  if (k + r0 + 8 > KMAXC) return knn_large_k(X, ldx, n, d, k, q_begin, n_q, r0, idx_out, dist_out, reinterpret_cast<char*>(workspace), st);
  const int M = choose_M(k + r0);

  char* ws = reinterpret_cast<char*>(workspace);
  size_t off = 0;
  float* sqn = reinterpret_cast<float*>(ws + off); off += align_up((size_t)n * 4, 256);
  int32_t* cand = reinterpret_cast<int32_t*>(ws + off); off += align_up((size_t)n_q * M * 4, 256);
  float* thr = reinterpret_cast<float*>(ws + off); off += align_up((size_t)n_q * 4, 256);
  int32_t* fail_list = reinterpret_cast<int32_t*>(ws + off); off += align_up((size_t)n_q * 4, 256);
  float* max_sqn = reinterpret_cast<float*>(ws + off);
  int32_t* fail_count = reinterpret_cast<int32_t*>(ws + off + 16);
  B2_CHECK_CUDA(cudaMemsetAsync(ws + off, 0, 64, st));

  row_sqnorm_kernel<<<grid_blocks(n, 8), 256, 0, st>>>(X, ldx, n, d, sqn, max_sqn);
  B2_CHECK_LAUNCH("row_sqnorm_kernel");
  float err_rel = 1.1920928955078125e-07f * (float)(d + 8);      // fp32 SIMT filter
  bool tc_done = false;
  if (ktc::eligible(n, d, n_q, M)) {
    const int rc = ktc::launch(X, ldx, sqn, n, d, q_begin, n_q, cand, thr, ws + off + 1024, workspace_bytes - off - 1024, st);
    if (rc == B2_OK) { tc_done = true; err_rel = ktc::tc_err_rel(d); }
    else if (rc != B2_ERR_UNSUPPORTED) return rc;
  }
  const unsigned grid = (unsigned)ceil_div(n_q, KQ);
  if (!tc_done) {
    auto kernel = M == 32 ? knn_candidates_kernel<32> : knn_candidates_kernel<64>;
    const size_t smem = cand_smem_bytes(M);
    const int rc = allow_dynamic_smem((const void*)kernel, smem);
    if (rc != B2_OK) return rc;
    kernel<<<grid, KTHREADS, smem, st>>>(X, ldx, sqn, n, d, q_begin, n_q, cand, thr);
    B2_CHECK_LAUNCH("knn_candidates_kernel");
  }
  const unsigned refine_grid = grid_blocks(n_q, 8);
  if (M == 32)
    knn_refine_kernel<32><<<refine_grid, 256, 0, st>>>(X, ldx, sqn, max_sqn, n, d, k, q_begin, n_q, r0, cand, thr, err_rel, idx_out,
                                                       dist_out, fail_list, fail_count);
  else
    knn_refine_kernel<64><<<refine_grid, 256, 0, st>>>(X, ldx, sqn, max_sqn, n, d, k, q_begin, n_q, r0, cand, thr, err_rel, idx_out,
                                                       dist_out, fail_list, fail_count);
  B2_CHECK_LAUNCH("knn_refine_kernel");
  knn_fallback_kernel<<<(unsigned)sm_count(), 256, 0, st>>>(X, ldx, n, d, k, q_begin, r0, fail_list, fail_count, idx_out,
                                                            dist_out);
  B2_CHECK_LAUNCH("knn_fallback_kernel");
  return B2_OK;
}

extern "C" int b2_pairwise_l2_dense_f32(const float* X, int64_t ldx, int32_t n, int32_t d, float* D, int64_t ldd,
                                        void* stream) {
  B2_REQUIRE(X && D && n >= 0 && d > 0 && ldx >= d && ldd >= n, "b2_pairwise_l2_dense_f32: bad arguments");
  if (n == 0) return B2_OK;
  pairwise_dense_kernel<<<grid_blocks((int64_t)n * n, 256, 32), 256, 0, as_stream(stream)>>>(X, ldx, n, d, D, ldd);
  B2_CHECK_LAUNCH("pairwise_dense_kernel");
  return B2_OK;
}
