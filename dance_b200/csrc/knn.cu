// Exact euclidean k-nearest-neighbour search: filter (fp32 tile distances, per-query
// candidate lists) → refine (fp64 re-rank exactly like the reference) → verify
// (error-bound proof that no non-candidate can enter the top-k) → rare fallback
// (fp64 brute force for unproven queries).
//
// Reference being replaced: calculateKNNgraphDistanceMatrixStatsSingleThread
// (scgnn2.py:675-689): per row scipy `cdist(..., "euclidean")` in fp64 on the fp32
// features, `argsort`, take sorted ranks 1..k.  Also the kNN inside NeighborGraph
// (neighbor_graph.py:50-57) and StagateGraph (spatial_graph.py:147-149).
#include "common.cuh"
#include "spatial_pair.cuh"

#include <math_constants.h>

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

extern "C" size_t b2_knn_workspace_bytes(int32_t n, int32_t d, int32_t k, int32_t n_queries) {
  const int M = choose_M(k + 1);
  return align_up((size_t)n * 4, 256) + align_up((size_t)n_queries * M * 4, 256) +
         2 * align_up((size_t)n_queries * 4, 256) + 1024 + (ktc::eligible(n, d, n_queries, M) ? ktc::workspace_bytes(n, d, n_queries) : 0);
}

extern "C" int b2_knn_l2_f32(const float* X, int64_t ldx, int32_t n, int32_t d, int32_t k, int32_t q_begin,
                             int32_t q_end, int include_rank0, int32_t* idx_out, double* dist_out, void* workspace,
                             size_t workspace_bytes, void* stream) {
  B2_REQUIRE(X && idx_out, "b2_knn_l2_f32: null pointer");
  B2_REQUIRE(n > 0 && d > 0 && ldx >= d, "b2_knn_l2_f32: bad shape");
  B2_REQUIRE(0 <= q_begin && q_begin <= q_end && q_end <= n, "b2_knn_l2_f32: bad query range");
  const int r0 = include_rank0 ? 0 : 1;
  B2_REQUIRE(k >= 1 && k + r0 <= n, "b2_knn_l2_f32: k=%d needs at least k+%d points, have %d", k, r0, n);
  B2_REQUIRE(k + r0 + 8 <= KMAXC, "b2_knn_l2_f32: k=%d too large (max %d)", k, KMAXC - 8 - r0);
  const int32_t n_q = q_end - q_begin;
  if (n_q == 0) return B2_OK;
  B2_REQUIRE(workspace && workspace_bytes >= b2_knn_workspace_bytes(n, d, k, n_q), "b2_knn_l2_f32: workspace too small");
  cudaStream_t st = as_stream(stream);
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
