// graph-sc (GraphSC) on mini-batch blocks of the cell–gene graph (graphsc.py:179-216, :355-484).
//
// A block is a list of destination node ids plus the parent graph's destination-indexed CSR (row v = sources of v's in-edges,
// GraphLite.csr_by_destination()).  dgl's MultiLayerFullNeighborSampler keeps every in-edge of a destination, so a block's
// in-degree is the full row length; its out-degree is not: source u counts only its edges INTO the destination list.  No
// relabelled block CSR is built: the degree histogram and the aggregate both walk the parent rows of the listed destinations.
//
// Dropout masks are keyed by GLOBAL node id (row) and feature (column), so a gene several batches touch draws an independent mask
// in each (the key differs per step).  The decoder's mask is keyed by the row within the batch.
#include "common.cuh"

namespace b2 {

// ---- block out-degrees ---------------------------------------------------------------------------------------------------------
// outdeg[u] += 1 for every edge u→v with v in dst (entries < 0 are padding).  With src_list, the first edge that reaches u also
// appends u to src_list (at slot k = (*n_src)++) and sets src_pos[u] = k: the block's source set, which is the previous layer's
// destination list.
__global__ void __launch_bounds__(256)
block_degrees_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx, const int32_t* __restrict__ dst,
                     int32_t n_dst, int32_t* outdeg, int32_t* src_list, int32_t* src_pos, int32_t* n_src, int32_t cap) {
  const int warp = (int)((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (warp >= n_dst) return;
  const int v = dst[warp];
  if (v < 0) return;
  for (int e = rowptr[v] + lane; e < rowptr[v + 1]; e += 32) {
    const int u = colidx[e];
    const int old = atomicAdd(&outdeg[u], 1);
    if (src_list && old == 0) {
      const int k = atomicAdd(n_src, 1);
      if (k < cap) { src_list[k] = u; src_pos[u] = k; }
    }
  }
}

// ---- block aggregate -----------------------------------------------------------------------------------------------------------
// Forward: out[i, f] = s_v · Σ_{e: u→v} w_e · c_u · keep(u, f) · scale · x[row(u), f],   v = dst[i]
// Transposed: dx[row(u), f] += s_v · w_e · c_u · keep(u, f) · scale · dout[i, f]  (dx zeroed by the host routine)
// c_u = clamp(outdeg[u], 1)^-1/2, s_v = clamp(indeg_v, 1)^-1/2 (· 1/clamp(indeg_v, 1) for agg = mean), row(u) = x_pos[u] or u.
// One warp per destination and 128-feature slice (grid.y), four features per lane.
struct AggArgs {
  const int32_t *rowptr, *colidx, *dst, *outdeg, *x_pos;
  const float* w;
  const float* in;   // x (forward) or dout (transposed)
  int64_t ldin;
  float* out;        // out (forward) or dx (transposed)
  int64_t ldout;
  int32_t n_dst, F, mean;
  float p, scale;
  uint32_t seed, key;
};

template <bool TRANSPOSED>
__global__ void __launch_bounds__(256) block_aggregate_kernel(AggArgs a) {
  const int i = (int)((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (i >= a.n_dst) return;
  const int f0 = blockIdx.y * 128 + lane;
  const int v = a.dst[i];
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  if (v < 0) {                      // padding slot: a zero row (forward); nothing to scatter (transposed)
    if (!TRANSPOSED)
      for (int k = 0; k < 4; ++k)
        if (f0 + 32 * k < a.F) a.out[(int64_t)i * a.ldout + f0 + 32 * k] = 0.f;
    return;
  }
  const int e0 = a.rowptr[v], e1 = a.rowptr[v + 1];
  const float indeg = fmaxf((float)(e1 - e0), 1.f);
  const float s = rsqrtf(indeg) * (a.mean ? 1.f / indeg : 1.f) * a.scale;
  float g[4];
  if (TRANSPOSED)
    for (int k = 0; k < 4; ++k) g[k] = f0 + 32 * k < a.F ? a.in[(int64_t)i * a.ldin + f0 + 32 * k] * s : 0.f;
  for (int e = e0; e < e1; ++e) {
    const int u = a.colidx[e];
    const float c = (a.w ? a.w[e] : 1.f) * rsqrtf(fmaxf((float)a.outdeg[u], 1.f));
    const int64_t r = a.x_pos ? a.x_pos[u] : u;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int f = f0 + 32 * k;
      if (f >= a.F) break;
      if (a.p > 0.f && !dropout_keep(a.seed, a.key, (uint32_t)u, (uint32_t)f, a.p)) continue;
      if (TRANSPOSED) atomicAdd(&a.out[r * a.ldout + f], c * g[k]);
      else acc[k] = fmaf(c, a.in[r * a.ldin + f], acc[k]);
    }
  }
  if (!TRANSPOSED)
    for (int k = 0; k < 4; ++k)
      if (f0 + 32 * k < a.F) a.out[(int64_t)i * a.ldout + f0 + 32 * k] = acc[k] * s;
}

// ---- fused mini-batch decoder --------------------------------------------------------------------------------------------------
// z̃ = keep ⊙ z · scale (p = 0.1 in graph-sc), S = z̃z̃ᵀ, y = I, pw = B − 1, norm = B / (2(B − 1)) (B = 1: pw = 0, norm = 1):
//   loss = norm/B² · Σ_ij [pw·y·softplus(−S) + (1−y)·softplus(S)],  C = ∂loss/∂S,  dz = keep ⊙ 2·C·z̃ · scale.
// Each CTA owns DEC_TI rows and sweeps the B columns in tiles of DEC_TJ: the S tile in DEC_KC-wide k-chunks from shared memory,
// then its C tile, then dz̃_I += C_tile · z̃_J into a [DEC_TI, d] shared accumulator.
constexpr int DEC_TI = 8, DEC_TJ = 32, DEC_KC = 32, DEC_THREADS = 256;

__device__ __forceinline__ float dropped(const float* z, int64_t ldz, int B, int r, int f, float p, float scale, uint32_t seed,
                                         uint32_t key) {
  if (r >= B) return 0.f;
  if (p > 0.f && !dropout_keep(seed, key, (uint32_t)r, (uint32_t)f, p)) return 0.f;
  return z[(int64_t)r * ldz + f] * scale;
}
__device__ __forceinline__ float softplus_f(float x) { return fmaxf(x, 0.f) + log1pf(__expf(-fabsf(x))); }
__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + __expf(-x)); }

__global__ void __launch_bounds__(DEC_THREADS, 1)
batch_decoder_kernel(const float* __restrict__ z, int64_t ldz, int B, int d, float p, float scale, uint32_t seed, uint32_t key,
                     float pw, float coef, float* __restrict__ dz, int64_t lddz, float* loss_out) {
  extern __shared__ float dzacc[];                       // [DEC_TI][d]
  __shared__ float zi[DEC_TI][DEC_KC + 1], zj[DEC_TJ][DEC_KC + 1], cs[DEC_TI][DEC_TJ], red[DEC_THREADS / 32];
  const int t = threadIdx.x, i0 = blockIdx.x * DEC_TI;
  const int ti = t / DEC_TJ, tj = t % DEC_TJ;
  for (int k = t; k < DEC_TI * d; k += DEC_THREADS) dzacc[k] = 0.f;
  float loss = 0.f;
  for (int j0 = 0; j0 < B; j0 += DEC_TJ) {
    float s = 0.f;
    for (int k0 = 0; k0 < d; k0 += DEC_KC) {
      __syncthreads();
      {
        const int f = k0 + tj;
        zi[ti][tj] = f < d ? dropped(z, ldz, B, i0 + ti, f, p, scale, seed, key) : 0.f;
      }
      for (int q = t; q < DEC_TJ * DEC_KC; q += DEC_THREADS) {
        const int r = q / DEC_KC, f = k0 + q % DEC_KC;
        zj[r][q % DEC_KC] = f < d ? dropped(z, ldz, B, j0 + r, f, p, scale, seed, key) : 0.f;
      }
      __syncthreads();
#pragma unroll 8
      for (int k = 0; k < DEC_KC; ++k) s = fmaf(zi[ti][k], zj[tj][k], s);
    }
    const int i = i0 + ti, j = j0 + tj;
    float c = 0.f;
    if (i < B && j < B) {
      if (i == j) { loss += coef * pw * softplus_f(-s); c = -coef * pw * sigmoid_f(-s); }
      else { loss += coef * softplus_f(s); c = coef * sigmoid_f(s); }
    }
    cs[ti][tj] = c;
    __syncthreads();
    for (int f = t; f < d; f += DEC_THREADS) {
      float acc[DEC_TI];
#pragma unroll
      for (int r = 0; r < DEC_TI; ++r) acc[r] = 0.f;
      for (int jj = 0; jj < DEC_TJ && j0 + jj < B; ++jj) {
        const float zv = dropped(z, ldz, B, j0 + jj, f, p, scale, seed, key);
#pragma unroll
        for (int r = 0; r < DEC_TI; ++r) acc[r] = fmaf(cs[r][jj], zv, acc[r]);
      }
#pragma unroll
      for (int r = 0; r < DEC_TI; ++r) dzacc[r * d + f] += acc[r];
    }
  }
  __syncthreads();
  for (int k = t; k < DEC_TI * d; k += DEC_THREADS) {
    const int r = i0 + k / d, f = k % d;
    if (r < B) dz[(int64_t)r * lddz + f] = (p > 0.f && !dropout_keep(seed, key, (uint32_t)r, (uint32_t)f, p)) ? 0.f : 2.f * dzacc[k] * scale;
  }
  loss = warp_sum(loss);
  if ((t & 31) == 0) red[t >> 5] = loss;
  __syncthreads();
  if (t == 0) {
    float tot = 0.f;
    for (int w = 0; w < DEC_THREADS / 32; ++w) tot += red[w];
    atomicAdd(loss_out, tot);
  }
}

// ---- scatter -------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
scatter_rows_kernel(const float* __restrict__ x, int64_t ldx, int32_t rows, int32_t cols, const int32_t* __restrict__ idx,
                    int32_t offset, float* out, int64_t ldo) {
  const int64_t total = (int64_t)rows * cols;
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = q / cols;
    const int c = (int)(q % cols);
    out[(int64_t)(idx[r] - offset) * ldo + c] = x[r * ldx + c];
  }
}

}  // namespace b2

using namespace b2;

extern "C" int b2_graphsc_block_degrees(const int32_t* rowptr, const int32_t* colidx, int32_t n_nodes, const int32_t* dst,
                                        int32_t n_dst, int32_t* outdeg, int32_t* src_list, int32_t* src_pos, int32_t* n_src,
                                        int32_t src_cap, void* stream) {
  B2_REQUIRE(n_nodes > 0 && n_dst >= 0, "b2_graphsc_block_degrees: bad sizes (n_nodes %d, n_dst %d)", n_nodes, n_dst);
  B2_REQUIRE(rowptr && colidx && outdeg && (dst || n_dst == 0), "b2_graphsc_block_degrees: null pointer");
  const bool list = src_list || src_pos || n_src;
  B2_REQUIRE(!list || (src_list && src_pos && n_src && src_cap > 0),
             "b2_graphsc_block_degrees: src_list, src_pos and n_src go together, with src_cap > 0");
  cudaStream_t st = as_stream(stream);
  B2_CHECK_CUDA(cudaMemsetAsync(outdeg, 0, sizeof(int32_t) * (size_t)n_nodes, st));
  if (list) {
    B2_CHECK_CUDA(cudaMemsetAsync(src_list, 0xFF, sizeof(int32_t) * (size_t)src_cap, st));   // -1: padding slots
    B2_CHECK_CUDA(cudaMemsetAsync(n_src, 0, sizeof(int32_t), st));
  }
  if (n_dst == 0) return B2_OK;
  block_degrees_kernel<<<ceil_div<int64_t>((int64_t)n_dst * 32, 256), 256, 0, st>>>(rowptr, colidx, dst, n_dst, outdeg, src_list,
                                                                                     src_pos, n_src, src_cap);
  B2_CHECK_LAUNCH("block_degrees_kernel");
  return B2_OK;
}

extern "C" int b2_graphsc_block_aggregate_f32(const int32_t* rowptr, const int32_t* colidx, const float* weights,
                                              const int32_t* dst, int32_t n_dst, const int32_t* outdeg, const float* in,
                                              int64_t ldin, const int32_t* x_pos, int32_t F, int agg_mean, float p, uint32_t seed,
                                              uint32_t key, int transposed, float* out, int64_t ldout, int64_t out_rows,
                                              void* stream) {
  B2_REQUIRE(n_dst >= 0 && F > 0 && ldin >= F && ldout >= F && out_rows >= 0,
             "b2_graphsc_block_aggregate_f32: bad shape (n_dst %d, F %d, ldin %lld, ldout %lld)", n_dst, F, (long long)ldin,
             (long long)ldout);
  B2_REQUIRE(rowptr && colidx && outdeg && in && out && (dst || n_dst == 0), "b2_graphsc_block_aggregate_f32: null pointer");
  B2_REQUIRE(agg_mean == 0 || agg_mean == 1, "b2_graphsc_block_aggregate_f32: agg_mean must be 0 (sum) or 1 (mean)");
  B2_REQUIRE(p >= 0.f && p < 1.f, "b2_graphsc_block_aggregate_f32: p must be in [0, 1)");
  B2_REQUIRE(transposed == 0 || transposed == 1, "b2_graphsc_block_aggregate_f32: transposed must be 0 or 1");
  B2_REQUIRE(!transposed || out_rows > 0, "b2_graphsc_block_aggregate_f32: the transposed form needs out_rows > 0");
  cudaStream_t st = as_stream(stream);
  // the [out_rows, F] block only: the columns past F of a row-padded `out` belong to the caller
  if (transposed)
    B2_CHECK_CUDA(cudaMemset2DAsync(out, sizeof(float) * (size_t)ldout, 0, sizeof(float) * (size_t)F, (size_t)out_rows, st));
  if (n_dst == 0) return B2_OK;
  AggArgs a{rowptr, colidx, dst, outdeg, x_pos, weights, in, ldin, out, ldout, n_dst, F, agg_mean, p, 1.f / (1.f - p), seed, key};
  const dim3 grid((unsigned)ceil_div<int64_t>((int64_t)n_dst * 32, 256), (unsigned)ceil_div(F, 128));
  if (transposed) block_aggregate_kernel<true><<<grid, 256, 0, st>>>(a);
  else block_aggregate_kernel<false><<<grid, 256, 0, st>>>(a);
  B2_CHECK_LAUNCH("block_aggregate_kernel");
  return B2_OK;
}

extern "C" int b2_graphsc_batch_decoder_f32(const float* z, int64_t ldz, int32_t B, int32_t d, float p, uint32_t seed, uint32_t key,
                                            float* dz, int64_t lddz, float* loss_out, void* stream) {
  B2_REQUIRE(B >= 1, "b2_graphsc_batch_decoder_f32: batch size must be >= 1 (got %d)", B);
  B2_REQUIRE(d >= 1 && d <= 1024, "b2_graphsc_batch_decoder_f32: embedding width must be in [1, 1024] (got %d)", d);
  B2_REQUIRE(ldz >= d && lddz >= d, "b2_graphsc_batch_decoder_f32: leading dimension below d");
  B2_REQUIRE(p >= 0.f && p < 1.f, "b2_graphsc_batch_decoder_f32: p must be in [0, 1)");
  B2_REQUIRE(z && dz && loss_out, "b2_graphsc_batch_decoder_f32: null pointer");
  const float pw = B > 1 ? (float)(B - 1) : 0.f;                          // (B² − ΣI) / ΣI
  const double norm = B > 1 ? (double)B / (2.0 * (B - 1)) : 1.0;          // B² / (2(B² − B)); factor == 0 ⇒ 1
  const float coef = (float)(norm / ((double)B * B));                      // BCE mean over B²
  cudaStream_t st = as_stream(stream);
  B2_CHECK_CUDA(cudaMemsetAsync(loss_out, 0, sizeof(float), st));
  batch_decoder_kernel<<<ceil_div(B, DEC_TI), DEC_THREADS, sizeof(float) * DEC_TI * d, st>>>(z, ldz, B, d, p, 1.f / (1.f - p), seed,
                                                                                            key, pw, coef, dz, lddz, loss_out);
  B2_CHECK_LAUNCH("batch_decoder_kernel");
  return B2_OK;
}

extern "C" int b2_graphsc_scatter_rows_f32(const float* x, int64_t ldx, int32_t rows, int32_t cols, const int32_t* idx,
                                           int32_t offset, float* out, int64_t ldo, void* stream) {
  B2_REQUIRE(rows >= 0 && cols >= 0 && ldx >= cols && ldo >= cols, "b2_graphsc_scatter_rows_f32: bad shape");
  if (rows == 0 || cols == 0) return B2_OK;
  B2_REQUIRE(x && idx && out, "b2_graphsc_scatter_rows_f32: null pointer");
  scatter_rows_kernel<<<grid_blocks((int64_t)rows * cols, 256), 256, 0, as_stream(stream)>>>(x, ldx, rows, cols, idx, offset, out, ldo);
  B2_CHECK_LAUNCH("scatter_rows_kernel");
  return B2_OK;
}
