// Pre-processing operators immediately upstream of scGNN / GraphSCI (SURVEY §8f row 1): the reductions behind
// FilterGenesScanpy / FilterCellsScanpy / FilterGenesTopK (reference dance/transforms/filter.py:56-158, 470-520, 592-664) and the
// cell-wise train / valid / test masking of CellwiseMaskData (dance/transforms/mask.py:80-291).  All of it is one or two passes
// over the cell × gene matrix: HBM-bound, coalesced row-major reads, fp64 accumulation.
#include "common.cuh"

namespace b2 {
namespace {

// ---- per-gene statistics: Σx, Σx², #(x > 0) over the cells ------------------------------------------------------------------------
// block = 32 × 8 threads: lane = column inside a 32-column strip, ty strides over rows; fp64 partials reduced through shared memory,
// one atomicAdd per column per block.
__global__ void __launch_bounds__(256)
gene_stats_kernel(const float* __restrict__ X, int64_t ldx, int64_t n, int32_t g, int64_t rows_per_block, double* __restrict__ sum,
                  double* __restrict__ sumsq, double* __restrict__ nnz) {
  __shared__ double sh[3][8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + tx;
  const int64_t r0 = (int64_t)blockIdx.y * rows_per_block, r1 = min(n, r0 + rows_per_block);
  double a = 0.0, b = 0.0, k = 0.0;
  if (c < g) {
    for (int64_t r = r0 + ty; r < r1; r += 8) {
      const float v = X[r * ldx + c];
      a += (double)v;
      b += (double)v * (double)v;
      k += v > 0.f ? 1.0 : 0.0;
    }
  }
  sh[0][ty][tx] = a; sh[1][ty][tx] = b; sh[2][ty][tx] = k;
  __syncthreads();
  if (ty == 0 && c < g) {
    for (int q = 1; q < 8; ++q) { a += sh[0][q][tx]; b += sh[1][q][tx]; k += sh[2][q][tx]; }
    atomicAdd(sum + c, a);
    if (sumsq) atomicAdd(sumsq + c, b);
    if (nnz) atomicAdd(nnz + c, k);
  }
}

// ---- per-cell statistics: Σx and #(x > 0): one warp per row ------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
cell_stats_kernel(const float* __restrict__ X, int64_t ldx, int64_t n, int32_t g, double* __restrict__ sum, double* __restrict__ nnz) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < n; r += nwarps) {
    double a = 0.0, k = 0.0;
    for (int c = lane; c < g; c += 32) {
      const float v = X[r * ldx + c];
      a += (double)v;
      k += v > 0.f ? 1.0 : 0.0;
    }
    a = warp_sum(a); k = warp_sum(k);
    if (lane == 0) { sum[r] = a; if (nnz) nnz[r] = k; }
  }
}

// ---- gather rows / columns (subsetting after a filter): out[i, j] = X[rows[i], cols[j]] ------------------------------------------
__global__ void __launch_bounds__(256)
subset_kernel(const float* __restrict__ X, int64_t ldx, const int64_t* __restrict__ rows, const int32_t* __restrict__ cols, int64_t n_out,
              int32_t g_out, float* __restrict__ out, int64_t ldo) {
  const int64_t total = n_out * g_out;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / g_out;
    const int j = (int)(t % g_out);
    out[i * ldo + j] = X[(rows ? rows[i] : i) * ldx + (cols ? cols[j] : j)];
  }
}

// ---- CellwiseMaskData -------------------------------------------------------------------------------------------------------------------
// uniform01 (common.cuh) with streams 1 and 2

// One block per cell.  Positive entries get the Efraimidis–Spirakis key log(u)/w (w = exp(−x/20) for distr "exp", 1 for
// "uniform"): the n_masked LARGEST keys are a weighted sample without replacement with probabilities ∝ w — the distribution of
// numpy's rng.choice(num_positive, n_masked, p=prob, replace=False).  Among the masked entries a second uniform key picks the
// n_valid = max(1, round(0.1·n_masked)) validation entries (add_test_mask), the rest are test entries.  Ranks are found by
// counting (positives per cell are few hundred), ties broken by column index.
constexpr int CM_MAX_POS = 3072;
__global__ void __launch_bounds__(256)
cellwise_mask_kernel(const float* __restrict__ X, int64_t ldx, int32_t g, float mask_rate, int32_t min_gene_counts, int distr_exp,
                     int add_test_mask, uint32_t seed, uint8_t* __restrict__ train, uint8_t* __restrict__ valid, uint8_t* __restrict__ test,
                     int32_t* __restrict__ overflow_rows) {
  __shared__ float key[CM_MAX_POS];
  __shared__ float key2[CM_MAX_POS];
  __shared__ int32_t colx[CM_MAX_POS];
  __shared__ uint8_t masked[CM_MAX_POS];
  __shared__ int32_t n_pos_s;
  const int64_t row = blockIdx.x;
  const float* x = X + row * ldx;
  uint8_t* tr = train + row * g;
  uint8_t* va = valid + row * g;
  uint8_t* te = test + row * g;
  if (threadIdx.x == 0) n_pos_s = 0;
  __syncthreads();
  for (int c = threadIdx.x; c < g; c += blockDim.x) {
    tr[c] = 1; va[c] = 0; te[c] = 0;
    const float v = x[c];
    if (v != 0.f) {                                   // scipy sparse "positive" entries = stored non-zeros
      const int slot = atomicAdd(&n_pos_s, 1);
      if (slot < CM_MAX_POS) {
        const float w = distr_exp ? __expf(-v * 0.05f) : 1.f;
        const float u = uniform01(seed, 1u, (uint32_t)row, (uint32_t)c);
        key[slot] = __logf(u) / fmaxf(w, 1e-30f);
        key2[slot] = uniform01(seed, 2u, (uint32_t)row, (uint32_t)c);
        colx[slot] = c;
      }
    }
  }
  __syncthreads();
  const int n_pos = n_pos_s;
  if (n_pos > CM_MAX_POS) {                            // more positives than the staging area holds: reported, row left unmasked
    if (threadIdx.x == 0) atomicAdd(overflow_rows, 1);
    return;
  }
  if (n_pos <= min_gene_counts) return;
  int n_masked = (int)floor((double)n_pos * (double)mask_rate);
  if (n_masked <= 0) return;
  if (n_masked >= n_pos) n_masked = 1 + (int)floor(0.5 * (double)n_pos);
  for (int a = threadIdx.x; a < n_pos; a += blockDim.x) {
    const float ka = key[a];
    const int ca = colx[a];
    int rank = 0;                                      // number of entries with a larger key (ties: smaller column first)
    for (int b = 0; b < n_pos; ++b) rank += (key[b] > ka) || (key[b] == ka && colx[b] < ca);
    masked[a] = rank < n_masked;
  }
  __syncthreads();
  int n_valid = n_masked;
  if (add_test_mask) {
    n_valid = (int)rint((double)n_masked * 0.1);       // np.round: half to even
    n_valid = n_masked > 1 ? max(1, n_valid) : n_masked;
  }
  for (int a = threadIdx.x; a < n_pos; a += blockDim.x) {
    if (!masked[a]) continue;
    const int ca = colx[a];
    tr[ca] = 0;
    if (!add_test_mask) { va[ca] = 1; continue; }
    const float ka = key2[a];
    int rank = 0;
    for (int b = 0; b < n_pos; ++b) rank += masked[b] && ((key2[b] < ka) || (key2[b] == ka && colx[b] < ca));
    if (rank < n_valid) va[ca] = 1; else te[ca] = 1;
  }
}

}  // namespace
}  // namespace b2

// sum / sumsq / nnz: [g] doubles (sumsq and nnz may be NULL); zero-filled here
extern "C" int b2_gene_stats_f32(const float* X, int64_t ldx, int64_t n, int32_t g, double* sum, double* sumsq, double* nnz, void* stream) {
  using namespace b2;
  B2_REQUIRE(X && sum && n >= 0 && g > 0 && ldx >= g, "b2_gene_stats_f32: bad arguments");
  cudaStream_t st = as_stream(stream);
  B2_CHECK_CUDA(cudaMemsetAsync(sum, 0, sizeof(double) * g, st));
  if (sumsq) B2_CHECK_CUDA(cudaMemsetAsync(sumsq, 0, sizeof(double) * g, st));
  if (nnz) B2_CHECK_CUDA(cudaMemsetAsync(nnz, 0, sizeof(double) * g, st));
  if (n == 0) return B2_OK;
  const int strips = ceil_div(g, 32);
  int64_t row_blocks = ceil_div<int64_t>((int64_t)sm_count() * 8, strips);
  if (row_blocks > ceil_div<int64_t>(n, 64)) row_blocks = ceil_div<int64_t>(n, 64);
  if (row_blocks < 1) row_blocks = 1;
  if (row_blocks > 65535) row_blocks = 65535;
  const int64_t rpb = ceil_div<int64_t>(n, row_blocks);
  gene_stats_kernel<<<dim3(strips, (unsigned)ceil_div<int64_t>(n, rpb)), 256, 0, st>>>(X, ldx, n, g, rpb, sum, sumsq, nnz);
  B2_CHECK_LAUNCH("gene_stats_kernel");
  return B2_OK;
}

extern "C" int b2_cell_stats_f32(const float* X, int64_t ldx, int64_t n, int32_t g, double* sum, double* nnz, void* stream) {
  using namespace b2;
  B2_REQUIRE(X && sum && n >= 0 && g > 0 && ldx >= g, "b2_cell_stats_f32: bad arguments");
  if (n == 0) return B2_OK;
  cell_stats_kernel<<<grid_blocks(n, 8), 256, 0, as_stream(stream)>>>(X, ldx, n, g, sum, nnz);
  B2_CHECK_LAUNCH("cell_stats_kernel");
  return B2_OK;
}

extern "C" int b2_subset_f32(const float* X, int64_t ldx, const int64_t* rows, const int32_t* cols, int64_t n_out, int32_t g_out,
                             float* out, int64_t ldo, void* stream) {
  using namespace b2;
  B2_REQUIRE(X && out && n_out >= 0 && g_out >= 0 && ldo >= g_out, "b2_subset_f32: bad arguments");
  if (n_out == 0 || g_out == 0) return B2_OK;
  subset_kernel<<<grid_blocks(n_out * g_out, 1024, 32), 256, 0, as_stream(stream)>>>(X, ldx, rows, cols, n_out, g_out, out, ldo);
  B2_CHECK_LAUNCH("subset_kernel");
  return B2_OK;
}

// masks: [n, g] bytes (0 / 1), densely packed; overflow_rows (device int32, zeroed here) counts rows with more than 3072 non-zeros,
// which are left unmasked
extern "C" int b2_cellwise_mask_u8(const float* X, int64_t ldx, int64_t n, int32_t g, float mask_rate, int32_t min_gene_counts,
                                   int distr_exp, int add_test_mask, uint32_t seed, uint8_t* train, uint8_t* valid, uint8_t* test,
                                   int32_t* overflow_rows, void* stream) {
  using namespace b2;
  B2_REQUIRE(X && train && valid && test && overflow_rows, "b2_cellwise_mask_u8: null pointer");
  B2_REQUIRE(n >= 0 && g > 0 && ldx >= g && n <= 2147483647ll, "b2_cellwise_mask_u8: bad shape");
  B2_REQUIRE(mask_rate >= 0.f && mask_rate <= 1.f, "b2_cellwise_mask_u8: mask_rate must be in [0, 1]");
  cudaStream_t st = as_stream(stream);
  B2_CHECK_CUDA(cudaMemsetAsync(overflow_rows, 0, sizeof(int32_t), st));
  if (n == 0) return B2_OK;
  cellwise_mask_kernel<<<(unsigned)n, 256, 0, st>>>(X, ldx, g, mask_rate, min_gene_counts, distr_exp, add_test_mask, seed, train, valid,
                                                    test, overflow_rows);
  B2_CHECK_LAUNCH("cellwise_mask_kernel");
  return B2_OK;
}
