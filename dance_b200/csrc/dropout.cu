// Inverted dropout with counter-based keep bits: y[r, c] = keep(seed, key, r, c) ? x[r, c] / (1 - p) : 0.
//
// Replaces, in the reference, the feature sites of scGNN's GATLayer dropout (scgnn2.py:1005 input, :1010 projection).  The
// keep bit is a pure function of (seed, key, r, c) (common.cuh dropout_keep), so the backward pass applies the forward's mask by
// calling the same routine on the gradient with the same key, and the attention site (gat.cu) draws from the same function.
#include "common.cuh"

namespace b2 {

__global__ void __launch_bounds__(256)
dropout_kernel(const float* __restrict__ x, int64_t ldx, int64_t rows, int32_t cols, float p, float scale, uint32_t seed,
               uint32_t key, float* y, int64_t ldy) {
  const int64_t total = rows * cols;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / cols;
    const int c = (int)(t % cols);
    const float v = x[r * ldx + c];   // read before the write: y may alias x
    y[r * ldy + c] = dropout_keep(seed, key, (uint32_t)r, (uint32_t)c, p) ? v * scale : 0.f;
  }
}

}  // namespace b2

using namespace b2;

extern "C" int b2_dropout_f32(const float* x, int64_t ldx, int64_t rows, int32_t cols, float p, uint32_t seed, uint32_t key,
                              float* y, int64_t ldy, void* stream) {
  B2_REQUIRE(rows >= 0 && cols >= 0 && ldx >= cols && ldy >= cols, "b2_dropout_f32: bad shape");
  B2_REQUIRE(p >= 0.f && p <= 1.f, "b2_dropout_f32: p must be in [0, 1]");
  if (rows == 0 || cols == 0) return B2_OK;
  B2_REQUIRE(x && y, "b2_dropout_f32: null pointer");
  dropout_kernel<<<grid_blocks(rows * cols, 1024), 256, 0, as_stream(stream)>>>(x, ldx, rows, cols, p, p < 1.f ? 1.f / (1.f - p) : 0.f,
                                                                                seed, key, y, ldy);
  B2_CHECK_LAUNCH("dropout_kernel");
  return B2_OK;
}
