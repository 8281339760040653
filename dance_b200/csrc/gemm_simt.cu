// CUDA-core fp32 GEMM with fused epilogue — the exact-fp32 path and the
// fallback for shapes the tensor-core kernel does not take (tiny / unaligned).
//   C = act(op(A)·op(B) + bias) ⊙ [mask > 0]  (+ beta·C)
// Replaces torch.mm / nn.Linear on the reference hot path
// (scgnn2.py:352-370,499; spagcn.py:358; gnn.py:57).
#include "common.cuh"

namespace b2 {

constexpr int SG_BM = 128, SG_BN = 128, SG_BK = 16, SG_THREADS = 256, SG_PAD = 4;

__global__ void __launch_bounds__(SG_THREADS)
gemm_simt_kernel(const float* __restrict__ A, int64_t lda, int transA, const float* __restrict__ B, int64_t ldb,
                 int transB, float* __restrict__ C, int64_t ldc, int M, int N, int K,
                 const float* __restrict__ bias, int act, const float* __restrict__ mask, int64_t ldmask,
                 float beta) {
  __shared__ __align__(16) float As[2][SG_BK][SG_BM + SG_PAD];
  __shared__ __align__(16) float Bs[2][SG_BK][SG_BN + SG_PAD];

  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * SG_BM, n0 = blockIdx.x * SG_BN;

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  float ra[8], rb[8];
  auto load_tiles = [&](int k0) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int idx = tid + i * SG_THREADS;
      int m, k;
      if (!transA) { k = idx & (SG_BK - 1); m = idx >> 4; } else { m = idx & (SG_BM - 1); k = idx >> 7; }
      const int gm = m0 + m, gk = k0 + k;
      float v = 0.f;
      if (gm < M && gk < K) v = transA ? __ldg(A + (int64_t)gk * lda + gm) : __ldg(A + (int64_t)gm * lda + gk);
      ra[i] = v;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int idx = tid + i * SG_THREADS;
      int n, k;
      if (!transB) { n = idx & (SG_BN - 1); k = idx >> 7; } else { k = idx & (SG_BK - 1); n = idx >> 4; }
      const int gn = n0 + n, gk = k0 + k;
      float v = 0.f;
      if (gn < N && gk < K) v = transB ? __ldg(B + (int64_t)gn * ldb + gk) : __ldg(B + (int64_t)gk * ldb + gn);
      rb[i] = v;
    }
  };
  auto store_tiles = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int idx = tid + i * SG_THREADS;
      int m, k;
      if (!transA) { k = idx & (SG_BK - 1); m = idx >> 4; } else { m = idx & (SG_BM - 1); k = idx >> 7; }
      As[buf][k][m] = ra[i];
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int idx = tid + i * SG_THREADS;
      int n, k;
      if (!transB) { n = idx & (SG_BN - 1); k = idx >> 7; } else { k = idx & (SG_BK - 1); n = idx >> 4; }
      Bs[buf][k][n] = rb[i];
    }
  };

  const int nk = (K + SG_BK - 1) / SG_BK;
  load_tiles(0);
  store_tiles(0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) load_tiles((kt + 1) * SG_BK);
#pragma unroll
    for (int k = 0; k < SG_BK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < nk) {
      store_tiles(buf ^ 1);
      __syncthreads();
    }
  }

#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int gm = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (gm >= M) continue;
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      const int gn0 = n0 + jh * 64 + tx * 4;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int gn = gn0 + j;
        if (gn >= N) continue;
        float v = acc[i][jh * 4 + j];
        if (bias) v += __ldg(bias + gn);
        v = apply_act(v, act);
        if (mask && !(__ldg(mask + (int64_t)gm * ldmask + gn) > 0.f)) v = 0.f;
        float* cp = C + (int64_t)gm * ldc + gn;
        if (beta != 0.f) v = fmaf(beta, *cp, v);
        *cp = v;
      }
    }
  }
}

int gemm_simt(const float* A, int64_t lda, int transA, const float* B, int64_t ldb, int transB, float* C,
              int64_t ldc, int M, int N, int K, const float* bias, int act, const float* mask, int64_t ldmask,
              float beta, cudaStream_t st) {
  dim3 grid(ceil_div(N, SG_BN), ceil_div(M, SG_BM));
  gemm_simt_kernel<<<grid, SG_THREADS, 0, st>>>(A, lda, transA, B, ldb, transB, C, ldc, M, N, K, bias, act, mask,
                                                ldmask, beta);
  B2_CHECK_LAUNCH("gemm_simt_kernel");
  return B2_OK;
}

// ---- column sums (bias gradient) -------------------------------------------
// out[n] = beta*out[n] + Σ_m X[m,n]; each block owns 32 columns and strides over rows.
__global__ void __launch_bounds__(256)
colsum_kernel(const float* __restrict__ X, int64_t ldx, int M, int N, float* __restrict__ out, float beta,
              float* __restrict__ partial, int row_splits) {
  __shared__ float red[8][33];
  const int col = blockIdx.x * 32 + (threadIdx.x & 31);
  const int wy = threadIdx.x >> 5;
  const int split = blockIdx.y;
  const int64_t rows_per = ceil_div<int64_t>(M, row_splits);
  const int64_t r0 = split * rows_per;
  const int64_t r1 = (r0 + rows_per < (int64_t)M) ? r0 + rows_per : (int64_t)M;
  float s = 0.f;
  if (col < N)
    for (int64_t r = r0 + wy; r < r1; r += 8) s += __ldg(X + r * ldx + col);
  red[wy][threadIdx.x & 31] = s;
  __syncthreads();
  if (wy == 0 && col < N) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i][threadIdx.x & 31];
    if (row_splits == 1) out[col] = (beta != 0.f ? beta * out[col] : 0.f) + t;
    else partial[(int64_t)split * N + col] = t;
  }
}

__global__ void colsum_finish_kernel(const float* __restrict__ partial, int N, int row_splits, float* out, float beta) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= N) return;
  float t = 0.f;
  for (int s = 0; s < row_splits; ++s) t += partial[(int64_t)s * N + col];
  out[col] = (beta != 0.f ? beta * out[col] : 0.f) + t;
}

}  // namespace b2

static int colsum_splits(int M, int N) {
  // enough blocks to fill the machine: (N/32 column blocks) x splits; each split covers >= 256 rows
  const int col_blocks = b2::ceil_div(N, 32);
  int splits = b2::ceil_div(b2::sm_count() * 4, col_blocks);
  const int max_splits = M / 256 > 0 ? M / 256 : 1;
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  return splits;
}

extern "C" size_t b2_colsum_workspace_bytes(int M, int N) {
  const int splits = colsum_splits(M, N);
  return splits > 1 ? (size_t)splits * N * sizeof(float) : 0;
}

extern "C" int b2_colsum_f32(const float* X, int64_t ldx, int M, int N, float* out, float beta, void* workspace,
                             size_t workspace_bytes, void* stream) {
  using namespace b2;
  B2_REQUIRE(X && out && M >= 0 && N > 0 && ldx >= N, "b2_colsum_f32: bad arguments");
  cudaStream_t st = as_stream(stream);
  const int splits = colsum_splits(M, N);
  if (splits == 1) {
    dim3 grid(ceil_div(N, 32), 1);
    colsum_kernel<<<grid, 256, 0, st>>>(X, ldx, M, N, out, beta, nullptr, 1);
    B2_CHECK_LAUNCH("colsum_kernel");
    return B2_OK;
  }
  B2_REQUIRE(workspace && workspace_bytes >= (size_t)splits * N * sizeof(float), "b2_colsum_f32: workspace too small");
  float* partial = reinterpret_cast<float*>(workspace);
  // deterministic two-stage reduction: fixed row ranges per split, fixed summation order in the finish kernel
  dim3 grid(ceil_div(N, 32), splits);
  colsum_kernel<<<grid, 256, 0, st>>>(X, ldx, M, N, out, beta, partial, splits);
  B2_CHECK_LAUNCH("colsum_kernel");
  colsum_finish_kernel<<<ceil_div(N, 256), 256, 0, st>>>(partial, N, splits, out, beta);
  B2_CHECK_LAUNCH("colsum_finish_kernel");
  return B2_OK;
}
