// Symmetric eigensolver + centring helpers for the PCA transforms.
//
// Replaces sklearn.decomposition.PCA inside WeightedFeaturePCA / CellPCA (reference transforms/cell_feature.py:49-75,
// 168-194): PCA = eigen-decomposition of the (small) Gram / covariance matrix, which is built by the tensor-core GEMM.
// The eigensolver is a parallel one-sided Jacobi (Hestenes) iteration on the rows of W = C:
//   every round rotates g/2 disjoint row pairs (p,q) so that <w_p, w_q> = 0, the same rotations are accumulated in V.
//   After convergence the rows of W are orthogonal, ||w_i|| = |λ_i| and row i of V is the eigenvector.
// One CTA per pair, round-robin tournament schedule (g-1 rounds per sweep), everything stays in L2 for g ≲ 3000.
#include "common.cuh"

namespace b2 {

__device__ __forceinline__ float block_sum_256(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) t += red[i];
  return t;
}

// one round of the tournament: pair i of round r (m = padded even size, player m-1 fixed)
__global__ void __launch_bounds__(256)
jacobi_round_kernel(float* __restrict__ W, float* __restrict__ V, int g, int m, int round, float tol,
                    float* __restrict__ off_max) {
  __shared__ float red[8];
  const int i = blockIdx.x;
  int p, q;
  if (i == 0) { p = m - 1; q = round; }
  else { p = (round + i) % (m - 1); q = (round - i + (m - 1)) % (m - 1); }
  if (p >= g || q >= g) return;   // dummy player of an odd-sized problem
  if (p > q) { const int t = p; p = q; q = t; }
  float* wp = W + (size_t)p * g;
  float* wq = W + (size_t)q * g;
  float a = 0.f, b = 0.f, c = 0.f;
  for (int j = threadIdx.x; j < g; j += 256) {
    const float x = wp[j], y = wq[j];
    a = fmaf(x, x, a); b = fmaf(y, y, b); c = fmaf(x, y, c);
  }
  a = block_sum_256(a, red);
  b = block_sum_256(b, red);
  c = block_sum_256(c, red);
  const float denom = sqrtf(a * b);
  const float rel = denom > 0.f ? fabsf(c) / denom : 0.f;
  if (threadIdx.x == 0 && rel > 0.f) atomicMax(reinterpret_cast<int*>(off_max), __float_as_int(rel));
  if (!(rel > tol)) return;
  // rotation that annihilates <w_p, w_q>
  const float zeta = (b - a) / (2.f * c);
  const float t = (zeta >= 0.f ? 1.f : -1.f) / (fabsf(zeta) + sqrtf(1.f + zeta * zeta));
  const float cs = rsqrtf(1.f + t * t), sn = cs * t;
  float* vp = V + (size_t)p * g;
  float* vq = V + (size_t)q * g;
  for (int j = threadIdx.x; j < g; j += 256) {
    const float x = wp[j], y = wq[j];
    wp[j] = cs * x - sn * y;
    wq[j] = sn * x + cs * y;
    const float u = vp[j], w = vq[j];
    vp[j] = cs * u - sn * w;
    vq[j] = sn * u + cs * w;
  }
}

__global__ void eye_kernel(float* V, int g) {
  const size_t total = (size_t)g * g;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x)
    V[t] = (t / g == t % g) ? 1.f : 0.f;
}

// At convergence w_i = λ_i v_i with the rows of W orthogonal to working precision (that is the stopping criterion),
// whereas the accumulated V drifts by ~1e-7 per rotation.  So: |λ_i| = ||w_i|| (sign from <w_i, v_i>) and, for every
// eigenvalue that is not negligibly small, the eigenvector is taken as w_i / ||w_i|| (written back into V).
__global__ void __launch_bounds__(256)
jacobi_finish_kernel(const float* __restrict__ W, float* __restrict__ V, int g, float* __restrict__ evals,
                     const float* __restrict__ max_norm) {
  __shared__ float red[8];
  const int i = blockIdx.x;
  float s = 0.f, nn = 0.f;
  for (int j = threadIdx.x; j < g; j += 256) {
    const float w = W[(size_t)i * g + j];
    s = fmaf(w, V[(size_t)i * g + j], s);
    nn = fmaf(w, w, nn);
  }
  s = block_sum_256(s, red);
  nn = sqrtf(block_sum_256(nn, red));
  if (threadIdx.x == 0) evals[i] = s >= 0.f ? nn : -nn;
  if (nn > 1e-5f * max_norm[0]) {
    const float inv = (s >= 0.f ? 1.f : -1.f) / nn;
    for (int j = threadIdx.x; j < g; j += 256) V[(size_t)i * g + j] = W[(size_t)i * g + j] * inv;
  }
}

__global__ void __launch_bounds__(256)
row_norm_max_kernel(const float* __restrict__ W, int g, float* __restrict__ max_norm) {
  __shared__ float red[8];
  const int i = blockIdx.x;
  float nn = 0.f;
  for (int j = threadIdx.x; j < g; j += 256) { const float w = W[(size_t)i * g + j]; nn = fmaf(w, w, nn); }
  nn = sqrtf(block_sum_256(nn, red));
  if (threadIdx.x == 0) atomicMax(reinterpret_cast<int*>(max_norm), __float_as_int(nn));
}

// C[i,j] -= n * mean[i] * mean[j]      (covariance from the raw second moment: XᵀX − n·m mᵀ)
__global__ void rank1_sub_kernel(float* __restrict__ C, const float* __restrict__ mean, int g, float n) {
  const size_t total = (size_t)g * g;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x)
    C[t] -= n * mean[t / g] * mean[t % g];
}

// X[i,:] -= rowmean(X[i,:])   (one warp per row; used to centre the samples of the Gram-side PCA)
__global__ void __launch_bounds__(256)
row_center_kernel(const float* __restrict__ X, int64_t ldx, int32_t n, int32_t g, float* __restrict__ out, int64_t ldo) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = warp; r < n; r += nwarps) {
    float s = 0.f;
    for (int j = lane; j < g; j += 32) s += X[r * ldx + j];
    s = warp_sum(s) / (float)g;
    for (int j = lane; j < g; j += 32) out[r * ldo + j] = X[r * ldx + j] - s;
  }
}

}  // namespace b2

using namespace b2;

extern "C" int b2_sym_eig_jacobi_f32(float* W, float* V, int32_t g, int32_t max_sweeps, float tol, float* evals,
                                     int32_t* sweeps_done_host, void* workspace, size_t workspace_bytes, void* stream) {
  B2_REQUIRE(W && V && evals && g > 0 && max_sweeps > 0, "b2_sym_eig_jacobi_f32: bad arguments");
  B2_REQUIRE(workspace && workspace_bytes >= 64, "b2_sym_eig_jacobi_f32: workspace too small");
  cudaStream_t st = as_stream(stream);
  float* off_max = reinterpret_cast<float*>(workspace);
  const int m = (g + 1) / 2 * 2;
  {
    size_t blocks = ((size_t)g * g + 255) / 256;
    if (blocks > (size_t)sm_count() * 16) blocks = (size_t)sm_count() * 16;
    eye_kernel<<<(unsigned)blocks, 256, 0, st>>>(V, g);
    B2_CHECK_LAUNCH("eye_kernel");
  }
  // One sweep = memset + (m-1) tiny launches (a few µs of work each): at g = 2000 the solver is launch-bound, so the sweep
  // is captured once into a CUDA graph and replayed; the convergence flag is read back after every replay.
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t exec = nullptr;
  bool use_graph = m - 1 >= 64;
  if (use_graph) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(st, &cs) != cudaSuccess || cs != cudaStreamCaptureStatusNone) use_graph = false;   // caller is capturing
  }
  if (use_graph) {
    if (cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
      cudaMemsetAsync(off_max, 0, sizeof(float), st);
      for (int r = 0; r < m - 1; ++r) jacobi_round_kernel<<<m / 2, 256, 0, st>>>(W, V, g, m, r, tol, off_max);
      if (cudaStreamEndCapture(st, &graph) != cudaSuccess || cudaGraphInstantiate(&exec, graph, 0) != cudaSuccess) {
        use_graph = false;
        (void)cudaGetLastError();
      }
    } else {
      use_graph = false;
      (void)cudaGetLastError();
    }
  }
  int sweep = 0;
  for (; sweep < max_sweeps; ++sweep) {
    if (use_graph) {
      B2_CHECK_CUDA(cudaGraphLaunch(exec, st));
      g_launch_count += (long long)(m - 1);
    } else {
      B2_CHECK_CUDA(cudaMemsetAsync(off_max, 0, sizeof(float), st));
      for (int r = 0; r < m - 1; ++r) {
        jacobi_round_kernel<<<m / 2, 256, 0, st>>>(W, V, g, m, r, tol, off_max);
        B2_CHECK_LAUNCH("jacobi_round_kernel");
      }
    }
    float h = 0.f;
    B2_CHECK_CUDA(cudaMemcpyAsync(&h, off_max, sizeof(float), cudaMemcpyDeviceToHost, st));
    B2_CHECK_CUDA(cudaStreamSynchronize(st));
    if (!(h > tol)) { ++sweep; break; }
  }
  if (exec) cudaGraphExecDestroy(exec);
  if (graph) cudaGraphDestroy(graph);
  if (sweeps_done_host) *sweeps_done_host = sweep;
  float* max_norm = off_max + 4;
  B2_CHECK_CUDA(cudaMemsetAsync(max_norm, 0, sizeof(float), st));
  row_norm_max_kernel<<<g, 256, 0, st>>>(W, g, max_norm);
  B2_CHECK_LAUNCH("row_norm_max_kernel");
  jacobi_finish_kernel<<<g, 256, 0, st>>>(W, V, g, evals, max_norm);
  B2_CHECK_LAUNCH("jacobi_finish_kernel");
  return B2_OK;
}

extern "C" int b2_cov_rank1_sub_f32(float* Cm, const float* mean, int32_t g, float n, void* stream) {
  B2_REQUIRE(Cm && mean && g > 0, "b2_cov_rank1_sub_f32: bad arguments");
  size_t blocks = ((size_t)g * g + 255) / 256;
  if (blocks > (size_t)sm_count() * 16) blocks = (size_t)sm_count() * 16;
  rank1_sub_kernel<<<(unsigned)blocks, 256, 0, as_stream(stream)>>>(Cm, mean, g, n);
  B2_CHECK_LAUNCH("rank1_sub_kernel");
  return B2_OK;
}

extern "C" int b2_row_center_f32(const float* X, int64_t ldx, int32_t n, int32_t g, float* out, int64_t ldo, void* stream) {
  B2_REQUIRE(X && out && n >= 0 && g > 0 && ldx >= g && ldo >= g, "b2_row_center_f32: bad arguments");
  if (n == 0) return B2_OK;
  int64_t blocks = ceil_div<int64_t>(n, 8);
  const int64_t cap = (int64_t)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  row_center_kernel<<<(unsigned)blocks, 256, 0, as_stream(stream)>>>(X, ldx, n, g, out, ldo);
  B2_CHECK_LAUNCH("row_center_kernel");
  return B2_OK;
}
