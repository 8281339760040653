// SpaGCN's deep-embedded-clustering head (reference modules/spatial/spatial_domain/spagcn.py, SimpleGCDEC :369-425):
//   q_ij ∝ ((1 + ||z_i - mu_j||²/alpha) + 1e-8)^-(alpha+1) / 2, row-normalised          (forward, :391-397)
//   p_ij = (q_ij² / Σ_i q_ij) / Σ_j (…)                                                  (target_distribution, :408-425)
//   loss = mean_i Σ_j p_ij log(p_ij / (q_ij + 1e-6))                                     (loss_function, :399-406)
// plus the SGD-with-momentum update the reference trains it with (optim.SGD(momentum=0.9), :463).
// One warp per spot; K ≤ 64 clusters, embedding width h ≤ 256.  The backward pass recomputes q (nothing N×K is kept
// besides p) and produces dz per spot and dmu through per-block shared-memory partials + atomics.
#include "common.cuh"
#include "spatial_pair.cuh"

namespace b2 {

constexpr int DEC_MAXK = 64;

// computes u_j (lanes own clusters j = lane, lane+32) and returns the row normaliser S
__device__ __forceinline__ void dec_row_q(const float* __restrict__ zi, const float* __restrict__ mu, int K, int h,
                                          float alpha, int lane, float (&u)[2], float (&t)[2]) {
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    const int j = lane + 32 * s;
    u[s] = 0.f;
    t[s] = 0.f;
    if (j < K) {
      float d2 = 0.f;
      for (int c = 0; c < h; ++c) { const float df = zi[c] - mu[(size_t)j * h + c]; d2 = fmaf(df, df, d2); }
      t[s] = 1.f / ((1.f + d2 / alpha) + 1e-8f);
      u[s] = powf(t[s], alpha + 1.f) / 2.f;       // q**(alpha+1.0)/2.0 — the precedence quirk of spagcn.py:395
    }
  }
}

__global__ void __launch_bounds__(256)
dec_q_kernel(const float* __restrict__ z, int64_t ldz, const float* __restrict__ mu, int32_t n, int32_t K, int32_t h,
             float alpha, float* __restrict__ q, int64_t ldq) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = warp; i < n; i += nwarps) {
    float u[2], t[2];
    dec_row_q(z + i * ldz, mu, K, h, alpha, lane, u, t);
    const float S = warp_sum(u[0] + u[1]);
#pragma unroll
    for (int s = 0; s < 2; ++s) { const int j = lane + 32 * s; if (j < K) q[i * ldq + j] = u[s] / S; }
  }
}

// p = q² / colsum(q), then row-normalised
__global__ void __launch_bounds__(256)
dec_target_kernel(const float* __restrict__ q, int64_t ldq, const float* __restrict__ colsum, int32_t n, int32_t K,
                  float* __restrict__ p, int64_t ldp) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = warp; i < n; i += nwarps) {
    float w[2] = {0.f, 0.f};
#pragma unroll
    for (int s = 0; s < 2; ++s) { const int j = lane + 32 * s; if (j < K) { const float v = q[i * ldq + j]; w[s] = v * v / colsum[j]; } }
    const float S = warp_sum(w[0] + w[1]);
#pragma unroll
    for (int s = 0; s < 2; ++s) { const int j = lane + 32 * s; if (j < K) p[i * ldp + j] = w[s] / S; }
  }
}

// loss + gradients wrt z and mu.  Two phases per spot (one warp each):
//   A (lanes own clusters j): d²_ij, t_ij, u_ij → q_ij, loss, c_ij = ∂L/∂d²_ij, argmax
//   B (lanes own embedding columns c): dz_i[c] = Σ_j 2 c_ij (z_ic − μ_jc), and the same terms, negated, go to dμ_j[c] through a
//     per-block shared-memory accumulator (K·h floats) that is flushed with one global atomic per entry per block — the
//     first version issued K·h global atomics PER SPOT onto K·h addresses and ran at 0.1 % of the HBM roofline.
__global__ void __launch_bounds__(256)
dec_kl_grad_kernel(const float* __restrict__ z, int64_t ldz, const float* __restrict__ mu, const float* __restrict__ p,
                   int64_t ldp, int32_t n, int32_t K, int32_t h, float alpha, float* __restrict__ q_out, int64_t ldq,
                   float* __restrict__ dz, int64_t lddz, float* __restrict__ dmu, float* __restrict__ loss_out,
                   int32_t* __restrict__ labels_out, int use_smem) {
  extern __shared__ float s_dmu[];       // [K*h] when use_smem
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const float inv_n = 1.f / (float)n;
  if (use_smem) {
    for (int t = threadIdx.x; t < K * h; t += blockDim.x) s_dmu[t] = 0.f;
    __syncthreads();
  }
  float* acc_mu = use_smem ? s_dmu : dmu;
  float loss = 0.f;
  for (int64_t i = warp; i < n; i += nwarps) {
    const float* zi = z + i * ldz;
    float u[2], t[2];
    dec_row_q(zi, mu, K, h, alpha, lane, u, t);
    const float S = warp_sum(u[0] + u[1]);
    float qv[2], g[2], gq = 0.f;
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      const int j = lane + 32 * s;
      qv[s] = 0.f; g[s] = 0.f;
      if (j < K) {
        qv[s] = u[s] / S;
        const float pv = p[i * ldp + j];
        loss += pv * logf(pv / (qv[s] + 1e-6f));
        g[s] = -inv_n * pv / (qv[s] + 1e-6f);               // dL/dq
        gq += g[s] * qv[s];
        if (q_out) q_out[i * ldq + j] = qv[s];
      }
    }
    gq = warp_sum(gq);
    if (labels_out) {   // torch.argmax(q, dim=1): first index of the maximum
      float bv = qv[0]; int bj = lane;
      if (lane + 32 < K && qv[1] > bv) { bv = qv[1]; bj = lane + 32; }
      if (lane >= K) { bv = -1.f; bj = 0x7fffffff; }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
        if (ov > bv || (ov == bv && oj < bj)) { bv = ov; bj = oj; }
      }
      if (lane == 0) labels_out[i] = bj;
    }
    // 2·dL/d(d²_ij), held by the lane that owns cluster j
    float cij[2];
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      const int j = lane + 32 * s;
      cij[s] = 0.f;
      if (j < K) {
        const float du = (g[s] - gq) / S;
        cij[s] = 2.f * du * (alpha + 1.f) * powf(t[s], alpha) * 0.5f * (-t[s] * t[s]) / alpha;
      }
    }
    // phase B: lanes over embedding columns
    for (int c0 = 0; c0 < h; c0 += 32) {
      const int c = c0 + lane;
      const float zc = c < h ? zi[c] : 0.f;
      float acc = 0.f;
      for (int j = 0; j < K; ++j) {
        const float cj = __shfl_sync(0xffffffffu, j < 32 ? cij[0] : cij[1], j & 31);
        if (c < h) {
          const float v = cj * (zc - mu[(size_t)j * h + c]);
          acc += v;
          atomicAdd(acc_mu + (size_t)j * h + c, -v);        // shared-memory atomic (conflict-free across lanes) unless K·h is huge
        }
      }
      if (c < h) dz[i * lddz + c] = acc;
    }
  }
  loss = warp_sum(loss);
  if (lane == 0 && loss != 0.f) atomicAdd(loss_out, loss * inv_n);
  if (use_smem) {
    __syncthreads();
    for (int t = threadIdx.x; t < K * h; t += blockDim.x) { const float v = s_dmu[t]; if (v != 0.f) atomicAdd(dmu + t, v); }
  }
}

// torch.optim.SGD(momentum, dampening=0, nesterov=False, weight_decay): buf = g (first step) | m·buf + g ; p -= lr·buf
__global__ void __launch_bounds__(256)
sgd_momentum_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ buf, int64_t n, float lr,
                    float momentum, float wd, int first) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float gi = g[i];
    if (wd != 0.f) gi = fmaf(wd, p[i], gi);
    const float b = first ? gi : fmaf(momentum, buf[i], gi);
    buf[i] = b;
    p[i] -= lr * b;
  }
}

// Σ_ij exp(-D_ij² / (2 l²)) over a dense distance matrix (SpaGCN.calculate_p / search_l, spagcn.py:249-251)
__global__ void __launch_bounds__(256)
exp_adj_sum_kernel(const float* __restrict__ D, int64_t total, float two_l2, double* __restrict__ acc) {
  double local = 0.0;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    local += (double)exp_adj_weight(D[t], two_l2);
  }
  local = warp_sum(local);
  if ((threadIdx.x & 31) == 0) atomicAdd(acc, local);
}

__global__ void __launch_bounds__(256)
exp_adj_kernel(const float* __restrict__ D, float* __restrict__ out, int64_t total, float two_l2) {
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    out[t] = exp_adj_weight(D[t], two_l2);
  }
}

}  // namespace b2

using namespace b2;

extern "C" int b2_dec_q_f32(const float* z, int64_t ldz, const float* mu, int32_t n, int32_t K, int32_t h, float alpha,
                            float* q, int64_t ldq, void* stream) {
  B2_REQUIRE(z && mu && q && n >= 0 && K > 0 && K <= DEC_MAXK && h > 0 && ldz >= h && ldq >= K, "b2_dec_q_f32: bad arguments (K <= 64)");
  if (n == 0) return B2_OK;
  dec_q_kernel<<<grid_blocks(n, 8), 256, 0, as_stream(stream)>>>(z, ldz, mu, n, K, h, alpha, q, ldq);
  B2_CHECK_LAUNCH("dec_q_kernel");
  return B2_OK;
}

extern "C" int b2_dec_target_f32(const float* q, int64_t ldq, const float* colsum, int32_t n, int32_t K, float* p,
                                 int64_t ldp, void* stream) {
  B2_REQUIRE(q && colsum && p && n >= 0 && K > 0 && K <= DEC_MAXK && ldq >= K && ldp >= K, "b2_dec_target_f32: bad arguments");
  if (n == 0) return B2_OK;
  dec_target_kernel<<<grid_blocks(n, 8), 256, 0, as_stream(stream)>>>(q, ldq, colsum, n, K, p, ldp);
  B2_CHECK_LAUNCH("dec_target_kernel");
  return B2_OK;
}

extern "C" int b2_dec_kl_grad_f32(const float* z, int64_t ldz, const float* mu, const float* p, int64_t ldp, int32_t n,
                                  int32_t K, int32_t h, float alpha, float* q_out, int64_t ldq, float* dz, int64_t lddz,
                                  float* dmu, float* loss_out, int32_t* labels_out, void* stream) {
  B2_REQUIRE(z && mu && p && dz && dmu && loss_out && n > 0 && K > 0 && K <= DEC_MAXK && h > 0, "b2_dec_kl_grad_f32: bad arguments");
  cudaStream_t st = as_stream(stream);
  B2_CHECK_CUDA(cudaMemsetAsync(dmu, 0, sizeof(float) * (size_t)K * h, st));
  B2_CHECK_CUDA(cudaMemsetAsync(loss_out, 0, sizeof(float), st));
  const size_t smem = sizeof(float) * (size_t)K * h;
  const int use_smem = smem <= 48 * 1024;
  const unsigned grid = grid_blocks(n, 8, use_smem ? 4 : 16);   // fewer, longer-lived blocks → fewer flushes
  dec_kl_grad_kernel<<<grid, 256, use_smem ? smem : 0, st>>>(z, ldz, mu, p, ldp, n, K, h, alpha, q_out, ldq, dz, lddz, dmu, loss_out,
                                                              labels_out, use_smem);
  B2_CHECK_LAUNCH("dec_kl_grad_kernel");
  return B2_OK;
}

extern "C" int b2_sgd_momentum_step_f32(float* param, const float* grad, float* momentum_buf, int64_t n, float lr,
                                        float momentum, float weight_decay, int32_t step, void* stream) {
  B2_REQUIRE(param && grad && momentum_buf && n >= 0 && step >= 1, "b2_sgd_momentum_step_f32: bad arguments");
  if (n == 0) return B2_OK;
  sgd_momentum_kernel<<<grid_blocks(n, 1024), 256, 0, as_stream(stream)>>>(param, grad, momentum_buf, n, lr, momentum, weight_decay,
                                                                           step == 1);
  B2_CHECK_LAUNCH("sgd_momentum_kernel");
  return B2_OK;
}

extern "C" int b2_exp_adj_f32(const float* D, float* out, int64_t n_elem, double l, double* sum_out_dev, void* stream) {
  B2_REQUIRE(D && n_elem >= 0 && l > 0.0 && (out || sum_out_dev), "b2_exp_adj_f32: bad arguments");
  if (n_elem == 0) return B2_OK;
  cudaStream_t st = as_stream(stream);
  const float two_l2 = exp_adj_two_l2(l);
  const unsigned blocks = grid_blocks(n_elem, 2048);
  if (sum_out_dev) {
    B2_CHECK_CUDA(cudaMemsetAsync(sum_out_dev, 0, sizeof(double), st));
    exp_adj_sum_kernel<<<blocks, 256, 0, st>>>(D, n_elem, two_l2, sum_out_dev);
    B2_CHECK_LAUNCH("exp_adj_sum_kernel");
  }
  if (out) {
    exp_adj_kernel<<<blocks, 256, 0, st>>>(D, out, n_elem, two_l2);
    B2_CHECK_LAUNCH("exp_adj_kernel");
  }
  return B2_OK;
}
