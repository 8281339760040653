// GraphSCI building blocks (reference modules/single_modality/imputation/graphsci.py):
//   BatchNorm1d forward / backward              buildNetwork :37-45 (training: batch statistics, eval: running statistics)
//   decoder heads + ZINB negative log-likelihood + reconstruction MSE, forward value and gradient in one pass
//                                               AEModel :93-112 (Sigmoid / DispActivation / MeanActivation), get_loss :463-483
//   adjacency loss: class-weighted soft-target cross entropy over the gene graph + the KL of the sampled embedding,
//   and the reparameterisation z = mean + exp(log_std)·eps with its backward            GNNModel :126-131, get_loss :455-462,479-481
// All of these are HBM-bound elementwise / row-reduction kernels over [cells, genes] or [genes, genes] matrices.
#include "common.cuh"

namespace b2 {

// ---------------------------------------------------------------------------------------------------------------
// BatchNorm1d over the rows of X [n, c]
// ---------------------------------------------------------------------------------------------------------------
// pass 0: Σx per column ; pass 1: Σ(x-mean)² per column (two-pass variance, fp64 partials)
__global__ void __launch_bounds__(256)
bn_stats_kernel(const float* __restrict__ X, int64_t ldx, int32_t n, int32_t c, int pass, double* __restrict__ sum,
                double* __restrict__ sq) {
  __shared__ double sh[8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int col = blockIdx.x * 32 + tx;
  const int64_t rows_per = ceil_div<int64_t>(n, gridDim.y);
  const int64_t r0 = (int64_t)blockIdx.y * rows_per;
  const int64_t r1 = (r0 + rows_per < (int64_t)n) ? r0 + rows_per : (int64_t)n;
  double s = 0.0;
  if (col < c) {
    if (pass == 0) for (int64_t r = r0 + ty; r < r1; r += 8) s += (double)X[r * ldx + col];
    else {
      const double m = sum[col] / (double)n;
      for (int64_t r = r0 + ty; r < r1; r += 8) { const double d = (double)X[r * ldx + col] - m; s += d * d; }
    }
  }
  sh[ty][tx] = s;
  __syncthreads();
  if (ty == 0 && col < c) {
    for (int i = 1; i < 8; ++i) s += sh[i][tx];
    atomicAdd((pass == 0 ? sum : sq) + col, s);
  }
}

// training: mean/var from the batch, running stats updated (momentum m, unbiased variance) ; eval: running stats
__global__ void bn_finalize_kernel(const double* __restrict__ sum, const double* __restrict__ sq, int32_t n, int32_t c,
                                   int training, float momentum, float eps, float* __restrict__ running_mean,
                                   float* __restrict__ running_var, float* __restrict__ save_mean,
                                   float* __restrict__ save_invstd) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < c; i += gridDim.x * blockDim.x) {
    float mean, var;
    if (training) {
      mean = (float)(sum[i] / (double)n);
      var = (float)(sq[i] / (double)n);                       // biased: used to normalise
      const float unbiased = n > 1 ? (float)(sq[i] / (double)(n - 1)) : var;
      running_mean[i] = (1.f - momentum) * running_mean[i] + momentum * mean;
      running_var[i] = (1.f - momentum) * running_var[i] + momentum * unbiased;
    } else {
      mean = running_mean[i];
      var = running_var[i];
    }
    save_mean[i] = mean;
    save_invstd[i] = 1.f / sqrtf(var + eps);
  }
}

__global__ void __launch_bounds__(256)
bn_apply_kernel(const float* __restrict__ X, int64_t ldx, int32_t n, int32_t c, const float* __restrict__ gamma,
                const float* __restrict__ beta, const float* __restrict__ mean, const float* __restrict__ invstd, int act,
                float* __restrict__ out, int64_t ldo) {
  const int64_t total = (int64_t)n * c;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / c;
    const int j = (int)(t - r * c);
    const float v = (X[r * ldx + j] - mean[j]) * invstd[j] * gamma[j] + beta[j];
    out[r * ldo + j] = apply_act(v, act);
  }
}

// backward (training statistics): with x̂ = (x-mean)·invstd, g = dY ⊙ act'(y):
//   dβ = Σg, dγ = Σ g x̂, dX = γ·invstd·(g - dβ/n - x̂·dγ/n)
// pass A accumulates dβ, dγ (fp64 atomics); pass B writes dX.  eval mode: dX = γ·invstd·g.
__global__ void __launch_bounds__(256)
bn_bwd_reduce_kernel(const float* __restrict__ dY, int64_t lddy, const float* __restrict__ Y, int64_t ldy,
                     const float* __restrict__ X, int64_t ldx, int32_t n, int32_t c, const float* __restrict__ mean,
                     const float* __restrict__ invstd, int act, double* __restrict__ dbeta, double* __restrict__ dgamma) {
  __shared__ double sb[8][33], sg[8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int col = blockIdx.x * 32 + tx;
  const int64_t rows_per = ceil_div<int64_t>(n, gridDim.y);
  const int64_t r0 = (int64_t)blockIdx.y * rows_per;
  const int64_t r1 = (r0 + rows_per < (int64_t)n) ? r0 + rows_per : (int64_t)n;
  double b = 0.0, g = 0.0;
  if (col < c) {
    const float m = mean[col], is = invstd[col];
    for (int64_t r = r0 + ty; r < r1; r += 8) {
      float gy = dY[r * lddy + col];
      if (act == B2_ACT_RELU) gy = Y[r * ldy + col] > 0.f ? gy : 0.f;
      b += gy;
      g += (double)gy * (double)((X[r * ldx + col] - m) * is);
    }
  }
  sb[ty][tx] = b; sg[ty][tx] = g;
  __syncthreads();
  if (ty == 0 && col < c) {
    for (int i = 1; i < 8; ++i) { b += sb[i][tx]; g += sg[i][tx]; }
    atomicAdd(dbeta + col, b);
    atomicAdd(dgamma + col, g);
  }
}

__global__ void __launch_bounds__(256)
bn_bwd_apply_kernel(const float* __restrict__ dY, int64_t lddy, const float* __restrict__ Y, int64_t ldy,
                    const float* __restrict__ X, int64_t ldx, int32_t n, int32_t c, const float* __restrict__ gamma,
                    const float* __restrict__ mean, const float* __restrict__ invstd, int act, int training,
                    const double* __restrict__ dbeta, const double* __restrict__ dgamma, float* __restrict__ dX, int64_t lddx,
                    float* __restrict__ dgamma_out, float* __restrict__ dbeta_out) {
  const int64_t total = (int64_t)n * c;
  const float inv_n = 1.f / (float)n;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / c;
    const int j = (int)(t - r * c);
    float gy = dY[r * lddy + j];
    if (act == B2_ACT_RELU) gy = Y[r * ldy + j] > 0.f ? gy : 0.f;
    const float is = invstd[j];
    float v;
    if (training) {
      const float xh = (X[r * ldx + j] - mean[j]) * is;
      v = gamma[j] * is * (gy - (float)dbeta[j] * inv_n - xh * (float)dgamma[j] * inv_n);
    } else {
      v = gamma[j] * is * gy;
    }
    dX[r * lddx + j] = v;
    if (r == 0) { dgamma_out[j] = (float)dgamma[j]; dbeta_out[j] = (float)dbeta[j]; }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// ZINB heads + loss
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float digammaf_pos(float x) {
  // ψ(x) for x > 0: recurrence up to x >= 6, then the asymptotic series
  float r = 0.f;
  while (x < 6.f) { r -= 1.f / x; x += 1.f; }
  const float f = 1.f / (x * x);
  return r + logf(x) - 0.5f / x - f * (1.f / 12.f - f * (1.f / 120.f - f * (1.f / 252.f - f * (1.f / 240.f))));
}

// The per-element formulas of zinb_kernel (below, kept as it is), as device functions for the fused heads kernels.
// The heads' activations (Sigmoid, clamp(softplus), clamp(exp)) of the three BatchNorm outputs a, b, c.
__device__ __forceinline__ void zinb_act(float a, float b, float cc, float& pi, float& sp, float& disp, float& ex, float& mean) {
  pi = 1.f / (1.f + expf(-a));
  sp = b > 20.f ? b : log1pf(expf(b));                                      // F.softplus (threshold 20)
  disp = fminf(fmaxf(sp, 1e-4f), 1e4f);
  ex = expf(cc);
  mean = fminf(fmaxf(ex, 1e-5f), 1e6f);
}

// ZINB negative log-likelihood of one counted entry (LOSS) and its derivatives w.r.t. pi, disp and mu = mean·sf (GRAD).
template <bool LOSS, bool GRAD>
__device__ __forceinline__ float zinb_nll(float pi, float disp, float mu, float y, float& dl_dpi, float& dl_dd, float& dl_dmu) {
  const float eps = 1e-10f;
  const float de = disp + eps;
  const float ratio = mu / de;
  float loss = 0.f;
  dl_dpi = dl_dd = dl_dmu = 0.f;
  if (y < 1e-8f) {
    const float base = disp / (disp + mu + eps);
    const float lb = logf(base);
    const float znb = expf(disp * lb);
    const float inner = pi + (1.f - pi) * znb + eps;
    if (LOSS) loss = -logf(inner);
    if (GRAD) {
      const float dz_dd = znb * (lb + disp * (1.f / disp - 1.f / (disp + mu + eps)));
      const float dz_dmu = znb * disp * (-1.f / (disp + mu + eps));
      const float k = -1.f / inner;
      dl_dpi = k * (1.f - znb);
      dl_dd = k * (1.f - pi) * dz_dd;
      dl_dmu = k * (1.f - pi) * dz_dmu;
    }
  } else {
    const float l1 = logf(1.f + ratio);
    if (LOSS) {
      const float t1 = lgammaf(de) + lgammaf(y + 1.f) - lgammaf(y + de);
      const float t2 = (disp + y) * l1 + y * (logf(de) - logf(mu + eps));
      loss = t1 + t2;
    }
    if (GRAD) {
      dl_dd = digammaf_pos(de) - digammaf_pos(y + de) + l1 + (disp + y) * (-(ratio / de)) / (1.f + ratio) + y / de;
      dl_dmu = (disp + y) * (1.f / de) / (1.f + ratio) - y / (mu + eps);
    }
  }
  return loss;
}

// Gradients of wn·nll + wm·(mu − y)² w.r.t. the three heads' pre-activations a, b, c (through the clamps).
__device__ __forceinline__ void zinb_grads(float wn, float wm, float b, float sp, float ex, float pi, float mean, float s, float diff,
                                           float dl_dpi, float dl_dd, float dl_dmu, float& ga, float& gb, float& gc) {
  const float g_mu = wn * dl_dmu + wm * 2.f * diff;
  ga = wn * dl_dpi * pi * (1.f - pi);
  gb = (sp > 1e-4f && sp < 1e4f) ? wn * dl_dd * (b > 20.f ? 1.f : 1.f / (1.f + expf(-b))) : 0.f;
  gc = (ex > 1e-5f && ex < 1e6f) ? g_mu * s * mean : 0.f;
}

// a, b, c: the three decoder outputs after BatchNorm (pre-activation) [n, g]; y raw counts; sf size factors [n];
// mask [n, g] bytes (nonzero = counted).  Outputs (all optional): pi/disp/mean activations, and, when da is given, the
// gradients of   le·mean_mask(nll) + ke·(0.5/g)·mean_mask((mean·sf - y)²)   w.r.t. a, b, c (needs the mask count → cnt_dev).
template <bool GRAD>
__global__ void __launch_bounds__(256)
zinb_kernel(const float* __restrict__ A, const float* __restrict__ Bm, const float* __restrict__ Cm, int64_t ld,
            const float* __restrict__ Y, int64_t ldy, const float* __restrict__ sf, const uint8_t* __restrict__ mask,
            int64_t ldm, int32_t n, int32_t g, float le, float ke, const double* __restrict__ cnt_dev,
            float* __restrict__ dA, float* __restrict__ dB, float* __restrict__ dC, int64_t ldd, float* __restrict__ mean_out,
            float* __restrict__ disp_out, float* __restrict__ pi_out, int64_t ldo, double* __restrict__ acc /* nll, mse, cnt */) {
  const int64_t total = (int64_t)n * g;
  const float eps = 1e-10f;
  double nll = 0.0, mse = 0.0, cnt = 0.0;
  float wn = 0.f, wm = 0.f;
  if (GRAD) {
    const float c = (float)cnt_dev[2];
    wn = c > 0.f ? le / c : 0.f;
    wm = c > 0.f ? ke * 0.5f / (float)g / c : 0.f;
  }
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / g;
    const int j = (int)(t - r * g);
    const float a = A[r * ld + j], b = Bm[r * ld + j], cc = Cm[r * ld + j];
    const float pi = 1.f / (1.f + expf(-a));
    const float sp = b > 20.f ? b : log1pf(expf(b));                        // F.softplus (threshold 20)
    const float disp = fminf(fmaxf(sp, 1e-4f), 1e4f);
    const float ex = expf(cc);
    const float mean = fminf(fmaxf(ex, 1e-5f), 1e6f);
    if (mean_out) { mean_out[r * ldo + j] = mean; disp_out[r * ldo + j] = disp; pi_out[r * ldo + j] = pi; }
    const bool m = mask ? mask[r * ldm + j] != 0 : true;
    if (!m) {
      if (GRAD) { dA[r * ldd + j] = 0.f; dB[r * ldd + j] = 0.f; dC[r * ldd + j] = 0.f; }
      continue;
    }
    const float y = Y[r * ldy + j];
    const float s = sf[r];
    const float mu = mean * s;
    const float de = disp + eps;
    const float ratio = mu / de;
    float loss, dl_dpi = 0.f, dl_dd, dl_dmu;
    if (y < 1e-8f) {
      const float base = disp / (disp + mu + eps);
      const float lb = logf(base);
      const float znb = expf(disp * lb);
      const float inner = pi + (1.f - pi) * znb + eps;
      loss = -logf(inner);
      if (GRAD) {
        const float dz_dd = znb * (lb + disp * (1.f / disp - 1.f / (disp + mu + eps)));
        const float dz_dmu = znb * disp * (-1.f / (disp + mu + eps));
        const float k = -1.f / inner;
        dl_dpi = k * (1.f - znb);
        dl_dd = k * (1.f - pi) * dz_dd;
        dl_dmu = k * (1.f - pi) * dz_dmu;
      }
    } else {
      const float t1 = lgammaf(de) + lgammaf(y + 1.f) - lgammaf(y + de);
      const float l1 = logf(1.f + ratio);
      const float t2 = (disp + y) * l1 + y * (logf(de) - logf(mu + eps));
      loss = t1 + t2;
      if (GRAD) {
        dl_dd = digammaf_pos(de) - digammaf_pos(y + de) + l1 + (disp + y) * (-(ratio / de)) / (1.f + ratio) + y / de;
        dl_dmu = (disp + y) * (1.f / de) / (1.f + ratio) - y / (mu + eps);
      }
    }
    const float diff = mu - y;
    nll += (double)loss;
    mse += (double)diff * diff;
    cnt += 1.0;
    if (GRAD) {
      const float g_mu = wn * dl_dmu + wm * 2.f * diff;
      dA[r * ldd + j] = wn * dl_dpi * pi * (1.f - pi);
      dB[r * ldd + j] = (sp > 1e-4f && sp < 1e4f) ? wn * dl_dd * (b > 20.f ? 1.f : 1.f / (1.f + expf(-b))) : 0.f;
      dC[r * ldd + j] = (ex > 1e-5f && ex < 1e6f) ? g_mu * s * mean : 0.f;
    }
  }
  if (!GRAD) {
    nll = warp_sum(nll); mse = warp_sum(mse); cnt = warp_sum(cnt);
    if ((threadIdx.x & 31) == 0) { atomicAdd(acc, nll); atomicAdd(acc + 1, mse); atomicAdd(acc + 2, cnt); }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// The three heads fused: BatchNorm of each head's pre-BatchNorm GEMM output, the activations and the ZINB / MSE loss in
// registers, so that no normalised output, activation or loss gradient is stored.  Per-element formulas are those of
// bn_apply_kernel, zinb_kernel and bn_bwd_apply_kernel.  Per-head vectors (gamma, beta, mean, invstd, dgamma, dbeta) are packed
// [3, g] in the order pi, disp, mean.
// ---------------------------------------------------------------------------------------------------------------
// Training, column-tiled as bn_stats_kernel (32 columns × 8 row lanes per block, gridDim.y row splits).
// PASS 0: acc += {Σ nll, Σ mse, count}; ws[h·g + j] += Σ_r g'_h, ws[(3 + h)·g + j] += Σ_r g'_h·x̂_h, where g' is the loss gradient
//         at a unit mask count (the count is not known yet; every gradient is linear in 1 / count).
// PASS 1: g recomputed with the count; pre_h ← γ·invstd·(g − Σg/n − x̂·Σg·x̂/n) in place; dgamma, dbeta.
template <int PASS>
__global__ void __launch_bounds__(256)
heads_train_kernel(float* __restrict__ P0, float* __restrict__ P1, float* __restrict__ P2, int64_t ldp,
                   const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ mean,
                   const float* __restrict__ invstd, const float* __restrict__ Y, int64_t ldy, const float* __restrict__ sf,
                   const uint8_t* __restrict__ mask, int64_t ldm, int32_t n, int32_t g, float le, float ke,
                   double* __restrict__ ws, double* __restrict__ acc, float* __restrict__ dgamma, float* __restrict__ dbeta) {
  __shared__ double sh[6][8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int col = blockIdx.x * 32 + tx;
  const int64_t rows_per = ceil_div<int64_t>(n, gridDim.y);
  const int64_t r0 = (int64_t)blockIdx.y * rows_per;
  const int64_t r1 = (r0 + rows_per < (int64_t)n) ? r0 + rows_per : (int64_t)n;
  double cs[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  double nll = 0.0, mse = 0.0, cnt = 0.0;
  if (col < g) {
    float m[3], is[3], gm[3], bt[3], sb[3], sg[3];
#pragma unroll
    for (int h = 0; h < 3; ++h) {
      m[h] = mean[h * g + col]; is[h] = invstd[h * g + col]; gm[h] = gamma[h * g + col]; bt[h] = beta[h * g + col];
    }
    float wn, wm;
    const float inv_n = 1.f / (float)n;
    if (PASS == 0) {
      wn = le;
      wm = ke * 0.5f / (float)g;
    } else {
      const double cd = acc[2];
      const float c = (float)cd;
      wn = c > 0.f ? le / c : 0.f;
      wm = c > 0.f ? ke * 0.5f / (float)g / c : 0.f;
#pragma unroll
      for (int h = 0; h < 3; ++h) {
        sb[h] = cd > 0.0 ? (float)(ws[h * g + col] / cd) : 0.f;
        sg[h] = cd > 0.0 ? (float)(ws[(3 + h) * g + col] / cd) : 0.f;
      }
      if (blockIdx.y == 0 && ty == 0) {
#pragma unroll
        for (int h = 0; h < 3; ++h) { dgamma[h * g + col] = sg[h]; dbeta[h * g + col] = sb[h]; }
      }
    }
    for (int64_t r = r0 + ty; r < r1; r += 8) {
      float x[3];
      x[0] = (P0[r * ldp + col] - m[0]) * is[0];
      x[1] = (P1[r * ldp + col] - m[1]) * is[1];
      x[2] = (P2[r * ldp + col] - m[2]) * is[2];
      const float b = x[1] * gm[1] + bt[1];
      float pi, sp, disp, ex, mn;
      zinb_act(x[0] * gm[0] + bt[0], b, x[2] * gm[2] + bt[2], pi, sp, disp, ex, mn);
      float gr[3] = {0.f, 0.f, 0.f};
      if (mask ? mask[r * ldm + col] != 0 : true) {
        const float y = Y[r * ldy + col];
        const float s = sf[r];
        const float mu = mn * s;
        float dl_dpi, dl_dd, dl_dmu;
        const float loss = zinb_nll<PASS == 0, true>(pi, disp, mu, y, dl_dpi, dl_dd, dl_dmu);
        const float diff = mu - y;
        if (PASS == 0) {
          nll += (double)loss;
          mse += (double)diff * diff;
          cnt += 1.0;
        }
        zinb_grads(wn, wm, b, sp, ex, pi, mn, s, diff, dl_dpi, dl_dd, dl_dmu, gr[0], gr[1], gr[2]);
      }
      if (PASS == 0) {
#pragma unroll
        for (int h = 0; h < 3; ++h) { cs[h] += gr[h]; cs[3 + h] += (double)gr[h] * (double)x[h]; }
      } else {
        P0[r * ldp + col] = gm[0] * is[0] * (gr[0] - sb[0] * inv_n - x[0] * sg[0] * inv_n);
        P1[r * ldp + col] = gm[1] * is[1] * (gr[1] - sb[1] * inv_n - x[1] * sg[1] * inv_n);
        P2[r * ldp + col] = gm[2] * is[2] * (gr[2] - sb[2] * inv_n - x[2] * sg[2] * inv_n);
      }
    }
  }
  if (PASS == 0) {
#pragma unroll
    for (int k = 0; k < 6; ++k) sh[k][ty][tx] = cs[k];
    nll = warp_sum(nll); mse = warp_sum(mse); cnt = warp_sum(cnt);
    if (tx == 0 && cnt > 0.0) { atomicAdd(acc, nll); atomicAdd(acc + 1, mse); atomicAdd(acc + 2, cnt); }
    __syncthreads();
    if (ty == 0 && col < g) {
#pragma unroll
      for (int k = 0; k < 6; ++k) {
        double v = cs[k];
        for (int i = 1; i < 8; ++i) v += sh[k][i][tx];
        atomicAdd(ws + k * g + col, v);
      }
    }
  }
}

// Evaluation (running statistics, no gradient) over a row range: acc += {Σ nll, Σ mse, count}; z_exp = mean·sf (optional).
__global__ void __launch_bounds__(256)
heads_eval_kernel(const float* __restrict__ P0, const float* __restrict__ P1, const float* __restrict__ P2, int64_t ldp,
                  const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ mean,
                  const float* __restrict__ invstd, const float* __restrict__ Y, int64_t ldy, const float* __restrict__ sf,
                  const uint8_t* __restrict__ mask, int64_t ldm, int32_t n, int32_t g, double* __restrict__ acc,
                  float* __restrict__ z_exp, int64_t ldz) {
  const int64_t total = (int64_t)n * g;
  double nll = 0.0, mse = 0.0, cnt = 0.0;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / g;
    const int j = (int)(t - r * g);
    const float a = (P0[r * ldp + j] - mean[j]) * invstd[j] * gamma[j] + beta[j];
    const float b = (P1[r * ldp + j] - mean[g + j]) * invstd[g + j] * gamma[g + j] + beta[g + j];
    const float c = (P2[r * ldp + j] - mean[2 * g + j]) * invstd[2 * g + j] * gamma[2 * g + j] + beta[2 * g + j];
    float pi, sp, disp, ex, mn;
    zinb_act(a, b, c, pi, sp, disp, ex, mn);
    const float s = sf[r];
    if (z_exp) z_exp[r * ldz + j] = mn * s;
    if (mask && mask[r * ldm + j] == 0) continue;
    const float y = Y[r * ldy + j];
    const float mu = mn * s;
    float dl_dpi, dl_dd, dl_dmu;
    const float loss = zinb_nll<true, false>(pi, disp, mu, y, dl_dpi, dl_dd, dl_dmu);
    const float diff = mu - y;
    nll += (double)loss;
    mse += (double)diff * diff;
    cnt += 1.0;
  }
  nll = warp_sum(nll); mse = warp_sum(mse); cnt = warp_sum(cnt);
  if ((threadIdx.x & 31) == 0 && cnt > 0.0) { atomicAdd(acc, nll); atomicAdd(acc + 1, mse); atomicAdd(acc + 2, cnt); }
}

// ---------------------------------------------------------------------------------------------------------------
// adjacency side: z = μ + exp(ls)·ε ; weighted soft-target CE over rows ; KL
// ---------------------------------------------------------------------------------------------------------------
// One block per row i of Z [g, g]:  ce_i = -Σ_c w_c t_ic log_softmax(z_i)_c ;  kl_i = Σ_c (1 + 2 ls - μ² - e^{2 ls})
// dZ[i,c] (+)= coef_ce · (softmax_ic Σ_c' w_c' t_ic' - w_c t_ic)
__global__ void __launch_bounds__(256)
adj_loss_kernel(const float* __restrict__ Z, const float* __restrict__ Mu, const float* __restrict__ Ls,
                const float* __restrict__ T, const float* __restrict__ w, int32_t g, float coef_ce, float* __restrict__ dZ,
                double* __restrict__ acc /* ce_sum, kl_sum */) {
  __shared__ float red[8];
  __shared__ float bc;
  const int i = blockIdx.x;
  const float* z = Z + (int64_t)i * g;
  const float* t = T + (int64_t)i * g;
  float mx = -3.4e38f;
  for (int c = threadIdx.x; c < g; c += 256) mx = fmaxf(mx, z[c]);
  mx = warp_max(mx);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x == 0) { float m = red[0]; for (int k = 1; k < 8; ++k) m = fmaxf(m, red[k]); bc = m; }
  __syncthreads();
  mx = bc;
  float se = 0.f, wt = 0.f, wtz = 0.f, kl = 0.f;
  for (int c = threadIdx.x; c < g; c += 256) {
    se += expf(z[c] - mx);
    const float wc = w[c] * t[c];
    wt += wc;
    wtz += wc * z[c];
    const float ls = Ls[(int64_t)i * g + c], mu = Mu[(int64_t)i * g + c];
    const float e = expf(ls);
    kl += 1.f + 2.f * ls - mu * mu - e * e;
  }
  __syncthreads();
  float vals[4] = {se, wt, wtz, kl};
  __shared__ float r4[4][8];
  for (int q = 0; q < 4; ++q) {
    const float v = warp_sum(vals[q]);
    if ((threadIdx.x & 31) == 0) r4[q][threadIdx.x >> 5] = v;
  }
  __syncthreads();
  for (int q = 0; q < 4; ++q) { float v = 0.f; for (int k = 0; k < 8; ++k) v += r4[q][k]; vals[q] = v; }
  const float lse = mx + logf(vals[0]);
  if (threadIdx.x == 0) {
    atomicAdd(acc, (double)(vals[1] * lse - vals[2]));      // -Σ w t (z - lse)
    atomicAdd(acc + 1, (double)vals[3]);
  }
  if (dZ) {
    const float inv = 1.f / vals[0];
    for (int c = threadIdx.x; c < g; c += 256)
      dZ[(int64_t)i * g + c] = coef_ce * (expf(z[c] - mx) * inv * vals[1] - w[c] * t[c]);
  }
}

// dμ = dZ + coef_kl·(-2μ) ; dls = dZ·ε·e^{ls} + coef_kl·(2 - 2e^{2ls})      (loss contains -ka·kl_adj → coef_kl = -ka·0.5/(n_cells·g))
__global__ void __launch_bounds__(256)
adj_reparam_bwd_kernel(const float* __restrict__ dZ, const float* __restrict__ Mu, const float* __restrict__ Ls,
                       const float* __restrict__ Eps, int64_t total, float coef_kl, float* __restrict__ dMu,
                       float* __restrict__ dLs) {
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const float e = expf(Ls[t]);
    dMu[t] = dZ[t] + coef_kl * (-2.f * Mu[t]);
    dLs[t] = dZ[t] * Eps[t] * e + coef_kl * (2.f - 2.f * e * e);
  }
}

__global__ void __launch_bounds__(256)
adj_sample_kernel(const float* __restrict__ Mu, const float* __restrict__ Ls, const float* __restrict__ Eps, int64_t total,
                  float* __restrict__ Z) {
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x)
    Z[t] = Mu[t] + expf(Ls[t]) * Eps[t];       // torch.normal(mean, exp(log_std)) with the noise made explicit
}

}  // namespace b2

using namespace b2;

extern "C" size_t b2_batchnorm_workspace_bytes(int32_t c) { return align_up(sizeof(double) * 2 * (size_t)c, 256); }

extern "C" int b2_batchnorm_stats_f32(const float* X, int64_t ldx, int32_t n, int32_t c, float* running_mean, float* running_var,
                                      int training, float momentum, float eps, float* save_mean, float* save_invstd, void* workspace,
                                      size_t workspace_bytes, void* stream) {
  B2_REQUIRE(running_mean && running_var && save_mean && save_invstd && n > 0 && c > 0, "b2_batchnorm_stats_f32: bad arguments");
  B2_REQUIRE(!training || (X && ldx >= c), "b2_batchnorm_stats_f32: training statistics need X with ldx >= c");
  B2_REQUIRE(workspace && workspace_bytes >= b2_batchnorm_workspace_bytes(c), "b2_batchnorm_stats_f32: workspace too small");
  cudaStream_t st = as_stream(stream);
  double* sum = reinterpret_cast<double*>(workspace);
  double* sq = sum + c;
  if (training) {
    B2_CHECK_CUDA(cudaMemsetAsync(sum, 0, sizeof(double) * 2 * c, st));
    const dim3 grid(ceil_div(c, 32), row_splits(ceil_div(c, 32), n, 64, 4));
    bn_stats_kernel<<<grid, 256, 0, st>>>(X, ldx, n, c, 0, sum, sq);
    B2_CHECK_LAUNCH("bn_stats_kernel<sum>");
    bn_stats_kernel<<<grid, 256, 0, st>>>(X, ldx, n, c, 1, sum, sq);
    B2_CHECK_LAUNCH("bn_stats_kernel<var>");
  }
  bn_finalize_kernel<<<ceil_div(c, 256), 256, 0, st>>>(sum, sq, n, c, training, momentum, eps, running_mean, running_var, save_mean,
                                                       save_invstd);
  B2_CHECK_LAUNCH("bn_finalize_kernel");
  return B2_OK;
}

extern "C" int b2_batchnorm_fwd_f32(const float* X, int64_t ldx, int32_t n, int32_t c, const float* gamma, const float* beta,
                                    float* running_mean, float* running_var, int training, float momentum, float eps, int act,
                                    float* out, int64_t ldo, float* save_mean, float* save_invstd, void* workspace,
                                    size_t workspace_bytes, void* stream) {
  B2_REQUIRE(X && gamma && beta && running_mean && running_var && out && save_mean && save_invstd && n > 0 && c > 0 && ldx >= c &&
                 ldo >= c, "b2_batchnorm_fwd_f32: bad arguments");
  B2_REQUIRE(workspace && workspace_bytes >= b2_batchnorm_workspace_bytes(c), "b2_batchnorm_fwd_f32: workspace too small");
  B2_REQUIRE(act == B2_ACT_NONE || act == B2_ACT_RELU, "b2_batchnorm_fwd_f32: fused activation must be none or relu");
  const int rc = b2_batchnorm_stats_f32(X, ldx, n, c, running_mean, running_var, training, momentum, eps, save_mean, save_invstd,
                                        workspace, workspace_bytes, stream);
  if (rc != B2_OK) return rc;
  bn_apply_kernel<<<grid_blocks((int64_t)n * c, 1024), 256, 0, as_stream(stream)>>>(X, ldx, n, c, gamma, beta, save_mean, save_invstd,
                                                                                    act, out, ldo);
  B2_CHECK_LAUNCH("bn_apply_kernel");
  return B2_OK;
}

extern "C" int b2_batchnorm_bwd_f32(const float* dY, int64_t lddy, const float* Y, int64_t ldy, const float* X, int64_t ldx,
                                    int32_t n, int32_t c, const float* gamma, const float* save_mean, const float* save_invstd,
                                    int act, int training, float* dX, int64_t lddx, float* dgamma, float* dbeta, void* workspace,
                                    size_t workspace_bytes, void* stream) {
  B2_REQUIRE(dY && X && gamma && save_mean && save_invstd && dX && dgamma && dbeta && n > 0 && c > 0,
             "b2_batchnorm_bwd_f32: bad arguments");
  B2_REQUIRE(act == B2_ACT_NONE || (act == B2_ACT_RELU && Y), "b2_batchnorm_bwd_f32: relu needs the forward output Y");
  B2_REQUIRE(workspace && workspace_bytes >= b2_batchnorm_workspace_bytes(c), "b2_batchnorm_bwd_f32: workspace too small");
  cudaStream_t st = as_stream(stream);
  double* db = reinterpret_cast<double*>(workspace);
  double* dg = db + c;
  B2_CHECK_CUDA(cudaMemsetAsync(db, 0, sizeof(double) * 2 * c, st));
  const dim3 grid(ceil_div(c, 32), row_splits(ceil_div(c, 32), n, 64, 4));
  bn_bwd_reduce_kernel<<<grid, 256, 0, st>>>(dY, lddy, Y, ldy, X, ldx, n, c, save_mean, save_invstd, act, db, dg);
  B2_CHECK_LAUNCH("bn_bwd_reduce_kernel");
  bn_bwd_apply_kernel<<<grid_blocks((int64_t)n * c, 1024), 256, 0, st>>>(dY, lddy, Y, ldy, X, ldx, n, c, gamma, save_mean, save_invstd,
                                                                         act, training, db, dg, dX, lddx, dgamma, dbeta);
  B2_CHECK_LAUNCH("bn_bwd_apply_kernel");
  return B2_OK;
}

extern "C" int b2_zinb_loss_grad_f32(const float* a_pi, const float* b_disp, const float* c_mean, int64_t ld, const float* Y,
                                     int64_t ldy, const float* size_factors, const uint8_t* mask, int64_t ldm, int32_t n,
                                     int32_t g, float le, float ke, float* d_a, float* d_b, float* d_c, int64_t ldd,
                                     float* mean_out, float* disp_out, float* pi_out, int64_t ldo, double* acc3, void* stream) {
  B2_REQUIRE(a_pi && b_disp && c_mean && Y && size_factors && acc3 && n > 0 && g > 0, "b2_zinb_loss_grad_f32: bad arguments");
  B2_REQUIRE((!d_a && !d_b && !d_c) || (d_a && d_b && d_c), "b2_zinb_loss_grad_f32: gradients are all-or-none");
  B2_REQUIRE((!mean_out && !disp_out && !pi_out) || (mean_out && disp_out && pi_out), "b2_zinb_loss_grad_f32: outputs are all-or-none");
  cudaStream_t st = as_stream(stream);
  B2_CHECK_CUDA(cudaMemsetAsync(acc3, 0, sizeof(double) * 3, st));
  const unsigned grid = grid_blocks((int64_t)n * g, 1024);
  zinb_kernel<false><<<grid, 256, 0, st>>>(a_pi, b_disp, c_mean, ld, Y, ldy, size_factors, mask, ldm, n, g, le, ke, nullptr, nullptr,
                                          nullptr, nullptr, 0, mean_out, disp_out, pi_out, ldo, acc3);
  B2_CHECK_LAUNCH("zinb_kernel<loss>");
  if (d_a) {
    zinb_kernel<true><<<grid, 256, 0, st>>>(a_pi, b_disp, c_mean, ld, Y, ldy, size_factors, mask, ldm, n, g, le, ke, acc3, d_a, d_b,
                                           d_c, ldd, nullptr, nullptr, nullptr, 0, acc3);
    B2_CHECK_LAUNCH("zinb_kernel<grad>");
  }
  return B2_OK;
}

extern "C" size_t b2_graphsci_heads_workspace_bytes(int32_t g) { return align_up(sizeof(double) * 6 * (size_t)(g > 0 ? g : 0), 256); }

extern "C" int b2_graphsci_heads_train_f32(float* pre_pi, float* pre_disp, float* pre_mean, int64_t ldp, const float* gamma,
                                           const float* beta, const float* mean, const float* invstd, const float* Y, int64_t ldy,
                                           const float* size_factors, const uint8_t* mask, int64_t ldm, int32_t n, int32_t g, float le,
                                           float ke, float* dgamma, float* dbeta, double* acc3, void* workspace, size_t workspace_bytes,
                                           void* stream) {
  B2_REQUIRE(pre_pi && pre_disp && pre_mean && gamma && beta && mean && invstd && Y && size_factors && dgamma && dbeta && acc3,
             "b2_graphsci_heads_train_f32: null pointer");
  B2_REQUIRE(n > 0 && g > 0, "b2_graphsci_heads_train_f32: n and g must be positive");
  B2_REQUIRE(ldp >= g && ldy >= g && (!mask || ldm >= g), "b2_graphsci_heads_train_f32: leading dimension below g");
  B2_REQUIRE(workspace && workspace_bytes >= b2_graphsci_heads_workspace_bytes(g), "b2_graphsci_heads_train_f32: workspace too small");
  cudaStream_t st = as_stream(stream);
  double* ws = reinterpret_cast<double*>(workspace);
  B2_CHECK_CUDA(cudaMemsetAsync(ws, 0, sizeof(double) * 6 * g, st));
  B2_CHECK_CUDA(cudaMemsetAsync(acc3, 0, sizeof(double) * 3, st));
  const dim3 grid(ceil_div(g, 32), row_splits(ceil_div(g, 32), n, 64, 4));
  heads_train_kernel<0><<<grid, 256, 0, st>>>(pre_pi, pre_disp, pre_mean, ldp, gamma, beta, mean, invstd, Y, ldy, size_factors, mask,
                                               ldm, n, g, le, ke, ws, acc3, dgamma, dbeta);
  B2_CHECK_LAUNCH("heads_train_kernel<sums>");
  heads_train_kernel<1><<<grid, 256, 0, st>>>(pre_pi, pre_disp, pre_mean, ldp, gamma, beta, mean, invstd, Y, ldy, size_factors, mask,
                                               ldm, n, g, le, ke, ws, acc3, dgamma, dbeta);
  B2_CHECK_LAUNCH("heads_train_kernel<apply>");
  return B2_OK;
}

extern "C" int b2_graphsci_heads_eval_f32(const float* pre_pi, const float* pre_disp, const float* pre_mean, int64_t ldp,
                                          const float* gamma, const float* beta, const float* mean, const float* invstd, const float* Y,
                                          int64_t ldy, const float* size_factors, const uint8_t* mask, int64_t ldm, int32_t n, int32_t g,
                                          int accumulate, double* acc3, float* z_exp, int64_t ldz, void* stream) {
  B2_REQUIRE(pre_pi && pre_disp && pre_mean && gamma && beta && mean && invstd && Y && size_factors && acc3,
             "b2_graphsci_heads_eval_f32: null pointer");
  B2_REQUIRE(n > 0 && g > 0, "b2_graphsci_heads_eval_f32: n and g must be positive");
  B2_REQUIRE(ldp >= g && ldy >= g && (!mask || ldm >= g) && (!z_exp || ldz >= g),
             "b2_graphsci_heads_eval_f32: leading dimension below g");
  cudaStream_t st = as_stream(stream);
  if (!accumulate) B2_CHECK_CUDA(cudaMemsetAsync(acc3, 0, sizeof(double) * 3, st));
  heads_eval_kernel<<<grid_blocks((int64_t)n * g, 1024), 256, 0, st>>>(pre_pi, pre_disp, pre_mean, ldp, gamma, beta, mean, invstd, Y,
                                                                       ldy, size_factors, mask, ldm, n, g, acc3, z_exp, ldz);
  B2_CHECK_LAUNCH("heads_eval_kernel");
  return B2_OK;
}

extern "C" int b2_adj_sample_f32(const float* mu, const float* log_std, const float* eps, int64_t n_elem, float* z, void* stream) {
  B2_REQUIRE(mu && log_std && eps && z && n_elem >= 0, "b2_adj_sample_f32: bad arguments");
  if (n_elem == 0) return B2_OK;
  adj_sample_kernel<<<grid_blocks(n_elem, 1024), 256, 0, as_stream(stream)>>>(mu, log_std, eps, n_elem, z);
  B2_CHECK_LAUNCH("adj_sample_kernel");
  return B2_OK;
}

extern "C" int b2_adj_loss_grad_f32(const float* z, const float* mu, const float* log_std, const float* target,
                                    const float* class_weight, int32_t g, float coef_ce, float* dz, double* acc2, void* stream) {
  B2_REQUIRE(z && mu && log_std && target && class_weight && acc2 && g > 0, "b2_adj_loss_grad_f32: bad arguments");
  cudaStream_t st = as_stream(stream);
  B2_CHECK_CUDA(cudaMemsetAsync(acc2, 0, sizeof(double) * 2, st));
  adj_loss_kernel<<<g, 256, 0, st>>>(z, mu, log_std, target, class_weight, g, coef_ce, dz, acc2);
  B2_CHECK_LAUNCH("adj_loss_kernel");
  return B2_OK;
}

extern "C" int b2_adj_reparam_bwd_f32(const float* dz, const float* mu, const float* log_std, const float* eps, int64_t n_elem,
                                      float coef_kl, float* dmu, float* dlog_std, void* stream) {
  B2_REQUIRE(dz && mu && log_std && eps && dmu && dlog_std && n_elem >= 0, "b2_adj_reparam_bwd_f32: bad arguments");
  if (n_elem == 0) return B2_OK;
  adj_reparam_bwd_kernel<<<grid_blocks(n_elem, 1024), 256, 0, as_stream(stream)>>>(dz, mu, log_std, eps, n_elem, coef_kl, dmu, dlog_std);
  B2_CHECK_LAUNCH("adj_reparam_bwd_kernel");
  return B2_OK;
}
