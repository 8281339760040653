// Adam update, gradient clipping and small elementwise kernels of the training steps (reparameterisation, activations).
#include "common.cuh"

namespace b2 {

// torch.optim.Adam single-tensor semantics (reference uses optim.Adam: scgnn2.py:301,573,850):
//   g += wd·p ; m = β1 m + (1-β1) g ; v = β2 v + (1-β2) g² ;
//   denom = sqrt(v)/sqrt(1-β2^t) + eps ; p -= (lr/(1-β1^t)) · m/denom
__global__ void __launch_bounds__(256)
adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
            int64_t n, float lr, float b1, float b2, float eps, float wd, float bc1, float bc2_sqrt) {
  const float step_size = lr / bc1;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float gi = g[i];
    const float pi = p[i];
    if (wd != 0.f) gi = fmaf(wd, pi, gi);
    const float mi = m[i] + (gi - m[i]) * (1.f - b1);            // lerp form used by torch (exp_avg.lerp_)
    const float vi = b2 * v[i] + (1.f - b2) * gi * gi;           // mul_(β2).addcmul_(g, g, 1-β2)
    m[i] = mi;
    v[i] = vi;
    const float denom = sqrtf(vi) / bc2_sqrt + eps;
    p[i] = pi - step_size * (mi / denom);
  }
}

// Standalone activation forward / backward over strided [rows, cols] matrices, for every B2_ACT_* code (act_value / act_bwd of
// common.cuh).
__global__ void __launch_bounds__(256)
act_fwd_kernel(const float* __restrict__ x, int64_t ldx, int64_t rows, int32_t cols, int act, float* y, int64_t ldy) {
  const int64_t total = rows * cols;
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = q / cols;
    const int c = (int)(q % cols);
    y[r * ldy + c] = act_value(x[r * ldx + c], act);
  }
}

__global__ void __launch_bounds__(256)
act_bwd_kernel(const float* __restrict__ dy, int64_t lddy, const float* __restrict__ y, int64_t ldy, const float* __restrict__ x,
               int64_t ldx, int64_t rows, int32_t cols, int act, float* dx, int64_t lddx) {
  // grid-stride over the rows·cols elements, stepping (row, column) by the stride's quotient and remainder: no 64-bit division
  // per element
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t dr = stride / cols, dc = stride % cols;
  for (int64_t r = q / cols, c = q % cols; r < rows;) {
    dx[r * lddx + c] = act_bwd(dy[r * lddy + c], y + r * ldy + c, x + r * ldx + c, act);
    r += dr;
    c += dc;
    if (c >= cols) { c -= cols; ++r; }
  }
}

__global__ void __launch_bounds__(256)
reparam_fwd_kernel(const float* __restrict__ mu, const float* __restrict__ logvar, int64_t ldm,
                   const float* __restrict__ eps, int64_t lde, float* __restrict__ z, int64_t ldz, int64_t n, int d) {
  const int64_t total = n * d;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / d;
    const int c = (int)(t % d);
    // eps.mul(std).add_(mu), std = exp(logvar)  (scgnn2.py:396-398)
    z[i * ldz + c] = fmaf(eps[i * lde + c], expf(logvar[i * ldm + c]), mu[i * ldm + c]);
  }
}

__global__ void __launch_bounds__(256)
reparam_bwd_kernel(const float* __restrict__ dz, int64_t lddz, const float* __restrict__ logvar, int64_t ldm,
                   const float* __restrict__ eps, int64_t lde, float* __restrict__ dmu, float* __restrict__ dlogvar,
                   int64_t ldd, int64_t n, int d) {
  const int64_t total = n * d;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / d;
    const int c = (int)(t % d);
    const float g = dz[i * lddz + c];
    dmu[i * ldd + c] += g;
    dlogvar[i * ldd + c] += g * eps[i * lde + c] * expf(logvar[i * ldm + c]);
  }
}

// torch.nn.utils.clip_grad_norm_(params, max_norm) over one flat gradient bucket (stagate.py:221), with an optional
// pre-scale folded in (the engines carry sum-reduced loss gradients; the mean's 1/numel is applied here):
//   g ← s·g ; total = ||g||₂ ; g ← g · min(1, max_norm / (total + 1e-6))
__global__ void __launch_bounds__(256)
sumsq_kernel(const float* __restrict__ g, int64_t n, double* __restrict__ acc) {
  double local = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const double v = (double)g[i];
    local += v * v;
  }
  local = warp_sum(local);
  if ((threadIdx.x & 31) == 0 && local != 0.0) atomicAdd(acc, local);
}

__global__ void __launch_bounds__(256)
clip_scale_kernel(float* __restrict__ g, int64_t n, float pre_scale, float max_norm, const double* __restrict__ acc,
                  float* __restrict__ norm_out) {
  const float total = (float)(sqrt(acc[0]) * (double)fabsf(pre_scale));
  float coef = max_norm / (total + 1e-6f);
  coef = coef < 1.f ? coef : 1.f;
  if (max_norm <= 0.f) coef = 1.f;     // max_norm <= 0: scale only
  if (norm_out && blockIdx.x == 0 && threadIdx.x == 0) norm_out[0] = total;
  const float f = pre_scale * coef;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) g[i] *= f;
}

}  // namespace b2

using namespace b2;

extern "C" int b2_clip_grad_norm_f32(float* grad, int64_t n, float pre_scale, float max_norm, double* sumsq_ws,
                                     float* norm_out, void* stream) {
  B2_REQUIRE(grad && sumsq_ws && n >= 0, "b2_clip_grad_norm_f32: bad arguments");
  if (n == 0) return B2_OK;
  cudaStream_t st = as_stream(stream);
  const unsigned blocks = grid_blocks(n, 1024, 8);
  B2_CHECK_CUDA(cudaMemsetAsync(sumsq_ws, 0, sizeof(double), st));
  sumsq_kernel<<<blocks, 256, 0, st>>>(grad, n, sumsq_ws);
  B2_CHECK_LAUNCH("sumsq_kernel");
  clip_scale_kernel<<<blocks, 256, 0, st>>>(grad, n, pre_scale, max_norm, sumsq_ws, norm_out);
  B2_CHECK_LAUNCH("clip_scale_kernel");
  return B2_OK;
}


extern "C" int b2_adam_step_f32(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n,
                                float lr, float beta1, float beta2, float eps, float weight_decay, int32_t step,
                                void* stream) {
  B2_REQUIRE(param && grad && exp_avg && exp_avg_sq && n >= 0 && step >= 1, "b2_adam_step_f32: bad arguments");
  if (n == 0) return B2_OK;
  // bias corrections are evaluated in double on the host exactly like torch (python floats)
  const double bc1 = 1.0 - pow((double)beta1, (double)step);
  const double bc2 = 1.0 - pow((double)beta2, (double)step);
  adam_kernel<<<grid_blocks(n, 1024), 256, 0, as_stream(stream)>>>(param, grad, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps,
                                                                   weight_decay, (float)bc1, (float)sqrt(bc2));
  B2_CHECK_LAUNCH("adam_kernel");
  return B2_OK;
}

extern "C" int b2_act_f32(const float* x, int64_t ldx, int64_t rows, int32_t cols, int act, float* y, int64_t ldy, void* stream) {
  B2_REQUIRE(rows >= 0 && cols >= 0 && ldx >= cols && ldy >= cols, "b2_act_f32: bad shape");
  B2_REQUIRE(act >= B2_ACT_NONE && act <= B2_ACT_GELU, "b2_act_f32: unknown activation %d", act);
  if (rows == 0 || cols == 0) return B2_OK;
  B2_REQUIRE(x && y, "b2_act_f32: null pointer");
  act_fwd_kernel<<<grid_blocks(rows * cols, 256), 256, 0, as_stream(stream)>>>(x, ldx, rows, cols, act, y, ldy);
  B2_CHECK_LAUNCH("act_fwd_kernel");
  return B2_OK;
}

extern "C" int b2_act_bwd_f32(const float* dy, int64_t lddy, const float* y, int64_t ldy, const float* x, int64_t ldx, int64_t rows,
                              int32_t cols, int act, float* dx, int64_t lddx, void* stream) {
  B2_REQUIRE(rows >= 0 && cols >= 0 && lddy >= cols && lddx >= cols, "b2_act_bwd_f32: bad shape");
  B2_REQUIRE(act >= B2_ACT_NONE && act <= B2_ACT_GELU, "b2_act_bwd_f32: unknown activation %d", act);
  if (rows == 0 || cols == 0) return B2_OK;
  B2_REQUIRE(dy && dx, "b2_act_bwd_f32: null pointer");
  if (act == B2_ACT_GELU) B2_REQUIRE(x && ldx >= cols, "b2_act_bwd_f32: gelu needs the pre-activation x");
  else if (act != B2_ACT_NONE) B2_REQUIRE(y && ldy >= cols, "b2_act_bwd_f32: activation %d needs the output y", act);
  act_bwd_kernel<<<grid_blocks(rows * cols, 256), 256, 0, as_stream(stream)>>>(dy, lddy, y, ldy, x, ldx, rows, cols, act, dx, lddx);
  B2_CHECK_LAUNCH("act_bwd_kernel");
  return B2_OK;
}

extern "C" int b2_reparam_fwd_f32(const float* mu, const float* logvar, int64_t ldm, const float* eps, int64_t lde,
                                  float* z, int64_t ldz, int64_t n, int32_t d, void* stream) {
  B2_REQUIRE(mu && logvar && eps && z && n >= 0 && d > 0 && ldm >= d && lde >= d && ldz >= d,
             "b2_reparam_fwd_f32: bad arguments");
  if (n == 0) return B2_OK;
  reparam_fwd_kernel<<<grid_blocks(n * d, 1024), 256, 0, as_stream(stream)>>>(mu, logvar, ldm, eps, lde, z, ldz, n, d);
  B2_CHECK_LAUNCH("reparam_fwd_kernel");
  return B2_OK;
}

extern "C" int b2_reparam_bwd_f32(const float* dz, int64_t lddz, const float* logvar, int64_t ldm, const float* eps,
                                  int64_t lde, float* dmu, float* dlogvar, int64_t ldd, int64_t n, int32_t d,
                                  void* stream) {
  B2_REQUIRE(dz && logvar && eps && dmu && dlogvar && n >= 0 && d > 0 && lddz >= d && ldm >= d && lde >= d && ldd >= d,
             "b2_reparam_bwd_f32: bad arguments");
  if (n == 0) return B2_OK;
  reparam_bwd_kernel<<<grid_blocks(n * d, 1024), 256, 0, as_stream(stream)>>>(dz, lddz, logvar, ldm, eps, lde, dmu, dlogvar, ldd,
                                                                              n, d);
  B2_CHECK_LAUNCH("reparam_bwd_kernel");
  return B2_OK;
}
