// Loss kernels of the scGNN path: value + gradient in one pass.
//   - Feature-AE reconstruction loss  (reference scgnn2.py:1298-1328)
//   - Graph-AE inner-product-decoder BCE + KLD, matrix-free
//     (reference scgnn2.py:423-426, 603-619): the N×N logits z zᵀ and the
//     dense label matrix (scgnn2.py:557) are never materialised.
#include "common.cuh"

namespace b2 {

// ---------------------------------------------------------------------------
// Feature-AE loss
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
mse_loss_grad_kernel(const float* __restrict__ recon, const float* __restrict__ target,
                     const float* __restrict__ ltmg, float regu, int relu_mask, float* __restrict__ grad,
                     float* __restrict__ loss_out, int64_t n) {
  double local = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float r = recon[i];
    const float d = r - target[i];
    // loss = (1-s)·d² + s·d²·T   ("LTMG", scgnn2.py:1313-1315);  "noregu" is s = 0.
    // A NULL regulariser matrix means T = 0 (the reference driver passes an all-zero TRS, scgnn2.py:40).
    const float w = (1.f - regu) + (ltmg ? regu * ltmg[i] : 0.f);
    local += (double)(w * d * d);
    float g = 2.f * w * d;
    if (relu_mask && !(r > 0.f)) g = 0.f;  // final decoder ReLU (scgnn2.py:362)
    grad[i] = g;
  }
  local = warp_sum(local);
  __shared__ double sred[8];
  if ((threadIdx.x & 31) == 0) sred[threadIdx.x >> 5] = local;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += sred[i];
    // per-block partials are reduced in fp64; the running total is the reference's fp32 `train_loss +=`
    atomicAdd(loss_out, (float)t);
  }
}

// ---------------------------------------------------------------------------
// Graph-AE loss.
//   S = Σ_{ij} softplus(x_ij)  +  Σ_{(i,j)∈L} h(x_ij),   x_ij = z_i·z_j
//   h(x) = pw·softplus(-x) - softplus(x)   (pos-weighted BCE, pos_weight = L·pw)
//        = -x                              (plain BCE, use_pos_weight = 0)
//   cost = c · S,  c = norm / n²   (mean over all n² logits, scgnn2.py:604)
//   L symmetric ⇒ dS/dz_i = 2·Σ_j σ(x_ij) z_j + 2·Σ_{j∈L_i} h'(x_ij) z_j
// ---------------------------------------------------------------------------
__device__ __forceinline__ float softplus_f(float x) {
  // max(x,0) + log1p(exp(-|x|)) — the same stable form ATen uses for BCE-with-logits
  return fmaxf(x, 0.f) + log1pf(__expf(-fabsf(x)));
}
__device__ __forceinline__ float sigmoid_f(float x) {
  const float e = __expf(-fabsf(x));
  const float s = 1.f / (1.f + e);
  return x >= 0.f ? s : e * s;
}

constexpr int GL_THREADS = 128;            // threads per CTA
// rows of z per thread (amortises the shared-memory operand reads); 1 for wide embeddings (register budget)
template <int D> struct GaeCfg { static constexpr int RPT = D <= 16 ? 2 : 1; static constexpr int ROWS = GL_THREADS * RPT; };
constexpr int GL_JT = 128;                 // j-tile staged in shared memory

__device__ __forceinline__ float ex2_approx(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float lg2_approx(float x) { float y; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float rcp_approx(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
// two independent fused multiply-adds on a feature pair (round-to-nearest, like one packed f32x2 FMA)
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }

// All-pairs part: thread t owns rows i0+t and i0+t+GL_THREADS, loops over every column j (tiles in smem,
// broadcast reads).  Per logit: 2·D FMA (dot + gradient accumulate) and three SFU ops
// (e = 2^(-|x|·log2e), r = 1/(1+e), log2(1+e)); softplus(x) = max(x,0) + ln2·log2(1+e), σ(x) = x≥0 ? r : e·r.
template <int D>
__global__ void __launch_bounds__(GL_THREADS)
gae_allpairs_kernel(const float* __restrict__ z, int64_t ldz, int32_t n, int32_t row_begin, int32_t n_rows,
                    int32_t j_chunk, float coef, float* __restrict__ dz, double* __restrict__ loss_acc) {
  constexpr int GL_RPT = GaeCfg<D>::RPT, GL_ROWS = GaeCfg<D>::ROWS;
  __shared__ __align__(16) float zj[GL_JT][D];
  float2 zi[GL_RPT][D / 2], acc[GL_RPT][D / 2];   // feature pairs (d, d+1), two FMA chains each
  bool live[GL_RPT];
#pragma unroll
  for (int r = 0; r < GL_RPT; ++r) {
    const int i = blockIdx.x * GL_ROWS + r * GL_THREADS + threadIdx.x;   // local row
    live[r] = i < n_rows;
#pragma unroll
    for (int d = 0; d < D / 2; ++d) {
      zi[r][d] = live[r] ? make_float2(z[(int64_t)(row_begin + i) * ldz + 2 * d], z[(int64_t)(row_begin + i) * ldz + 2 * d + 1])
                         : make_float2(0.f, 0.f);
      acc[r][d] = make_float2(0.f, 0.f);
    }
  }
  const int j_begin = blockIdx.y * j_chunk;
  const int j_end = min(n, j_begin + j_chunk);
  double loss = 0.0;
  constexpr float LOG2E = 1.4426950408889634f, LN2 = 0.6931471805599453f;
  for (int j0 = j_begin; j0 < j_end; j0 += GL_JT) {
    const int cnt = min(GL_JT, j_end - j0);
    __syncthreads();
    for (int t = threadIdx.x; t < GL_JT * D / 4; t += GL_THREADS) {
      const int jj = t / (D / 4), q = t % (D / 4);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (jj < cnt) {
        const float* src = z + (int64_t)(j0 + jj) * ldz + 4 * q;
        v = make_float4(src[0], src[1], src[2], src[3]);
      }
      *reinterpret_cast<float4*>(&zj[jj][4 * q]) = v;
    }
    __syncthreads();
    // Σ_j log2(1+e_j) = log2 Π_j (1+e_j): each factor is in (1,2], so 32 of them stay far below FLT_MAX —
    // one MUFU.LG2 per 32 logits instead of one per logit.
    float relu_sum[GL_RPT], lg_sum[GL_RPT], prod[GL_RPT];
#pragma unroll
    for (int r = 0; r < GL_RPT; ++r) { relu_sum[r] = 0.f; lg_sum[r] = 0.f; prod[r] = 1.f; }
#pragma unroll 2
    for (int jj = 0; jj < cnt; ++jj) {
      if ((jj & 31) == 31) {
#pragma unroll
        for (int r = 0; r < GL_RPT; ++r) { lg_sum[r] += lg2_approx(prod[r]); prod[r] = 1.f; }
      }
      float2 zv[D / 2];
#pragma unroll
      for (int d = 0; d < D; d += 4) {
        const float4 v = *reinterpret_cast<const float4*>(&zj[jj][d]);
        zv[d / 2] = make_float2(v.x, v.y);
        zv[d / 2 + 1] = make_float2(v.z, v.w);
      }
#pragma unroll
      for (int r = 0; r < GL_RPT; ++r) {
        float2 xa = make_float2(0.f, 0.f), xb = make_float2(0.f, 0.f);   // two packed chains = 4 partial sums
#pragma unroll
        for (int d = 0; d < D / 2; d += 2) { xa = ffma2(zi[r][d], zv[d], xa); xb = ffma2(zi[r][d + 1], zv[d + 1], xb); }
        const float x = (xa.x + xa.y) + (xb.x + xb.y);
        const float e = ex2_approx(-fabsf(x) * LOG2E);
        const float inv = rcp_approx(1.f + e);
        const float sgm = x >= 0.f ? inv : e * inv;          // sigmoid(x)
        relu_sum[r] += fmaxf(x, 0.f);
        prod[r] *= (1.f + e);                                // softplus(x) = max(x,0) + ln2·log2(1+e)
        const float2 sg2 = make_float2(sgm, sgm);
#pragma unroll
        for (int d = 0; d < D / 2; ++d) acc[r][d] = ffma2(sg2, zv[d], acc[r][d]);
      }
    }
#pragma unroll
    for (int r = 0; r < GL_RPT; ++r)
      if (live[r]) loss += (double)(relu_sum[r] + LN2 * (lg_sum[r] + lg2_approx(prod[r])));
  }
  const float c2 = 2.f * coef;
#pragma unroll
  for (int r = 0; r < GL_RPT; ++r) {
    if (!live[r]) continue;
    const int64_t i = (int64_t)blockIdx.x * GL_ROWS + r * GL_THREADS + threadIdx.x;
    if (gridDim.y == 1) {
#pragma unroll
      for (int d = 0; d < D / 2; ++d) { dz[i * D + 2 * d] += c2 * acc[r][d].x; dz[i * D + 2 * d + 1] += c2 * acc[r][d].y; }
    } else {
#pragma unroll
      for (int d = 0; d < D / 2; ++d) { atomicAdd(dz + i * D + 2 * d, c2 * acc[r][d].x); atomicAdd(dz + i * D + 2 * d + 1, c2 * acc[r][d].y); }
    }
  }
  loss = warp_sum(loss);
  __shared__ double sred[GL_THREADS / 32];
  if ((threadIdx.x & 31) == 0) sred[threadIdx.x >> 5] = loss;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < GL_THREADS / 32; ++w) t += sred[w];
    atomicAdd(loss_acc, t * (double)coef);
  }
}

// edge (label) correction: one warp per row i, lanes stride over the row's entries
template <int D>
__global__ void __launch_bounds__(256)
gae_edges_kernel(const float* __restrict__ z, int64_t ldz, const int32_t* __restrict__ rowptr,
                 const int32_t* __restrict__ colidx, int32_t row_begin, int32_t n_rows, float coef, float pw, int use_pw,
                 float* __restrict__ dz, double* __restrict__ loss_acc) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  double loss = 0.0;
  for (int64_t i = warp; i < n_rows; i += nwarps) {
    float zi[D], acc[D];
#pragma unroll
    for (int d = 0; d < D; ++d) { zi[d] = __ldg(z + (row_begin + i) * ldz + d); acc[d] = 0.f; }
    const int32_t s = rowptr[i], e = rowptr[i + 1];
    for (int32_t p = s + lane; p < e; p += 32) {
      const int32_t j = colidx[p];
      float zjv[D];
      float x = 0.f;
#pragma unroll
      for (int d = 0; d < D; ++d) { zjv[d] = __ldg(z + (int64_t)j * ldz + d); x = fmaf(zi[d], zjv[d], x); }
      float hval, hgrad;
      if (use_pw) {
        const float sg = sigmoid_f(x);
        hval = pw * softplus_f(-x) - softplus_f(x);
        hgrad = -pw * (1.f - sg) - sg;
      } else {
        hval = -x;
        hgrad = -1.f;
      }
      loss += (double)hval;
#pragma unroll
      for (int d = 0; d < D; ++d) acc[d] = fmaf(hgrad, zjv[d], acc[d]);
    }
#pragma unroll
    for (int d = 0; d < D; ++d) acc[d] = warp_sum(acc[d]);
    if (lane == 0) {
      const float c2 = 2.f * coef;
#pragma unroll
      for (int d = 0; d < D; ++d) dz[i * D + d] += c2 * acc[d];
    }
  }
  loss = warp_sum(loss);
  if (lane == 0 && loss != 0.0) atomicAdd(loss_acc, loss * (double)coef);
}

// KLD = -0.5/n · mean_i Σ_d (1 + 2·lv - mu² - exp(lv)²)        (scgnn2.py:614)
__global__ void __launch_bounds__(256)
gae_kld_kernel(const float* __restrict__ mu, const float* __restrict__ logvar, int64_t ldm, int32_t n, int32_t n_rows,
               int32_t d, float* __restrict__ dmu, float* __restrict__ dlogvar, int64_t ldd, double* __restrict__ loss_acc) {
  const double c = -0.5 / ((double)n * (double)n);
  const float cf = (float)c;
  double local = 0.0;
  const int64_t total = (int64_t)n_rows * d;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / d;
    const int dd = (int)(t % d);
    const float m = mu[i * ldm + dd], lv = logvar[i * ldm + dd];
    const float ev = expf(lv);
    local += (double)(1.f + 2.f * lv - m * m - ev * ev);
    dmu[i * ldd + dd] = cf * (-2.f * m);
    dlogvar[i * ldd + dd] = cf * (2.f - 2.f * ev * ev);
  }
  local = warp_sum(local);
  if ((threadIdx.x & 31) == 0 && local != 0.0) atomicAdd(loss_acc, local * c);
}

__global__ void gae_finish_kernel(const double* acc, float* loss_out) { loss_out[0] = (float)acc[0]; }

namespace gtc {   // gae_tc.cu: wgmma version of the all-pairs part
size_t workspace_bytes(int32_t n);
int super_blocks(int32_t n);
bool eligible(int32_t n, int32_t d, int32_t n_rows);
int launch(const float* z, int64_t ldz, int32_t n, int32_t d, int32_t row_begin, int32_t n_rows, float coef, float* dz,
           double* loss_acc, void* ws, size_t ws_bytes, cudaStream_t st);
int launch_super_blocks(const float* z, int64_t ldz, int32_t n, int32_t d, int32_t sb_begin, int32_t sb_end, float coef, float* dz,
                        double* loss_acc, void* ws, size_t ws_bytes, cudaStream_t st);
}  // namespace gtc

template <int D>
static int launch_gae_edges(const float* z, int64_t ldz, const int32_t* rp, const int32_t* ci, int32_t row_begin, int32_t n_rows,
                            float coef, float pw, int use_pw, float* dz, double* acc, cudaStream_t st) {
  int64_t blocks = ceil_div<int64_t>(n_rows, 8);
  const int64_t cap = (int64_t)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  gae_edges_kernel<D><<<(unsigned)blocks, 256, 0, st>>>(z, ldz, rp, ci, row_begin, n_rows, coef, pw, use_pw, dz, acc);
  B2_CHECK_LAUNCH("gae_edges_kernel");
  return B2_OK;
}

template <int D>
static int launch_gae(const float* z, int64_t ldz, const int32_t* rp, const int32_t* ci, int32_t n, int32_t row_begin,
                      int32_t n_rows, float coef, float pw, int use_pw, float* dz, double* acc, bool skip_allpairs,
                      cudaStream_t st) {
  if (skip_allpairs) return launch_gae_edges<D>(z, ldz, rp, ci, row_begin, n_rows, coef, pw, use_pw, dz, acc, st);
  const int row_blocks = ceil_div(n_rows, GaeCfg<D>::ROWS);
  // split the j range so that small graphs still fill the machine
  int j_splits = 1;
  const int target = sm_count() * 4;
  if (row_blocks < target) j_splits = min(ceil_div(target, row_blocks), ceil_div(n, GL_JT));
  if (j_splits < 1) j_splits = 1;
  if (j_splits > 65535) j_splits = 65535;
  int j_chunk = ceil_div(ceil_div(n, j_splits), GL_JT) * GL_JT;
  j_splits = ceil_div(n, j_chunk);
  dim3 grid(row_blocks, j_splits);
  gae_allpairs_kernel<D><<<grid, GL_THREADS, 0, st>>>(z, ldz, n, row_begin, n_rows, j_chunk, coef, dz, acc);
  B2_CHECK_LAUNCH("gae_allpairs_kernel");
  return launch_gae_edges<D>(z, ldz, rp, ci, row_begin, n_rows, coef, pw, use_pw, dz, acc, st);
}

}  // namespace b2

using namespace b2;

extern "C" int b2_mse_sum_loss_grad_f32(const float* recon, const float* target, const float* ltmg_regu,
                                        float regu_strength, int relu_mask, float* grad, float* loss_out,
                                        int64_t n_elem, void* stream) {
  B2_REQUIRE(recon && target && grad && loss_out && n_elem >= 0, "b2_mse_sum_loss_grad_f32: bad arguments");
  if (n_elem == 0) return B2_OK;
  cudaStream_t st = as_stream(stream);
  int64_t blocks = ceil_div<int64_t>(n_elem, 256 * 8);
  const int64_t cap = (int64_t)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  mse_loss_grad_kernel<<<(unsigned)blocks, 256, 0, st>>>(recon, target, ltmg_regu, regu_strength, relu_mask, grad,
                                                         loss_out, n_elem);
  B2_CHECK_LAUNCH("mse_loss_grad_kernel");
  return B2_OK;
}

extern "C" size_t b2_gae_loss_workspace_bytes(int32_t n, int32_t d) {
  // 256 B of accumulators + the hi/lo tf32 planes of z for the tensor-core path
  return 256 + (d <= 32 ? gtc::workspace_bytes(n) : 0);
}

extern "C" int b2_gae_loss_grad_f32(const float* z, int64_t ldz, const float* mu, const float* logvar, int64_t ldm,
                                    const int32_t* lab_rowptr, const int32_t* lab_colidx, int32_t n, int32_t d,
                                    int32_t row_begin, int32_t n_rows, float norm, float pos_weight, int use_pos_weight, float* dz, float* dmu,
                                    float* dlogvar, int64_t ldd, float* loss_out, void* workspace,
                                    size_t workspace_bytes, void* stream) {
  B2_REQUIRE(z && lab_rowptr && lab_colidx && dz && loss_out, "b2_gae_loss_grad_f32: null pointer");
  B2_REQUIRE(n > 0 && d > 0 && ldz >= d, "b2_gae_loss_grad_f32: bad shape");
  B2_REQUIRE(row_begin >= 0 && n_rows >= 0 && row_begin + n_rows <= n, "b2_gae_loss_grad_f32: bad row range");
  B2_REQUIRE(workspace && workspace_bytes >= 256, "b2_gae_loss_grad_f32: workspace too small");
  B2_REQUIRE((mu == nullptr) == (logvar == nullptr), "b2_gae_loss_grad_f32: mu/logvar must both be given or both NULL");
  if (mu) B2_REQUIRE(dmu && dlogvar && ldm >= d && ldd >= d, "b2_gae_loss_grad_f32: dmu/dlogvar required with mu/logvar");
  cudaStream_t st = as_stream(stream);
  double* acc = reinterpret_cast<double*>(workspace);
  B2_CHECK_CUDA(cudaMemsetAsync(acc, 0, sizeof(double), st));
  B2_CHECK_CUDA(cudaMemsetAsync(dz, 0, sizeof(float) * (size_t)n_rows * d, st));
  const float coef = (use_pos_weight ? norm : 1.f) / ((float)n * (float)n);
  int rc;
  // large problems: the all-pairs part runs on the tensor cores (gae_tc.cu); the CUDA-core kernel serves small graphs
  bool tc_done = false;
  if (gtc::eligible(n, d, n_rows) && workspace_bytes >= 256 + gtc::workspace_bytes(n)) {
    rc = gtc::launch(z, ldz, n, d, row_begin, n_rows, coef, dz, acc, reinterpret_cast<char*>(workspace) + 256, workspace_bytes - 256, st);
    if (rc == B2_OK) tc_done = true;
    else if (rc != B2_ERR_UNSUPPORTED) return rc;
  }
  switch (d) {
    case 8: rc = launch_gae<8>(z, ldz, lab_rowptr, lab_colidx, n, row_begin, n_rows, coef, pos_weight, use_pos_weight, dz, acc, tc_done, st); break;
    case 16: rc = launch_gae<16>(z, ldz, lab_rowptr, lab_colidx, n, row_begin, n_rows, coef, pos_weight, use_pos_weight, dz, acc, tc_done, st); break;
    case 32: rc = launch_gae<32>(z, ldz, lab_rowptr, lab_colidx, n, row_begin, n_rows, coef, pos_weight, use_pos_weight, dz, acc, tc_done, st); break;
    case 64: rc = launch_gae<64>(z, ldz, lab_rowptr, lab_colidx, n, row_begin, n_rows, coef, pos_weight, use_pos_weight, dz, acc, tc_done, st); break;
    default:
      set_error("b2_gae_loss_grad_f32: embedding size %d unsupported (8, 16, 32, 64)", d);
      return B2_ERR_UNSUPPORTED;
  }
  if (rc != B2_OK) return rc;
  if (mu) {
    int64_t blocks = ceil_div<int64_t>((int64_t)n_rows * d, 256);
    if (blocks < 1) blocks = 1;
    const int64_t cap = (int64_t)sm_count() * 16;
    if (blocks > cap) blocks = cap;
    gae_kld_kernel<<<(unsigned)blocks, 256, 0, st>>>(mu, logvar, ldm, n, n_rows, d, dmu, dlogvar, ldd, acc);
    B2_CHECK_LAUNCH("gae_kld_kernel");
  }
  gae_finish_kernel<<<1, 1, 0, st>>>(acc, loss_out);
  B2_CHECK_LAUNCH("gae_finish_kernel");
  return B2_OK;
}


// Pair-sharded form of b2_gae_loss_grad_f32 for multi-GPU runs.  Rank r evaluates the all-pairs part of the super-blocks
// [sb_begin, sb_end) (b2_gae_sym_super_blocks(n) in total, equal work each: super-block s = the 128-row blocks s and nb−1−s)
// plus the label / KLD terms of its own rows [row_begin, row_begin + n_rows):
//   dz_full [n, d]  : zero-filled here, receives this rank's all-pairs contributions (the rows of its super-blocks) and the label
//                     terms of its own rows — the caller sums dz_full over ranks (all-reduce) and keeps its rows;
//   loss_out        : this rank's share of the loss (sum over ranks = the loss).
extern "C" int b2_gae_sym_super_blocks(int32_t n) { return b2::gtc::super_blocks(n); }

extern "C" int b2_gae_loss_grad_sym_f32(const float* z, int64_t ldz, const float* mu, const float* logvar, int64_t ldm,
                                        const int32_t* lab_rowptr, const int32_t* lab_colidx, int32_t n, int32_t d,
                                        int32_t sb_begin, int32_t sb_end, int32_t row_begin, int32_t n_rows, float norm, float pos_weight,
                                        int use_pos_weight, float* dz_full, float* dmu, float* dlogvar, int64_t ldd, float* loss_out,
                                        void* workspace, size_t workspace_bytes, void* stream) {
  B2_REQUIRE(z && lab_rowptr && lab_colidx && dz_full && loss_out, "b2_gae_loss_grad_sym_f32: null pointer");
  B2_REQUIRE(n > 0 && d > 0 && d <= 16 && ldz >= d, "b2_gae_loss_grad_sym_f32: bad shape (d <= 16)");
  B2_REQUIRE(row_begin >= 0 && n_rows >= 0 && row_begin + n_rows <= n, "b2_gae_loss_grad_sym_f32: bad row range");
  B2_REQUIRE(sb_begin >= 0 && sb_begin <= sb_end && sb_end <= gtc::super_blocks(n), "b2_gae_loss_grad_sym_f32: bad super-block range");
  B2_REQUIRE(workspace && workspace_bytes >= 256 + gtc::workspace_bytes(n), "b2_gae_loss_grad_sym_f32: workspace too small");
  B2_REQUIRE((mu == nullptr) == (logvar == nullptr), "b2_gae_loss_grad_sym_f32: mu/logvar must both be given or both NULL");
  if (mu) B2_REQUIRE(dmu && dlogvar && ldm >= d && ldd >= d, "b2_gae_loss_grad_sym_f32: dmu/dlogvar required with mu/logvar");
  cudaStream_t st = as_stream(stream);
  double* acc = reinterpret_cast<double*>(workspace);
  B2_CHECK_CUDA(cudaMemsetAsync(acc, 0, sizeof(double), st));
  B2_CHECK_CUDA(cudaMemsetAsync(dz_full, 0, sizeof(float) * (size_t)n * d, st));
  const float coef = (use_pos_weight ? norm : 1.f) / ((float)n * (float)n);
  int rc = gtc::launch_super_blocks(z, ldz, n, d, sb_begin, sb_end, coef, dz_full, acc, reinterpret_cast<char*>(workspace) + 256,
                                    workspace_bytes - 256, st);
  if (rc != B2_OK) {
    if (rc == B2_ERR_UNSUPPORTED) set_error("b2_gae_loss_grad_sym_f32: workspace too small");
    return rc;
  }
  float* dz_rows = dz_full + (size_t)row_begin * d;
  switch (d) {
    case 8: rc = launch_gae<8>(z, ldz, lab_rowptr, lab_colidx, n, row_begin, n_rows, coef, pos_weight, use_pos_weight, dz_rows, acc, true, st); break;
    case 16: rc = launch_gae<16>(z, ldz, lab_rowptr, lab_colidx, n, row_begin, n_rows, coef, pos_weight, use_pos_weight, dz_rows, acc, true, st); break;
    default:
      set_error("b2_gae_loss_grad_sym_f32: embedding size %d unsupported (8, 16)", d);
      return B2_ERR_UNSUPPORTED;
  }
  if (rc != B2_OK) return rc;
  if (mu) {
    int64_t blocks = ceil_div<int64_t>((int64_t)n_rows * d, 256);
    if (blocks < 1) blocks = 1;
    const int64_t cap = (int64_t)sm_count() * 16;
    if (blocks > cap) blocks = cap;
    gae_kld_kernel<<<(unsigned)blocks, 256, 0, st>>>(mu, logvar, ldm, n, n_rows, d, dmu, dlogvar, ldd, acc);
    B2_CHECK_LAUNCH("gae_kld_kernel");
  }
  gae_finish_kernel<<<1, 1, 0, st>>>(acc, loss_out);
  B2_CHECK_LAUNCH("gae_finish_kernel");
  return B2_OK;
}
