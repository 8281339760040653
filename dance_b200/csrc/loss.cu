// Loss kernels of the scGNN path: value + gradient in one pass.
//   - Feature-AE reconstruction loss  (reference scgnn2.py:1298-1328)
//   - Graph-AE inner-product-decoder BCE + KLD, matrix-free
//     (reference scgnn2.py:423-426, 603-619): the N×N logits z zᵀ and the
//     dense label matrix (scgnn2.py:557) are never materialised.  Labels are unit and symmetric (A + I), or real-valued and
//     asymmetric (W + I of graph_AE_retain_weights, scgnn2.py:659-670), then walked as L and as Lᵀ.
#include "common.cuh"

#include <type_traits>

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

// Label correction (graph_AE_retain_weights: real-valued, asymmetric labels y, scgnn2.py:555-569, 603-619).
// Per entry ℓ = (1−y)·softplus(x) + y·(y·pw)·softplus(−x)  (pos_weight = labels·pw), so over the label pattern
//   h(x, y) = y²·pw·softplus(−x) − y·softplus(x),   h' = −y²·pw·σ(−x) − y·σ(x)     (pos-weighted BCE)
//   h(x, y) = −y·x,                                 h' = −y                        (plain BCE)
// x_ij = x_ji, so dS/dz_i = 2·Σ_j σ(x_ij) z_j + Σ_{j∈L_i} h'(x_ij, y_ij) z_j + Σ_{j∈Lᵀ_i} h'(x_ij, y_ji) z_j:
// row i of L (entries (i, j), values y_ij) gives the loss and the first sum, row i of Lᵀ (entries (j, i), values y_ji) the
// second.  Unit labels (!WEIGHTED, y = 1) have L = Lᵀ: one pass over row i of L with the label sum doubled.
// One warp per row, lanes stride over the row's entries.
__device__ __forceinline__ void gae_label_terms(float x, float y, float pw, int use_pw, float& hval, float& hgrad) {
  if (use_pw) {
    const float sg = sigmoid_f(x), ypw = y * y * pw;
    hval = ypw * softplus_f(-x) - y * softplus_f(x);
    hgrad = -ypw * (1.f - sg) - y * sg;
  } else {
    hval = -y * x;
    hgrad = -y;
  }
}

template <int D, bool WEIGHTED>
__global__ void __launch_bounds__(256)
gae_edges_weighted_kernel(const float* __restrict__ z, int64_t ldz, const int32_t* __restrict__ rowptr,
                          const int32_t* __restrict__ colidx, const float* __restrict__ y, const int32_t* __restrict__ t_rowptr,
                          const int32_t* __restrict__ t_colidx, const float* __restrict__ t_y, int32_t row_begin, int32_t n_rows,
                          float coef, float pw, int use_pw, float* __restrict__ dz, double* __restrict__ loss_acc) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  double loss = 0.0;
  for (int64_t i = warp; i < n_rows; i += nwarps) {
    float zi[D], acc[D];
#pragma unroll
    for (int d = 0; d < D; ++d) { zi[d] = __ldg(z + (row_begin + i) * ldz + d); acc[d] = 0.f; }
#pragma unroll 1
    for (int pass = 0; pass < (WEIGHTED ? 2 : 1); ++pass) {   // pass 0: row i of L (loss + gradient), pass 1: row i of Lᵀ (gradient)
      const int32_t* rp = pass ? t_rowptr : rowptr;
      const int32_t* ci = pass ? t_colidx : colidx;
      const float* yv = pass ? t_y : y;
      const int32_t s = rp[i], e = rp[i + 1];
      for (int32_t p = s + lane; p < e; p += 32) {
        const int32_t j = ci[p];
        float zjv[D];
        float x = 0.f;
#pragma unroll
        for (int d = 0; d < D; ++d) { zjv[d] = __ldg(z + (int64_t)j * ldz + d); x = fmaf(zi[d], zjv[d], x); }
        float hval, hgrad;
        gae_label_terms(x, WEIGHTED ? yv[p] : 1.f, pw, use_pw, hval, hgrad);
        if (pass == 0) loss += (double)hval;
#pragma unroll
        for (int d = 0; d < D; ++d) acc[d] = fmaf(hgrad, zjv[d], acc[d]);
      }
    }
#pragma unroll
    for (int d = 0; d < D; ++d) acc[d] = warp_sum(acc[d]);
    if (lane == 0) {
      const float c = WEIGHTED ? coef : 2.f * coef;
#pragma unroll
      for (int d = 0; d < D; ++d) dz[i * D + d] += c * acc[d];
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
bool eligible(int32_t n, int32_t d, int32_t n_rows, size_t ws_bytes);
int launch(const float* z, int64_t ldz, int32_t n, int32_t d, bool sym, int32_t begin, int32_t end, float coef, float* dz,
           double* loss_acc, void* ws, cudaStream_t st);
}  // namespace gtc

// The workspace starts with the loss accumulator; the tensor-core path's planes of z follow it.
constexpr size_t GAE_ACC_BYTES = 256;

// The embedding sizes the CUDA-core kernels are built for: f(std::integral_constant<int, D>()).  The caller has checked d.
template <class F>
static int with_d(int32_t d, F f) {
  switch (d) {
    case 8: return f(std::integral_constant<int, 8>());
    case 16: return f(std::integral_constant<int, 16>());
    case 32: return f(std::integral_constant<int, 32>());
    default: return f(std::integral_constant<int, 64>());
  }
}

template <int D>
static int launch_gae_allpairs(const float* z, int64_t ldz, int32_t n, int32_t row_begin, int32_t n_rows, float coef, float* dz,
                               double* acc, cudaStream_t st) {
  if (n_rows == 0) return B2_OK;   // nothing to sweep, and no row blocks to spread the j range over
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
  return B2_OK;
}

// The label matrix of a call: the local rows of L, with unit entries when vals is NULL (then L must be symmetric and the
// transposed rows are not read), else with their values and the local rows of Lᵀ with theirs.
struct Labels {
  const int32_t *rowptr, *colidx;
  const float* vals;
  const int32_t *t_rowptr, *t_colidx;
  const float* t_vals;
};

template <int D>
static int launch_gae_edges(const float* z, int64_t ldz, const Labels& lab, int32_t row_begin, int32_t n_rows, float coef, float pw,
                            int use_pw, float* dz, double* acc, cudaStream_t st) {
  const auto kernel = lab.vals ? gae_edges_weighted_kernel<D, true> : gae_edges_weighted_kernel<D, false>;
  kernel<<<grid_blocks(n_rows, 8), 256, 0, st>>>(z, ldz, lab.rowptr, lab.colidx, lab.vals, lab.t_rowptr, lab.t_colidx, lab.t_vals,
                                                 row_begin, n_rows, coef, pw, use_pw, dz, acc);
  B2_CHECK_LAUNCH("gae_edges_weighted_kernel");
  return B2_OK;
}

// The all-pairs part of a call.  Row form: rows [row_begin, row_begin + n_rows) against every column, dz holds those rows.
// Pair-sharded form (sym): super-blocks [sb_begin, sb_end) on the tensor cores, dz holds all n rows.
struct AllPairs {
  bool sym;
  int32_t sb_begin, sb_end;
};

// Every decoder entry point; fn names the one called in error messages.
static int gae_loss_grad(const char* fn, const AllPairs& ap, const float* z, int64_t ldz, const float* mu, const float* logvar,
                         int64_t ldm, const Labels& lab, int32_t n, int32_t d, int32_t row_begin,
                         int32_t n_rows, float norm, float pos_weight, int use_pos_weight, float* dz, float* dmu, float* dlogvar,
                         int64_t ldd, float* loss_out, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  B2_REQUIRE(z && lab.rowptr && lab.colidx && dz && loss_out, "%s: null pointer", fn);
  if (lab.vals)
    B2_REQUIRE(lab.t_rowptr && lab.t_colidx && lab.t_vals, "%s: null pointer (label values need the transposed labels)", fn);
  B2_REQUIRE(n > 0 && d > 0 && ldz >= d, "%s: bad shape", fn);
  B2_REQUIRE(row_begin >= 0 && n_rows >= 0 && row_begin + n_rows <= n, "%s: bad row range", fn);
  B2_REQUIRE((mu == nullptr) == (logvar == nullptr), "%s: mu/logvar must both be given or both NULL", fn);
  if (mu) B2_REQUIRE(dmu && dlogvar && ldm >= d && ldd >= d, "%s: dmu/dlogvar required with mu/logvar", fn);
  if (ap.sym) {
    B2_REQUIRE(d <= 16, "%s: bad shape (d <= 16)", fn);
    B2_REQUIRE(ap.sb_begin >= 0 && ap.sb_begin <= ap.sb_end && ap.sb_end <= gtc::super_blocks(n), "%s: bad super-block range", fn);
  }
  B2_REQUIRE(workspace && workspace_bytes >= GAE_ACC_BYTES + (ap.sym ? gtc::workspace_bytes(n) : 0), "%s: workspace too small", fn);
  if (d != 8 && d != 16 && d != 32 && d != 64) {
    set_error("%s: embedding size %d unsupported (%s)", fn, d, ap.sym ? "8, 16" : "8, 16, 32, 64");
    return B2_ERR_UNSUPPORTED;
  }

  double* acc = reinterpret_cast<double*>(workspace);
  void* tc_ws = reinterpret_cast<char*>(workspace) + GAE_ACC_BYTES;
  float* dz_rows = ap.sym ? dz + (size_t)row_begin * d : dz;   // where this call's label terms go
  B2_CHECK_CUDA(cudaMemsetAsync(acc, 0, sizeof(double), st));
  B2_CHECK_CUDA(cudaMemsetAsync(dz, 0, sizeof(float) * (size_t)(ap.sym ? n : n_rows) * d, st));
  const float coef = (use_pos_weight ? norm : 1.f) / ((float)n * (float)n);
  // the all-pairs part: the pair-sharded form and large problems on the tensor cores (gae_tc.cu), small graphs on the CUDA cores
  int rc;
  if (ap.sym)
    rc = gtc::launch(z, ldz, n, d, true, ap.sb_begin, ap.sb_end, coef, dz, acc, tc_ws, st);
  else if (gtc::eligible(n, d, n_rows, workspace_bytes - GAE_ACC_BYTES))
    rc = gtc::launch(z, ldz, n, d, false, row_begin, row_begin + n_rows, coef, dz, acc, tc_ws, st);
  else
    rc = with_d(d, [&](auto D) { return launch_gae_allpairs<D>(z, ldz, n, row_begin, n_rows, coef, dz, acc, st); });
  if (rc != B2_OK) return rc;
  rc = with_d(d, [&](auto D) {
    return launch_gae_edges<D>(z, ldz, lab, row_begin, n_rows, coef, pos_weight, use_pos_weight, dz_rows, acc, st);
  });
  if (rc != B2_OK) return rc;
  if (mu) {
    gae_kld_kernel<<<grid_blocks((int64_t)n_rows * d, 256), 256, 0, st>>>(mu, logvar, ldm, n, n_rows, d, dmu, dlogvar, ldd, acc);
    B2_CHECK_LAUNCH("gae_kld_kernel");
  }
  gae_finish_kernel<<<1, 1, 0, st>>>(acc, loss_out);
  B2_CHECK_LAUNCH("gae_finish_kernel");
  return B2_OK;
}

}  // namespace b2

using namespace b2;

extern "C" int b2_mse_sum_loss_grad_f32(const float* recon, const float* target, const float* ltmg_regu,
                                        float regu_strength, int relu_mask, float* grad, float* loss_out,
                                        int64_t n_elem, void* stream) {
  B2_REQUIRE(recon && target && grad && loss_out && n_elem >= 0, "b2_mse_sum_loss_grad_f32: bad arguments");
  if (n_elem == 0) return B2_OK;
  cudaStream_t st = as_stream(stream);
  mse_loss_grad_kernel<<<grid_blocks(n_elem, 2048), 256, 0, st>>>(recon, target, ltmg_regu, regu_strength, relu_mask, grad,
                                                                  loss_out, n_elem);
  B2_CHECK_LAUNCH("mse_loss_grad_kernel");
  return B2_OK;
}

extern "C" size_t b2_gae_loss_workspace_bytes(int32_t n, int32_t d) {
  return GAE_ACC_BYTES + (d <= 32 ? gtc::workspace_bytes(n) : 0);
}

extern "C" int b2_gae_loss_grad_f32(const float* z, int64_t ldz, const float* mu, const float* logvar, int64_t ldm,
                                    const int32_t* lab_rowptr, const int32_t* lab_colidx, const float* lab_vals,
                                    const int32_t* labt_rowptr, const int32_t* labt_colidx, const float* labt_vals, int32_t n, int32_t d,
                                    int32_t row_begin, int32_t n_rows, float norm, float pos_weight, int use_pos_weight, float* dz,
                                    float* dmu, float* dlogvar, int64_t ldd, float* loss_out, void* workspace, size_t workspace_bytes,
                                    void* stream) {
  return gae_loss_grad("b2_gae_loss_grad_f32", AllPairs{false, 0, 0}, z, ldz, mu, logvar, ldm,
                       Labels{lab_rowptr, lab_colidx, lab_vals, labt_rowptr, labt_colidx, labt_vals}, n, d, row_begin, n_rows, norm,
                       pos_weight, use_pos_weight, dz, dmu, dlogvar, ldd, loss_out, workspace, workspace_bytes, as_stream(stream));
}

// Pair-sharded form of b2_gae_loss_grad_f32 for multi-GPU runs.  Rank r evaluates the all-pairs part of the super-blocks
// [sb_begin, sb_end) (b2_gae_sym_super_blocks(n) in total, equal work each: super-block s = the 128-row blocks s and nb−1−s)
// plus the label / KLD terms of its own rows [row_begin, row_begin + n_rows):
//   dz_full [n, d]  : zero-filled here, receives this rank's all-pairs contributions (the rows of its super-blocks) and the label
//                     terms of its own rows — the caller sums dz_full over ranks (all-reduce) and keeps its rows;
//   loss_out        : this rank's share of the loss (sum over ranks = the loss).
extern "C" int b2_gae_sym_super_blocks(int32_t n) { return b2::gtc::super_blocks(n); }

extern "C" int b2_gae_loss_grad_sym_f32(const float* z, int64_t ldz, const float* mu, const float* logvar, int64_t ldm,
                                        const int32_t* lab_rowptr, const int32_t* lab_colidx, const float* lab_vals,
                                        const int32_t* labt_rowptr, const int32_t* labt_colidx, const float* labt_vals, int32_t n,
                                        int32_t d, int32_t sb_begin, int32_t sb_end, int32_t row_begin, int32_t n_rows, float norm,
                                        float pos_weight, int use_pos_weight, float* dz_full, float* dmu, float* dlogvar, int64_t ldd,
                                        float* loss_out, void* workspace, size_t workspace_bytes, void* stream) {
  return gae_loss_grad("b2_gae_loss_grad_sym_f32", AllPairs{true, sb_begin, sb_end}, z, ldz, mu, logvar, ldm,
                       Labels{lab_rowptr, lab_colidx, lab_vals, labt_rowptr, labt_colidx, labt_vals}, n, d, row_begin, n_rows, norm,
                       pos_weight, use_pos_weight, dz_full, dmu, dlogvar, ldd, loss_out, workspace, workspace_bytes, as_stream(stream));
}
