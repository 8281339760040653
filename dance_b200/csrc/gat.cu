// Graph attention (GAT) message passing: fused edge score + neighbourhood softmax + aggregate,
// forward and backward, on a CSR indexed by TARGET node (row v lists the sources u of its in-edges).
//
// Replaces, in the reference:
//   scGNN GATLayer.forward           scgnn2.py:989-1051 (lift :1163-1174, neighborhood_aware_softmax
//                                    :1057-1095 — note the GLOBAL max shift :1076, scatter_add aggregate
//                                    :1116-1131, skip/concat/bias :1189-1215)
//   STAGATE GATConv.forward/message  stagate.py:61-125 (sigmoid scores, PyG per-target softmax)
// The E×NH×F "lifted" temporaries of the reference are never materialised: each target row streams its
// in-edges once (twice when the attention coefficients are kept for the backward pass).
//
// Attention dropout (GATLayer's third dropout site, scgnn2.py:1029: α' = drop(α) after the softmax) is a compile-time
// parameter of the aggregate and of both backward sweeps (DROP = false is the plain GAT).  The keep bit of (edge, head) is
// dropout_keep(seed, key, p, h) with p the edge's position in the target CSR: nothing is stored, the backward regenerates
// it, and alpha_out keeps the UNDROPPED α.  Per 32 edges each lane draws one edge's bits, shared by ballot / shuffle.
#include "common.cuh"

#include <math_constants.h>

namespace b2 {

__device__ __forceinline__ float score_act_f(float x, int act, float slope) {
  return act == 0 ? (x > 0.f ? x : slope * x) : 1.f / (1.f + expf(-x));
}
__device__ __forceinline__ float score_act_grad(float pre, int act, float slope) {
  if (act == 0) return pre > 0.f ? 1.f : slope;
  const float s = 1.f / (1.f + expf(-pre));
  return s * (1.f - s);
}

// s_src[n,h] = <H[n,h,:], a_src[h,:]>, s_trg likewise.  One warp per node.
__global__ void __launch_bounds__(256)
gat_scores_kernel(const float* __restrict__ H, int64_t ldh, const float* __restrict__ a_src,
                  const float* __restrict__ a_trg, int32_t n, int32_t nh, int32_t F, float* __restrict__ s_src,
                  float* __restrict__ s_trg) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = warp; i < n; i += nwarps) {
    for (int h = 0; h < nh; ++h) {
      float ps = 0.f, pt = 0.f;
      for (int f = lane; f < F; f += 32) {
        const float v = H[i * ldh + h * F + f];
        ps = fmaf(v, a_src[h * F + f], ps);
        pt = fmaf(v, a_trg[h * F + f], pt);
      }
      ps = warp_sum(ps);
      pt = warp_sum(pt);
      if (lane == 0) { s_src[i * nh + h] = ps; s_trg[i * nh + h] = pt; }
    }
  }
}

__device__ __forceinline__ void atomic_max_float(float* addr, float v) {
  // total order on floats via signed/unsigned integer views, chosen by the sign BIT: -0.0 compares >= 0 but its int view is
  // INT_MIN, which would never replace the initial -inf under the signed max
  if (!signbit(v)) atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
  else atomicMin(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}

__global__ void set_neg_inf_kernel(float* p) { *p = -CUDART_INF_F; }

// Attention-dropout parameters: keep with probability 1 - p, kept coefficients scaled by `scale` = 1 / (1 - p).
struct AttnDrop {
  float p, scale;
  uint32_t seed, key;
};

// keep bits of edge `pos` for heads 0..nh-1 (nh <= 32), bit h = head h
__device__ __forceinline__ uint32_t edge_keep_bits(const AttnDrop& dr, int32_t pos, int32_t nh) {
  uint32_t kb = 0;
  for (int h = 0; h < nh; ++h) kb |= (uint32_t)dropout_keep(dr.seed, dr.key, (uint32_t)pos, (uint32_t)h, dr.p) << h;
  return kb;
}

// scores_per_edge.max() over every edge and head (scgnn2.py:1076)
__global__ void __launch_bounds__(256)
gat_edge_max_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx,
                    const float* __restrict__ s_src, const float* __restrict__ s_trg, int32_t n, int32_t nh, int act,
                    float slope, float* __restrict__ gmax) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  float m = -CUDART_INF_F;
  for (int64_t v = warp; v < n; v += nwarps) {
    const int32_t s = rowptr[v], e = rowptr[v + 1];
    for (int32_t p = s + lane; p < e; p += 32) {
      const int32_t u = colidx[p];
      for (int h = 0; h < nh; ++h) m = fmaxf(m, score_act_f(s_src[(int64_t)u * nh + h] + s_trg[v * nh + h], act, slope));
    }
  }
  m = warp_max(m);
  if (lane == 0 && m > -CUDART_INF_F) atomic_max_float(gmax, m);
}

// Forward aggregate.  One warp per target row; lanes stride over the NH·F row of H.
//   p_e,h = exp(act(s_src[u,h] + s_trg[v,h]) - shift_h) ; α = p / (Σp + 1e-16) ; out[v] = Σ α H[u]
// DROP: out[v] = Σ keep_e α_e scale H[u]; a dropped edge is not gathered.
template <bool DROP>
__global__ void __launch_bounds__(256)
gat_aggregate_fwd_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx,
                         const float* __restrict__ H, int64_t ldh, const float* __restrict__ s_src,
                         const float* __restrict__ s_trg, int32_t n, int32_t nh, int32_t F, int act, float slope,
                         int shift_mode, const float* __restrict__ gmax, float* __restrict__ out, int64_t ldo,
                         float* __restrict__ alpha_out, AttnDrop dr) {
  constexpr int MAXV = 16;  // NH*F <= 32*16 = 512 floats per row
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int W = nh * F;
  const float gshift = shift_mode == 0 ? *gmax : 0.f;
  if ((F & 31) == 0) {
    // Wide heads (F a multiple of 32, e.g. STAGATE's 1×512): every lane of a t-slot belongs to the same head, so the edge
    // coefficient is computed ONCE per (edge, head) instead of once per (edge, 32-column slot) — the exponentials, not the
    // gather, dominated the first version of this kernel.
    const int tper = F >> 5;
    for (int64_t v = warp; v < n; v += nwarps) {
      const int32_t s = rowptr[v], e = rowptr[v + 1];
      float acc[MAXV];
#pragma unroll
      for (int t = 0; t < MAXV; ++t) acc[t] = 0.f;
      for (int h = 0; h < nh; ++h) {
        const float st = s_trg[v * nh + h];
        float sh = gshift;
        if (shift_mode == 1) {
          float m = -CUDART_INF_F;
          for (int32_t p = s + lane; p < e; p += 32) m = fmaxf(m, score_act_f(s_src[(int64_t)colidx[p] * nh + h] + st, act, slope));
          m = warp_max(m);
          sh = (e > s) ? m : 0.f;
        }
        float den = 0.f;
        const int t0 = h * tper, t1 = t0 + tper;
        uint32_t kmask = 0;  // DROP: bit j = keep bit of edge (p - s) rounded down to 32, + j
        for (int32_t p = s; p < e; ++p) {
          if constexpr (DROP) {
            if (((p - s) & 31) == 0)
              kmask = __ballot_sync(0xffffffffu, p + lane < e && dropout_keep(dr.seed, dr.key, (uint32_t)(p + lane), (uint32_t)h, dr.p));
          }
          const int32_t u = colidx[p];
          const float pe = expf(score_act_f(s_src[(int64_t)u * nh + h] + st, act, slope) - sh);
          den += pe;
          if (DROP && !((kmask >> ((p - s) & 31)) & 1u)) continue;
          const float* hu = H + (int64_t)u * ldh + lane;
#pragma unroll
          for (int t = 0; t < MAXV; ++t)
            if (t >= t0 && t < t1) acc[t] = fmaf(pe, hu[32 * t], acc[t]);
        }
        const float inv = DROP ? dr.scale / (den + 1e-16f) : 1.f / (den + 1e-16f);
#pragma unroll
        for (int t = 0; t < MAXV; ++t)
          if (t >= t0 && t < t1) out[v * ldo + lane + 32 * t] = acc[t] * inv;
        if (alpha_out) {
          const float ainv = DROP ? 1.f / (den + 1e-16f) : inv;   // α is stored undropped
          for (int32_t p = s + lane; p < e; p += 32)
            alpha_out[(int64_t)p * nh + h] = expf(score_act_f(s_src[(int64_t)colidx[p] * nh + h] + st, act, slope) - sh) * ainv;
        }
      }
    }
    return;
  }
  for (int64_t v = warp; v < n; v += nwarps) {
    const int32_t s = rowptr[v], e = rowptr[v + 1];
    float acc[MAXV], den[MAXV], shift[MAXV];
#pragma unroll
    for (int t = 0; t < MAXV; ++t) { acc[t] = 0.f; den[t] = 0.f; shift[t] = gshift; }
    if (shift_mode == 1) {
      // per-target max (PyG softmax): one extra sweep over the in-edges
#pragma unroll
      for (int t = 0; t < MAXV; ++t) {
        const int c = lane + 32 * t;
        if (c < W) {
          const int h = c / F;
          float m = -CUDART_INF_F;
          for (int32_t p = s; p < e; ++p)
            m = fmaxf(m, score_act_f(s_src[(int64_t)colidx[p] * nh + h] + s_trg[v * nh + h], act, slope));
          shift[t] = (e > s) ? m : 0.f;
        }
      }
    }
    uint32_t kb = 0;  // DROP: lane j holds the keep bits (one per head) of edge (p - s) rounded down to 32, + j
    for (int32_t p = s; p < e; ++p) {
      uint32_t bits = 0;
      if constexpr (DROP) {
        if (((p - s) & 31) == 0) kb = p + lane < e ? edge_keep_bits(dr, p + lane, nh) : 0u;
        bits = __shfl_sync(0xffffffffu, kb, (p - s) & 31);
      }
      const int32_t u = colidx[p];
#pragma unroll
      for (int t = 0; t < MAXV; ++t) {
        const int c = lane + 32 * t;
        if (c < W) {
          const int h = c / F;
          const float pe = expf(score_act_f(s_src[(int64_t)u * nh + h] + s_trg[v * nh + h], act, slope) - shift[t]);
          den[t] += pe;
          if (!DROP || ((bits >> h) & 1u)) acc[t] = fmaf(pe, H[(int64_t)u * ldh + c], acc[t]);
        }
      }
    }
#pragma unroll
    for (int t = 0; t < MAXV; ++t) {
      const int c = lane + 32 * t;
      if (c < W) out[v * ldo + c] = DROP ? acc[t] / (den[t] + 1e-16f) * dr.scale : acc[t] / (den[t] + 1e-16f);
    }
    if (alpha_out) {
      // attention coefficients per (edge, head) for the backward pass: lanes own heads
      for (int h = lane; h < nh; h += 32) {
        float sh = gshift, d = 0.f;
        if (shift_mode == 1) {
          float m = -CUDART_INF_F;
          for (int32_t p = s; p < e; ++p)
            m = fmaxf(m, score_act_f(s_src[(int64_t)colidx[p] * nh + h] + s_trg[v * nh + h], act, slope));
          sh = (e > s) ? m : 0.f;
        }
        for (int32_t p = s; p < e; ++p)
          d += expf(score_act_f(s_src[(int64_t)colidx[p] * nh + h] + s_trg[v * nh + h], act, slope) - sh);
        for (int32_t p = s; p < e; ++p)
          alpha_out[(int64_t)p * nh + h] =
              expf(score_act_f(s_src[(int64_t)colidx[p] * nh + h] + s_trg[v * nh + h], act, slope) - sh) / (d + 1e-16f);
      }
    }
  }
}

// Backward, part 1 (by target): dα_e,h = <dOut[v,h,:], H[u,h,:]> ; dscore = α (dα - Σ α dα) ;
// dpre = dscore · act'(pre) → dpre_edge[p,h] ; ds_trg[v,h] = Σ_e dpre.
// With a global shift c (gmax != NULL) the softmax is shift-invariant only up to the +1e-16 of the denominator:
// ∂α_e/∂c = -α_e ε/(S+ε) with S = Σ_e exp(score - c), so ∂L/∂c = -Σ_{v,h} (Σ α dα) ε/(S+ε).  That sum goes to
// shift_acc[0] and the number of (edge, head) scores equal to c to shift_acc[1]; gat_bwd_shift_kernel routes it.
// DROP: the dot is the gradient of the dropped coefficient α' = keep α scale, so dα = keep scale <dOut[v], H[u]>.
template <bool DROP>
__global__ void __launch_bounds__(256)
gat_bwd_target_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx,
                      const float* __restrict__ H, int64_t ldh, const float* __restrict__ s_src,
                      const float* __restrict__ s_trg, const float* __restrict__ alpha,
                      const float* __restrict__ dOut, int64_t lddo, const float* __restrict__ H2, int64_t ldh2,
                      const float* __restrict__ dOut2, int64_t lddo2, int32_t n, int32_t nh, int32_t F, int act,
                      float slope, const float* __restrict__ gmax, float* __restrict__ dpre_edge, float* __restrict__ ds_trg,
                      float* __restrict__ shift_acc, AttnDrop dr) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const float gm = gmax ? *gmax : 0.f;
  float dshift = 0.f, ties = 0.f;
  for (int64_t v = warp; v < n; v += nwarps) {
    const int32_t s = rowptr[v], e = rowptr[v + 1];
    for (int h = 0; h < nh; ++h) {
      float t = 0.f;
      uint32_t kmask = 0;
      for (int32_t p = s; p < e; ++p) {
        const int32_t u = colidx[p];
        float d = 0.f;
        if constexpr (DROP) {
          if (((p - s) & 31) == 0)
            kmask = __ballot_sync(0xffffffffu, p + lane < e && dropout_keep(dr.seed, dr.key, (uint32_t)(p + lane), (uint32_t)h, dr.p));
        }
        if (!DROP || ((kmask >> ((p - s) & 31)) & 1u)) {
          for (int f = lane; f < F; f += 32) d = fmaf(dOut[v * lddo + h * F + f], H[(int64_t)u * ldh + h * F + f], d);
          if (H2)   // tied attention: the same α also weights a second layer's messages (stagate.py:197)
            for (int f = lane; f < F; f += 32) d = fmaf(dOut2[v * lddo2 + h * F + f], H2[(int64_t)u * ldh2 + h * F + f], d);
          d = warp_sum(d);
          if constexpr (DROP) d *= dr.scale;
        }
        if (lane == 0) dpre_edge[(int64_t)p * nh + h] = d;          // kept for the second sweep (same lane reads it back)
        t = fmaf(alpha[(int64_t)p * nh + h], d, t);
      }
      __syncwarp();
      float st = 0.f, S = 0.f;
      for (int32_t p = s; p < e; ++p) {
        const int32_t u = colidx[p];
        const float d = dpre_edge[(int64_t)p * nh + h];      // the dot of the first sweep (written by lane 0, visible after __syncwarp)
        const float a = alpha[(int64_t)p * nh + h];
        const float pre = s_src[(int64_t)u * nh + h] + s_trg[v * nh + h];
        const float g = a * (d - t) * score_act_grad(pre, act, slope);
        if (lane == 0) dpre_edge[(int64_t)p * nh + h] = g;
        st += g;
        if (gmax) {
          const float sc = score_act_f(pre, act, slope);
          S += expf(sc - gm);
          ties += (sc == gm) ? 1.f : 0.f;
        }
      }
      if (lane == 0) ds_trg[v * nh + h] = st;
      // ε/(S+ε) directly: 1 - Σα would cancel catastrophically wherever S ≫ ε
      if (gmax && e > s) dshift = fmaf(-t, 1e-16f / (S + 1e-16f), dshift);
    }
  }
  if (gmax && lane == 0 && (dshift != 0.f || ties != 0.f)) {
    atomicAdd(shift_acc, dshift);
    atomicAdd(shift_acc + 1, ties);
  }
}

// Backward of the global shift c = max over every (edge, head) score: ∂L/∂c (shift_acc[0]) is split evenly over the
// scores equal to c (shift_acc[1] of them), as torch's full-reduction max does, then taken through the score activation
// into dpre_edge and ds_trg (gat_bwd_source_kernel sums dpre_edge into ds_src afterwards).
__global__ void __launch_bounds__(256)
gat_bwd_shift_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx,
                     const float* __restrict__ s_src, const float* __restrict__ s_trg, int32_t n, int32_t nh, int act,
                     float slope, const float* __restrict__ gmax, const float* __restrict__ shift_acc,
                     float* __restrict__ dpre_edge, float* __restrict__ ds_trg) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const float gm = *gmax, ties = shift_acc[1];
  if (ties == 0.f) return;
  const float dc = shift_acc[0] / ties;
  if (dc == 0.f) return;
  for (int64_t v = warp; v < n; v += nwarps) {
    const int32_t s = rowptr[v], e = rowptr[v + 1];
    for (int32_t p = s + lane; p < e; p += 32) {
      const int32_t u = colidx[p];
      for (int h = 0; h < nh; ++h) {
        const float pre = s_src[(int64_t)u * nh + h] + s_trg[v * nh + h];
        if (score_act_f(pre, act, slope) == gm) {
          const float g = dc * score_act_grad(pre, act, slope);
          dpre_edge[(int64_t)p * nh + h] += g;
          atomicAdd(ds_trg + v * nh + h, g);
        }
      }
    }
  }
}

// Backward, part 2 (by source, on the transposed CSR; t_perm maps each entry to its position in the
// target CSR): dH[u] = Σ_out-edges α dOut[v] ; ds_src[u,h] = Σ dpre.  DROP: α' = keep α scale in place of α.
template <bool DROP>
__global__ void __launch_bounds__(256)
gat_bwd_source_kernel(const int32_t* __restrict__ t_rowptr, const int32_t* __restrict__ t_colidx,
                      const int32_t* __restrict__ t_perm, const float* __restrict__ alpha,
                      const float* __restrict__ dpre_edge, const float* __restrict__ dOut, int64_t lddo,
                      const float* __restrict__ dOut2, int64_t lddo2, int32_t n, int32_t nh, int32_t F,
                      float* __restrict__ dH, int64_t lddh, float* __restrict__ dH2, int64_t lddh2,
                      float* __restrict__ ds_src, AttnDrop dr) {
  constexpr int MAXV = 16;
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int W = nh * F;
  for (int64_t u = warp; u < n; u += nwarps) {
    const int32_t s = t_rowptr[u], e = t_rowptr[u + 1];
    float acc[MAXV], acc2[MAXV];
#pragma unroll
    for (int t = 0; t < MAXV; ++t) { acc[t] = 0.f; acc2[t] = 0.f; }
    float ssrc = 0.f;  // lanes < nh accumulate ds_src for their head
    uint32_t kb = 0;  // DROP: lane j holds the keep bits of out-edge (q - s) rounded down to 32, + j
    for (int32_t q = s; q < e; ++q) {
      uint32_t bits = 0;
      if constexpr (DROP) {
        if (((q - s) & 31) == 0) kb = q + lane < e ? edge_keep_bits(dr, t_perm[q + lane], nh) : 0u;
        bits = __shfl_sync(0xffffffffu, kb, (q - s) & 31);
      }
      const int32_t v = t_colidx[q];
      const int32_t p = t_perm[q];
#pragma unroll
      for (int t = 0; t < MAXV; ++t) {
        const int c = lane + 32 * t;
        if (c < W) {
          if constexpr (DROP) {
            const int h = c / F;
            if (!((bits >> h) & 1u)) continue;
          }
          const float a = DROP ? alpha[(int64_t)p * nh + c / F] * dr.scale : alpha[(int64_t)p * nh + c / F];
          acc[t] = fmaf(a, dOut[(int64_t)v * lddo + c], acc[t]);
          if (dOut2) acc2[t] = fmaf(a, dOut2[(int64_t)v * lddo2 + c], acc2[t]);
        }
      }
      if (lane < nh) ssrc += dpre_edge[(int64_t)p * nh + lane];
    }
#pragma unroll
    for (int t = 0; t < MAXV; ++t) {
      const int c = lane + 32 * t;
      if (c < W) {
        dH[u * lddh + c] = acc[t];
        if (dH2) dH2[u * lddh2 + c] = acc2[t];
      }
    }
    if (lane < nh) ds_src[u * nh + lane] = ssrc;
  }
}

// Backward, part 3: dH[n,h,f] += ds_src[n,h] a_src[h,f] + ds_trg[n,h] a_trg[h,f] ;
// da_src[h,f] += Σ_n ds_src[n,h] H[n,h,f] (and a_trg).  Block = 32 columns x row slice, atomics on da.
__global__ void __launch_bounds__(256)
gat_bwd_scores_kernel(const float* __restrict__ H, int64_t ldh, const float* __restrict__ a_src,
                      const float* __restrict__ a_trg, const float* __restrict__ ds_src,
                      const float* __restrict__ ds_trg, int32_t n, int32_t nh, int32_t F, float* __restrict__ dH,
                      int64_t lddh, float* __restrict__ da_src, float* __restrict__ da_trg) {
  __shared__ float rs[8][33], rt[8][33];
  const int W = nh * F;
  const int c = blockIdx.x * 32 + (threadIdx.x & 31);
  const int wy = threadIdx.x >> 5;
  const int64_t rows_per = ceil_div<int64_t>(n, gridDim.y);
  const int64_t r0 = (int64_t)blockIdx.y * rows_per;
  const int64_t r1 = (r0 + rows_per < (int64_t)n) ? r0 + rows_per : (int64_t)n;
  float ss = 0.f, st = 0.f;
  if (c < W) {
    const int h = c / F;
    const float as = a_src[c], at = a_trg[c];
    for (int64_t r = r0 + wy; r < r1; r += 8) {
      const float gs = ds_src[r * nh + h], gt = ds_trg[r * nh + h];
      const float hv = H[r * ldh + c];
      dH[r * lddh + c] += gs * as + gt * at;
      ss = fmaf(gs, hv, ss);
      st = fmaf(gt, hv, st);
    }
  }
  rs[wy][threadIdx.x & 31] = ss;
  rt[wy][threadIdx.x & 31] = st;
  __syncthreads();
  if (wy == 0 && c < W) {
    float a = 0.f, b = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) { a += rs[i][threadIdx.x & 31]; b += rt[i][threadIdx.x & 31]; }
    atomicAdd(da_src + c, a);
    atomicAdd(da_trg + c, b);
  }
}

// skip / concat-or-mean / bias / activation  (scgnn2.py:1189-1215)
// IDENTITY: skip is [n, F], added to every head (the FIN == FOUT branch, scgnn2.py:1167-1171)
template <bool IDENTITY>
__global__ void __launch_bounds__(256)
gat_combine_fwd_kernel(const float* __restrict__ agg, int64_t lda, const float* __restrict__ skip, int64_t lds,
                       const float* __restrict__ bias, int32_t n, int32_t nh, int32_t F, int concat, int act,
                       float* __restrict__ out, int64_t ldo) {
  const int OW = concat ? nh * F : F;
  const int64_t total = (int64_t)n * OW;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / OW;
    const int c = (int)(t % OW);
    float v;
    if (concat) {
      v = agg[i * lda + c] + (skip ? skip[i * lds + (IDENTITY ? c % F : c)] : 0.f);
    } else {
      v = 0.f;
      for (int h = 0; h < nh; ++h) v += agg[i * lda + h * F + c] + (skip ? skip[i * lds + (IDENTITY ? c : h * F + c)] : 0.f);
      v = v / (float)nh;   // mean over heads
    }
    if (bias) v += bias[c];
    out[i * ldo + c] = apply_act(v, act);
  }
}

// d(pre-combine)[n, nh*F] and d(pre-activation)[n, OW] (the latter feeds the bias gradient)
__global__ void __launch_bounds__(256)
gat_combine_bwd_kernel(const float* __restrict__ dout, int64_t lddo, const float* __restrict__ out, int64_t ldo,
                       int32_t n, int32_t nh, int32_t F, int concat, int act, float* __restrict__ dpre, int64_t ldp,
                       float* __restrict__ dact, int64_t ldact) {
  const int OW = concat ? nh * F : F;
  const int64_t total = (int64_t)n * OW;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / OW;
    const int c = (int)(t % OW);
    const float g = act_bwd(dout[i * lddo + c], out + i * ldo + c, nullptr, act);
    if (dact) dact[i * ldact + c] = g;
    if (concat) dpre[i * ldp + c] = g;
    else for (int h = 0; h < nh; ++h) dpre[i * ldp + h * F + c] = g / (float)nh;
  }
}

// The same with an identity skip: additionally dskip[n, F] = Σ_h dpre[n, h·F:(h+1)·F], the skip's share of d(input).
// One thread per (row, feature) walks the heads.
__global__ void __launch_bounds__(256)
gat_combine_bwd_identity_kernel(const float* __restrict__ dout, int64_t lddo, const float* __restrict__ out, int64_t ldo,
                                int32_t n, int32_t nh, int32_t F, int concat, int act, float* __restrict__ dpre, int64_t ldp,
                                float* __restrict__ dact, int64_t ldact, float* __restrict__ dskip, int64_t ldsk) {
  const int64_t total = (int64_t)n * F;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / F;
    const int f = (int)(t % F);
    float sum = 0.f;
    if (concat) {
      for (int h = 0; h < nh; ++h) {
        const int c = h * F + f;
        const float g = act_bwd(dout[i * lddo + c], out + i * ldo + c, nullptr, act);
        if (dact) dact[i * ldact + c] = g;
        dpre[i * ldp + c] = g;
        sum += g;
      }
    } else {
      const float g = act_bwd(dout[i * lddo + f], out + i * ldo + f, nullptr, act);
      if (dact) dact[i * ldact + f] = g;
      const float gh = g / (float)nh;
      for (int h = 0; h < nh; ++h) { dpre[i * ldp + h * F + f] = gh; sum += gh; }
    }
    dskip[i * ldsk + f] = sum;
  }
}

}  // namespace b2

using namespace b2;

extern "C" int b2_gat_scores_f32(const float* H, int64_t ldh, const float* a_src, const float* a_trg, int32_t n,
                                 int32_t nheads, int32_t F, float* s_src, float* s_trg, void* stream) {
  B2_REQUIRE(n >= 0 && nheads > 0 && F > 0 && ldh >= (int64_t)nheads * F, "b2_gat_scores_f32: bad arguments");
  if (n == 0) return B2_OK;
  B2_REQUIRE(H && a_src && a_trg && s_src && s_trg, "b2_gat_scores_f32: null pointer");
  gat_scores_kernel<<<grid_blocks(n, 8), 256, 0, as_stream(stream)>>>(H, ldh, a_src, a_trg, n, nheads, F, s_src, s_trg);
  B2_CHECK_LAUNCH("gat_scores_kernel");
  return B2_OK;
}

extern "C" int b2_gat_edge_max_f32(const int32_t* rowptr, const int32_t* colidx, const float* s_src,
                                   const float* s_trg, int32_t n, int32_t nheads, int score_act, float slope,
                                   float* gmax_dev, void* stream) {
  B2_REQUIRE(gmax_dev && n >= 0 && nheads > 0, "b2_gat_edge_max_f32: bad arguments");
  cudaStream_t st = as_stream(stream);
  set_neg_inf_kernel<<<1, 1, 0, st>>>(gmax_dev);
  B2_CHECK_LAUNCH("set_neg_inf_kernel");
  if (n == 0) return B2_OK;
  B2_REQUIRE(rowptr && colidx && s_src && s_trg, "b2_gat_edge_max_f32: null pointer");
  gat_edge_max_kernel<<<grid_blocks(n, 8), 256, 0, st>>>(rowptr, colidx, s_src, s_trg, n, nheads, score_act, slope, gmax_dev);
  B2_CHECK_LAUNCH("gat_edge_max_kernel");
  return B2_OK;
}

static bool drop_prob_ok(float p) { return p >= 0.f && p <= 1.f; }   // false for NaN
static AttnDrop make_drop(float p, uint32_t seed, uint32_t key) { return AttnDrop{p, p < 1.f ? 1.f / (1.f - p) : 0.f, seed, key}; }

extern "C" int b2_gat_aggregate_fwd_f32(const int32_t* rowptr, const int32_t* colidx, const float* H, int64_t ldh,
                                        const float* s_src, const float* s_trg, int32_t n, int32_t nheads, int32_t F,
                                        int score_act, float slope, int shift_mode, const float* gmax_dev, float* out,
                                        int64_t ldo, float* alpha_out, float drop_p, uint32_t seed, uint32_t key, void* stream) {
  B2_REQUIRE(n >= 0 && nheads > 0 && F > 0 && (int64_t)nheads * F <= 512 && ldh >= (int64_t)nheads * F && ldo >= (int64_t)nheads * F,
             "b2_gat_aggregate_fwd_f32: nheads*F must be <= 512 and leading dimensions >= nheads*F");
  B2_REQUIRE(drop_prob_ok(drop_p), "b2_gat_aggregate_fwd_f32: drop_p must be in [0, 1]");
  B2_REQUIRE(drop_p == 0.f || nheads <= 32, "b2_gat_aggregate_fwd_f32: attention dropout needs nheads <= 32");
  B2_REQUIRE(shift_mode == 1 || gmax_dev, "b2_gat_aggregate_fwd_f32: global shift needs gmax_dev");
  if (n == 0) return B2_OK;
  B2_REQUIRE(rowptr && colidx && H && s_src && s_trg && out, "b2_gat_aggregate_fwd_f32: null pointer");
  const auto kernel = drop_p > 0.f ? gat_aggregate_fwd_kernel<true> : gat_aggregate_fwd_kernel<false>;
  kernel<<<grid_blocks(n, 8), 256, 0, as_stream(stream)>>>(rowptr, colidx, H, ldh, s_src, s_trg, n, nheads, F, score_act, slope,
                                                           shift_mode, gmax_dev, out, ldo, alpha_out, make_drop(drop_p, seed, key));
  B2_CHECK_LAUNCH("gat_aggregate_fwd_kernel");
  return B2_OK;
}

extern "C" int b2_gat_aggregate_bwd_f32(const int32_t* rowptr, const int32_t* colidx, const int32_t* t_rowptr,
                                        const int32_t* t_colidx, const int32_t* t_perm, const float* H, int64_t ldh,
                                        const float* a_src, const float* a_trg, const float* s_src, const float* s_trg,
                                        const float* alpha, const float* dOut, int64_t lddo, const float* H2, int64_t ldh2,
                                        const float* dOut2, int64_t lddo2, int32_t n, int32_t nheads, int32_t F, int score_act,
                                        float slope, const float* gmax_dev, float* dH, int64_t lddh, float* dH2, int64_t lddh2,
                                        float* da_src, float* da_trg, float* ds_src_ws, float* ds_trg_ws, float* dpre_edge_ws,
                                        float* shift_ws, float drop_p, uint32_t seed, uint32_t key, void* stream) {
  B2_REQUIRE(n >= 0 && nheads > 0 && nheads <= 32 && F > 0 && (int64_t)nheads * F <= 512, "b2_gat_aggregate_bwd_f32: bad shape");
  B2_REQUIRE(a_src && a_trg && da_src && da_trg, "b2_gat_aggregate_bwd_f32: null pointer");
  B2_REQUIRE(!gmax_dev || shift_ws, "b2_gat_aggregate_bwd_f32: a global shift (gmax_dev) needs shift_ws");
  B2_REQUIRE(!H2 || dOut2, "b2_gat_aggregate_bwd_f32: a tied second layer (H2) needs its dOut2");
  B2_REQUIRE(drop_prob_ok(drop_p), "b2_gat_aggregate_bwd_f32: drop_p must be in [0, 1]");
  B2_REQUIRE(!H2 || drop_p == 0.f, "b2_gat_aggregate_bwd_f32: the tied backward has no attention dropout");
  cudaStream_t st = as_stream(stream);
  const int W = nheads * F;
  B2_CHECK_CUDA(cudaMemsetAsync(da_src, 0, sizeof(float) * W, st));
  B2_CHECK_CUDA(cudaMemsetAsync(da_trg, 0, sizeof(float) * W, st));
  if (n == 0) return B2_OK;
  B2_REQUIRE(rowptr && colidx && t_rowptr && t_colidx && t_perm && H && s_src && s_trg && alpha && dOut && dH && ds_src_ws &&
                 ds_trg_ws && dpre_edge_ws,
             "b2_gat_aggregate_bwd_f32: null pointer");
  if (gmax_dev) B2_CHECK_CUDA(cudaMemsetAsync(shift_ws, 0, sizeof(float) * 2, st));
  const AttnDrop drop = make_drop(drop_p, seed, key);
  const auto target_kernel = drop_p > 0.f ? gat_bwd_target_kernel<true> : gat_bwd_target_kernel<false>;
  target_kernel<<<grid_blocks(n, 8), 256, 0, st>>>(rowptr, colidx, H, ldh, s_src, s_trg, alpha, dOut, lddo, H2, ldh2, dOut2, lddo2, n,
                                                   nheads, F, score_act, slope, gmax_dev, dpre_edge_ws, ds_trg_ws, shift_ws, drop);
  B2_CHECK_LAUNCH("gat_bwd_target_kernel");
  if (gmax_dev) {
    gat_bwd_shift_kernel<<<grid_blocks(n, 8), 256, 0, st>>>(rowptr, colidx, s_src, s_trg, n, nheads, score_act, slope, gmax_dev,
                                                           shift_ws, dpre_edge_ws, ds_trg_ws);
    B2_CHECK_LAUNCH("gat_bwd_shift_kernel");
  }
  const auto source_kernel = drop_p > 0.f ? gat_bwd_source_kernel<true> : gat_bwd_source_kernel<false>;
  source_kernel<<<grid_blocks(n, 8), 256, 0, st>>>(t_rowptr, t_colidx, t_perm, alpha, dpre_edge_ws, dOut, lddo, dH2 ? dOut2 : nullptr,
                                                   lddo2, n, nheads, F, dH, lddh, dH2, lddh2, ds_src_ws, drop);
  B2_CHECK_LAUNCH("gat_bwd_source_kernel");
  dim3 grid(ceil_div(W, 32), row_splits(ceil_div(W, 32), n, 256, 2));
  gat_bwd_scores_kernel<<<grid, 256, 0, st>>>(H, ldh, a_src, a_trg, ds_src_ws, ds_trg_ws, n, nheads, F, dH, lddh, da_src, da_trg);
  B2_CHECK_LAUNCH("gat_bwd_scores_kernel");
  return B2_OK;
}

extern "C" int b2_gat_combine_fwd_f32(const float* agg, int64_t ldagg, const float* skip, int64_t ldskip, const float* bias,
                                      int32_t n, int32_t nheads, int32_t F, int concat, int act, int identity_skip, float* out,
                                      int64_t ldo, void* stream) {
  B2_REQUIRE(n >= 0 && nheads > 0 && F > 0, "b2_gat_combine_fwd_f32: bad arguments");
  B2_REQUIRE(act >= B2_ACT_NONE && act <= B2_ACT_TANH, "b2_gat_combine_fwd_f32: activation %d is not an epilogue code", act);
  B2_REQUIRE(!identity_skip || ldskip >= F, "b2_gat_combine_fwd_f32: an identity skip needs ldskip >= F");
  if (n == 0) return B2_OK;
  B2_REQUIRE(agg && out && (skip || !identity_skip), "b2_gat_combine_fwd_f32: null pointer");
  const auto kernel = identity_skip ? gat_combine_fwd_kernel<true> : gat_combine_fwd_kernel<false>;
  kernel<<<grid_blocks((int64_t)n * (concat ? nheads * F : F), 1024), 256, 0, as_stream(stream)>>>(agg, ldagg, skip, ldskip, bias, n,
                                                                                                   nheads, F, concat, act, out, ldo);
  B2_CHECK_LAUNCH("gat_combine_fwd_kernel");
  return B2_OK;
}

extern "C" int b2_gat_combine_bwd_f32(const float* dout, int64_t lddo, const float* out, int64_t ldo, int32_t n,
                                      int32_t nheads, int32_t F, int concat, int act, float* dpre, int64_t ldp, float* dact,
                                      int64_t ldact, float* dx_skip, int64_t ldx, void* stream) {
  B2_REQUIRE(n >= 0 && nheads > 0 && F > 0, "b2_gat_combine_bwd_f32: bad arguments");
  B2_REQUIRE(act >= B2_ACT_NONE && act <= B2_ACT_TANH, "b2_gat_combine_bwd_f32: activation %d is not an epilogue code", act);
  B2_REQUIRE(!dx_skip || ldx >= F, "b2_gat_combine_bwd_f32: dx_skip needs ldx >= F");
  if (n == 0) return B2_OK;
  B2_REQUIRE(dout && out && dpre, "b2_gat_combine_bwd_f32: null pointer");
  if (dx_skip) {
    gat_combine_bwd_identity_kernel<<<grid_blocks((int64_t)n * F, 1024), 256, 0, as_stream(stream)>>>(
        dout, lddo, out, ldo, n, nheads, F, concat, act, dpre, ldp, dact, ldact, dx_skip, ldx);
    B2_CHECK_LAUNCH("gat_combine_bwd_identity_kernel");
  } else {
    gat_combine_bwd_kernel<<<grid_blocks((int64_t)n * (concat ? nheads * F : F), 1024), 256, 0, as_stream(stream)>>>(
        dout, lddo, out, ldo, n, nheads, F, concat, act, dpre, ldp, dact, ldact);
    B2_CHECK_LAUNCH("gat_combine_bwd_kernel");
  }
  return B2_OK;
}
