// The per-pair arithmetic of SpaGCN's spot graph, shared by the dense kernels (knn.cu pairwise_dense_kernel, dec.cu exp_adj*)
// and the coordinate sweeps (spatial_adj.cu), so that a pair's distance and weight are the same bits on both paths.
#pragma once
#include "common.cuh"

namespace b2 {

// Euclidean distance of two points of d coordinates, evaluated like the reference's numba kernel (utils/matrix.py:100-105):
// (a-b)² in fp32, summed in fp64 in coordinate order, fp64 sqrt, cast to fp32.  `a` and `b` are anything indexable (a row of a
// matrix, or a register array).  Coordinates padded with zeros on both sides add +0.0 to the sum, so a point set padded to
// more coordinates gives the same bits.
template <typename A, typename B>
__device__ __forceinline__ float pair_l2(const A& a, const B& b, int d) {
  double s = 0.0;
  for (int c = 0; c < d; ++c) {
    const float diff = __fsub_rn(a[c], b[c]);
    s = __dadd_rn(s, (double)__fmul_rn(diff, diff));
  }
  return (float)sqrt(s);
}

// SpaGCN's adjacency weight exp(-D²/(2 l²)) of one distance (np.exp(-1 * adj**2 / (2 * l**2)), spagcn.py:807-809), IEEE
// division and the accurate expf.
__device__ __forceinline__ float exp_adj_weight(float dist, float two_l2) { return expf(-(dist * dist) / two_l2); }

// numpy divides the fp32 array by the python float 2·l², which it rounds to fp32 first
static inline float exp_adj_two_l2(double l) { return (float)(2.0 * (l * l)); }

}  // namespace b2
