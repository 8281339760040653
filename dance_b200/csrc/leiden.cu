// Leiden community detection on the device: SpaGCN's init="louvain" (spagcn.py:481-492 → scanpy 1.10 tl.leiden →
// leidenalg.RBConfigurationVertexPartition, resolution γ, weights = the connectivities, n_iterations = -1).
//
// Quality, for a symmetric CSR A with W = Σᵢⱼ Aᵢⱼ, kᵢ = Σⱼ Aᵢⱼ and K_c = Σ_{i∈c} kᵢ:  Q = Σ_c (e_c − γ·K_c²/W), e_c = Σ_{i,j∈c} Aᵢⱼ.
// Moving v from A to B changes Q by 2·[w(v,B) − w(v,A∖v) − γ·k_v·(K_B − K_{A∖v})/W].
//
// Exact sums.  Every weight is converted once to 64-bit fixed point, q = round(w · 2^s) with 2^s·nnz·max(w) ≤ 2^61, and every
// sum that decides a move (kᵢ, K_c, w(v,c), the aggregate weights, e_c) is an integer sum: exact, so it does not depend on the
// order in which threads add, and the result is run-to-run deterministic.  Gains are then formed in fp64 from those integers,
// in units of 2^-s (W cancels out of every comparison).  The fixed-point resolution is 2^-61 of nnz·max(w).
//
// One iteration (Traag, Waltman & van Eck 2019), repeated from the last membership until one leaves it unchanged and moves no
// vertex of the input graph (so that no single-vertex move improves the result):
//   local moving   sweeps over the pending vertices, alternately allowing only moves to a lower and to a higher community id
//                  (synchronous moves cannot then swap two vertices back and forth); a move to an empty community is allowed in
//                  both.  Each vertex's weights per neighbouring community come from a radix sort of (v, comm[u]) keys and a
//                  reduce-by-key, whatever its degree, so a hub with 10⁵ neighbour communities takes the same path as a leaf.
//                  The moves of one sweep are checked as if applied one after another in vertex order: each mover is
//                  charged what the earlier movers can cost it (arrivals into its target, departures from its community,
//                  adjacent movers), and a move that may no longer gain is dropped and stays pending.  So every sweep that
//                  moves raises Q and the phase cannot cycle; without this, thousands of leaves pile into a hub's community on
//                  the same stale K_B, and neighbours swap communities back and forth.  A moved vertex re-queues its
//                  neighbours for both directions.  The phase ends when a lower and a higher sweep
//                  in a row move nothing (or after LD_MAX_SWEEPS).
//   refinement     inside each community S, from singletons, in rounds of alternating direction: a singleton v well connected
//                  to S proposes the well-connected sub-community T with the largest non-negative gain w(v,T) − γ·k_v·K_T/W; a
//                  vertex whose own sub-community is a target stays, so every join is through an edge to a member that stays
//                  and refined communities are connected.  Ends after two rounds in a row without a proposal.  leidenalg draws T
//                  at random with probability ∝ exp(Δ/θ), θ = 0.01; the greedy choice here is the θ → 0 limit.
//   aggregation    refined communities become vertices; edge weights summed per (r_u, r_v) by sort + reduce-by-key, internal
//                  weight kept as a self-loop; the aggregate's membership starts from the unrefined communities.  Levels stop
//                  when aggregation would not reduce the vertex count.
// Labels are numbered by decreasing community size, ties by the smallest member vertex.
#include "common.cuh"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cmath>
#include <cstring>

namespace b2 {
namespace {

using u64 = unsigned long long;

constexpr int LD_MAX_ITERATIONS = 100;   // safety cap of max_iterations = -1 (iterations usually settle within a few)
constexpr int LD_MAX_SWEEPS = 1000;      // safety cap of one local-moving phase
constexpr int LD_THREADS = 256;
constexpr double LD_EPS = 1e-13;         // a local move must gain more than LD_EPS·W: fp64 rounding of the gain stays below it

struct U64Sum {
  __device__ __forceinline__ u64 operator()(u64 a, u64 b) const { return a + b; }
};
struct U64Eq {
  __device__ __forceinline__ bool operator()(u64 a, u64 b) const { return a == b; }
};

__device__ __forceinline__ u64 warp_sum_u64(u64 v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// order-preserving key of a non-negative gain (0 = no candidate)
__device__ __forceinline__ u64 gain_key(double g) { return (u64)__double_as_longlong(g == 0.0 ? 0.0 : g) + 1ull; }
__device__ __forceinline__ double key_gain(u64 k) { return __longlong_as_double((long long)(k - 1ull)); }

__device__ __forceinline__ int warp_id() { return (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5); }

// ---- input checks and fixed-point weights -------------------------------------------------------------------------------------
__global__ void __launch_bounds__(LD_THREADS)
ld_check_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx, const float* __restrict__ vals, int32_t n,
                int64_t nnz, unsigned* __restrict__ max_bits, int* __restrict__ bad) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += stride) {
    const int32_t u = colidx[e];
    const float w = vals ? vals[e] : 1.f;
    if (u < 0 || u >= n) atomicOr(bad, 1);
    if (!(w >= 0.f) || isinf(w)) atomicOr(bad, 2);
    else atomicMax(max_bits, __float_as_uint(w));   // non-negative floats order as their bit patterns
  }
  for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v <= n; v += stride) {
    const int32_t r = rowptr[v];
    if ((v == 0 && r != 0) || (v == n && r != nnz) || (v > 0 && r < rowptr[v - 1])) atomicOr(bad, 1);
  }
}

__global__ void __launch_bounds__(LD_THREADS)
ld_quantize_kernel(const float* __restrict__ vals, int64_t nnz, double scale, u64* __restrict__ qw) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += stride)
    qw[e] = (u64)llrint((double)(vals ? vals[e] : 1.f) * scale);
}

// ---- per-vertex edge sums (a warp per vertex; integer sums, so any order gives the same bits) ---------------------------------
// Σ qw over row v's edges to u with same[u] == same[v] (same NULL: all), diff[u] != diff[v] (diff NULL: all), u != v when
// skip_self.  out[v] = sum, or out[scat[v]] += sum; total += sum.
__global__ void __launch_bounds__(LD_THREADS)
ld_rowsum_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx, const u64* __restrict__ qw, int32_t n,
                 const int32_t* __restrict__ same, const int32_t* __restrict__ diff, int skip_self, u64* __restrict__ out,
                 const int32_t* __restrict__ scat, u64* __restrict__ total) {
  const int v = warp_id(), lane = threadIdx.x & 31;
  if (v >= n) return;
  const int32_t sv = same ? same[v] : 0, dv = diff ? diff[v] : 0;
  u64 s = 0;
  for (int32_t e = rowptr[v] + lane; e < rowptr[v + 1]; e += 32) {
    const int32_t u = colidx[e];
    if ((!skip_self || u != v) && (!same || same[u] == sv) && (!diff || diff[u] != dv)) s += qw[e];
  }
  s = warp_sum_u64(s);
  if (lane == 0) {
    if (out) {
      if (scat) atomicAdd(&out[scat[v]], s);
      else out[v] = s;
    }
    if (total) atomicAdd(total, s);
  }
}

// K[lab[v]] += kq[v], size[lab[v]] += 1, minv[lab[v]] = min(v); each output optional
__global__ void __launch_bounds__(LD_THREADS)
ld_group_kernel(int32_t n, const int32_t* __restrict__ lab, const u64* __restrict__ kq, u64* __restrict__ K, int32_t* __restrict__ size,
                int32_t* __restrict__ minv) {
  const int32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  const int32_t c = lab[v];
  if (K) atomicAdd(&K[c], kq[v]);
  if (size) atomicAdd(&size[c], 1);
  if (minv) atomicMin(&minv[c], v);
}

// ---- grouping: keys (hi[v] << shift | lab[u]) with the edge weight, for the selected vertices ----------------------------------
// sel NULL: every vertex; else sel[v] & selbit.  same NULL: every neighbour, else only u with same[u] == same[v].  The ballot keeps
// each row's edge order, so the (stable) sort sees the same input on every run.
template <bool FILL>
__global__ void __launch_bounds__(LD_THREADS)
ld_gather_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx, const u64* __restrict__ qw, int32_t n,
                 const uint8_t* __restrict__ sel, int selbit, const int32_t* __restrict__ hi, const int32_t* __restrict__ lab,
                 const int32_t* __restrict__ same, int skip_self, int shift, int32_t* __restrict__ counts,
                 const int32_t* __restrict__ offs, u64* __restrict__ keys, u64* __restrict__ vals) {
  const int v = warp_id(), lane = threadIdx.x & 31;
  if (v >= n) return;
  if (sel && !(sel[v] & selbit)) {
    if (!FILL && lane == 0) counts[v] = 0;
    return;
  }
  const int32_t beg = rowptr[v], end = rowptr[v + 1];
  const int32_t sv = same ? same[v] : 0;
  const u64 khi = (u64)(hi ? hi[v] : v) << shift;
  int32_t pos = FILL ? offs[v] : 0;
  for (int32_t base = beg; base < end; base += 32) {
    const int32_t e = base + lane;
    int32_t u = 0;
    bool keep = false;
    if (e < end) {
      u = colidx[e];
      keep = (!skip_self || u != v) && (!same || same[u] == sv);
    }
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    if (FILL && keep) {
      const int32_t p = pos + __popc(m & ((1u << lane) - 1u));
      keys[p] = khi | (u64)lab[u];
      vals[p] = qw[e];
    }
    pos += __popc(m);
  }
  if (!FILL && lane == 0) counts[v] = pos;
}

// ---- local moving ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(LD_THREADS)
ld_own_kernel(const u64* __restrict__ ukeys, const u64* __restrict__ agg, const int32_t* __restrict__ nruns, int shift,
              const int32_t* __restrict__ comm, u64* __restrict__ own) {
  const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= *nruns) return;
  const int32_t v = (int32_t)(ukeys[s] >> shift), c = (int32_t)(ukeys[s] & ((1ull << shift) - 1));
  if (c == comm[v]) own[v] = agg[s];
}

// PASS 0: best[v] = max gain key over the allowed neighbouring communities; PASS 1: bestc[v] = smallest community at that key
template <int PASS>
__global__ void __launch_bounds__(LD_THREADS)
ld_move_gain_kernel(const u64* __restrict__ ukeys, const u64* __restrict__ agg, const int32_t* __restrict__ nruns, int shift,
                    const int32_t* __restrict__ comm, const u64* __restrict__ kq, const u64* __restrict__ K,
                    const u64* __restrict__ own, double g, double eps, int dir, u64* __restrict__ best, int32_t* __restrict__ bestc) {
  const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= *nruns) return;
  const int32_t v = (int32_t)(ukeys[s] >> shift), c = (int32_t)(ukeys[s] & ((1ull << shift) - 1));
  const int32_t a = comm[v];
  if (c == a || (dir == 0 ? c > a : c < a)) return;
  const double gain = (double)((long long)agg[s] - (long long)own[v]) -
                      g * (double)kq[v] * ((double)K[c] - (double)(K[a] - kq[v]));
  if (!(gain > eps)) return;
  const u64 key = gain_key(gain);
  if (PASS == 0) atomicMax(&best[v], key);
  else if (key == best[v]) atomicMin(&bestc[v], c);
}

// target[v]: the chosen community, -1 (stay); want_empty[v] = 1 when an empty community gains most (ties go to the neighbour);
// gain[v]: the gain of the chosen move
__global__ void __launch_bounds__(LD_THREADS)
ld_move_decide_kernel(int32_t n, uint8_t* __restrict__ pend, int selbit, const int32_t* __restrict__ comm, const u64* __restrict__ kq,
                      const u64* __restrict__ K, const int32_t* __restrict__ size, const u64* __restrict__ own,
                      const u64* __restrict__ best, const int32_t* __restrict__ bestc, double g, double eps,
                      int32_t* __restrict__ target, int32_t* __restrict__ want_empty, double* __restrict__ gain) {
  const int32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  int32_t t = -1, we = 0;
  double gv = 0.0;
  if (pend[v] & selbit) {
    pend[v] &= (uint8_t)~selbit;
    const int32_t a = comm[v];
    const double ge = size[a] > 1 ? -(double)own[v] + g * (double)kq[v] * (double)(K[a] - kq[v]) : -1.0;
    const double gb = best[v] ? key_gain(best[v]) : -1.0;
    if (ge > eps && ge > gb) {
      we = 1;
      gv = ge;
    } else if (best[v]) {
      t = bestc[v];
      gv = gb;
    }
  }
  target[v] = t;
  want_empty[v] = we;
  gain[v] = gv;
}

__global__ void __launch_bounds__(LD_THREADS)
ld_flag_kernel(int32_t n, const int32_t* __restrict__ size, int32_t* __restrict__ flags) {
  const int32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c <= n) flags[c] = c < n && size[c] == 0;
}

__global__ void __launch_bounds__(LD_THREADS)
ld_empty_list_kernel(int32_t n, const int32_t* __restrict__ size, const int32_t* __restrict__ epos, int32_t* __restrict__ list) {
  const int32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < n && size[c] == 0) list[epos[c]] = c;
}

// the empty ids in increasing order go to the requesters in increasing vertex order; a requester left without one stays pending
__global__ void __launch_bounds__(LD_THREADS)
ld_take_empty_kernel(int32_t n, const int32_t* __restrict__ epos, const int32_t* __restrict__ want, const int32_t* __restrict__ rank,
                     const int32_t* __restrict__ list, int32_t* __restrict__ target, uint8_t* __restrict__ pend,
                     int32_t* __restrict__ ndeferred) {
  const int32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n || !want[v]) return;
  if (rank[v] < epos[n]) {
    target[v] = list[rank[v]];
  } else {
    pend[v] = 3;
    atomicAdd(ndeferred, 1);
  }
}

// Joint moves.  Every mover's gain was computed from the state before the sweep.  Apply the moves one after another in vertex
// order: a mover's gain then changes only through the movers before it, and the changes that can lower it are
//   strength  an earlier arrival into its target B, an earlier departure from its own community A (γ·k_v·Δ/W each);
//   edges     an earlier neighbour u that leaves B or joins A (A_uv each).
// A move is kept when its gain minus all of those still exceeds eps.  Dropping a move only removes changes, and the changes the
// bound ignores can only raise a gain, so every kept move gains more than eps in that sequence: each sweep that moves raises Q,
// and local moving cannot cycle.  A dropped vertex stays pending.
//
// mover keys (by target, or by own community), stable: ascending vertex within a key; the others sort last
__global__ void __launch_bounds__(LD_THREADS)
ld_mover_key_kernel(int32_t n, const int32_t* __restrict__ target, const int32_t* __restrict__ comm, int by_target,
                    u64* __restrict__ keys, u64* __restrict__ vals) {
  const int32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  const bool mover = target[v] >= 0 && target[v] != comm[v];
  keys[v] = mover ? (u64)(by_target ? target[v] : comm[v]) : 0xffffffffull;
  vals[v] = (u64)v;
}

__global__ void __launch_bounds__(LD_THREADS)
ld_mover_strength_kernel(int32_t n, const u64* __restrict__ sorted_v, const u64* __restrict__ kq, u64* __restrict__ out) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = kq[sorted_v[i]];
}

// before[v] = the strength of the movers before v that share its key
__global__ void __launch_bounds__(LD_THREADS)
ld_mover_scatter_kernel(int32_t n, const u64* __restrict__ keys, const u64* __restrict__ sorted_v, const u64* __restrict__ prefix,
                        u64* __restrict__ before) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && keys[i] != 0xffffffffull) before[sorted_v[i]] = prefix[i];
}

// a warp per vertex; kept[v] = the target of a kept move, else -1 (target itself is read by other warps, so it is not written)
__global__ void __launch_bounds__(LD_THREADS)
ld_mover_check_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx, const u64* __restrict__ qw, int32_t n,
                      const int32_t* __restrict__ comm, const int32_t* __restrict__ target, const double* __restrict__ gain,
                      const u64* __restrict__ kq, const u64* __restrict__ arrived, const u64* __restrict__ departed, double g,
                      double eps, int32_t* __restrict__ kept, uint8_t* __restrict__ pend, int32_t* __restrict__ ndropped) {
  const int v = warp_id(), lane = threadIdx.x & 31;
  if (v >= n) return;
  const int32_t a = comm[v], b = target[v];
  if (b < 0 || b == a) {
    if (lane == 0) kept[v] = -1;
    return;
  }
  u64 harm = 0;
  for (int32_t e = rowptr[v] + lane; e < rowptr[v + 1]; e += 32) {
    const int32_t u = colidx[e];
    if (u >= v) continue;
    const int32_t cu = comm[u], tu = target[u];
    if (tu >= 0 && tu != cu && (cu == b || tu == a)) harm += qw[e];
  }
  harm = warp_sum_u64(harm);
  if (lane == 0) {
    const double bound = gain[v] - (double)harm - g * (double)kq[v] * ((double)arrived[v] + (double)departed[v]);
    if (bound > eps) {
      kept[v] = b;
    } else {
      kept[v] = -1;
      pend[v] = 3;
      atomicAdd(ndropped, 1);
    }
  }
}

__global__ void __launch_bounds__(LD_THREADS)
ld_apply_kernel(int32_t n, const int32_t* __restrict__ target, int32_t* __restrict__ comm, uint8_t* __restrict__ moved,
                int32_t* __restrict__ nmoves) {
  const int32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  const int32_t t = target[v];
  const bool mv = t >= 0 && t != comm[v];
  if (mv) {
    comm[v] = t;
    atomicAdd(nmoves, 1);
  }
  moved[v] = mv;
}

// a moved vertex and its neighbours are pending in both directions
__global__ void __launch_bounds__(LD_THREADS)
ld_activate_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx, int32_t n, const uint8_t* __restrict__ moved,
                   uint8_t* __restrict__ pend) {
  const int v = warp_id(), lane = threadIdx.x & 31;
  if (v >= n || !moved[v]) return;
  if (lane == 0) pend[v] = 3;
  for (int32_t e = rowptr[v] + lane; e < rowptr[v + 1]; e += 32) pend[colidx[e]] = 3;
}

// ---- refinement --------------------------------------------------------------------------------------------------------------
// singleton v, well connected to its community S: w(v, S∖v) ≥ γ·k_v·(K_S − k_v)/W
__global__ void __launch_bounds__(LD_THREADS)
ld_refine_sel_kernel(int32_t n, const int32_t* __restrict__ comm, const int32_t* __restrict__ refined, const int32_t* __restrict__ rsize,
                     const u64* __restrict__ kq, const u64* __restrict__ K, const u64* __restrict__ wS, double g,
                     uint8_t* __restrict__ sel) {
  const int32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  sel[v] = rsize[refined[v]] == 1 && (double)wS[v] >= g * (double)kq[v] * (double)(K[comm[v]] - kq[v]);
}

template <int PASS>
__global__ void __launch_bounds__(LD_THREADS)
ld_refine_gain_kernel(const u64* __restrict__ ukeys, const u64* __restrict__ agg, const int32_t* __restrict__ nruns, int shift,
                      const int32_t* __restrict__ comm, const u64* __restrict__ kq, const u64* __restrict__ K,
                      const u64* __restrict__ Kt, const u64* __restrict__ wout, double g, int dir, u64* __restrict__ best,
                      int32_t* __restrict__ bestc) {
  const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= *nruns) return;
  const int32_t v = (int32_t)(ukeys[s] >> shift), T = (int32_t)(ukeys[s] & ((1ull << shift) - 1));
  if (T == v || (dir == 0 ? T > v : T < v)) return;
  const u64 KS = K[comm[v]];
  if (!((double)wout[T] >= g * (double)Kt[T] * (double)(KS - Kt[T]))) return;   // T well connected to S
  const double gain = (double)agg[s] - g * (double)kq[v] * (double)Kt[T];
  if (!(gain >= 0.0)) return;
  const u64 key = gain_key(gain);
  if (PASS == 0) atomicMax(&best[v], key);
  else if (key == best[v]) atomicMin(&bestc[v], T);
}

__global__ void __launch_bounds__(LD_THREADS)
ld_refine_decide_kernel(int32_t n, const uint8_t* __restrict__ sel, const u64* __restrict__ best, const int32_t* __restrict__ bestc,
                        int32_t* __restrict__ target, int32_t* __restrict__ targeted, int32_t* __restrict__ nprop) {
  const int32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  int32_t t = -1;
  if (sel[v] && best[v]) {
    t = bestc[v];
    targeted[t] = 1;
    atomicAdd(nprop, 1);
  }
  target[v] = t;
}

// a singleton's sub-community id is its own vertex id, so targeted[v] says whether anyone proposed to join v
__global__ void __launch_bounds__(LD_THREADS)
ld_refine_apply_kernel(int32_t n, const int32_t* __restrict__ target, const int32_t* __restrict__ targeted, int32_t* __restrict__ refined) {
  const int32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  if (target[v] >= 0 && !targeted[v]) refined[v] = target[v];
}

// ---- aggregation and relabelling -----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(LD_THREADS)
ld_mark_kernel(int32_t n, const int32_t* __restrict__ ids, int32_t* __restrict__ flags) {
  const int32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < n) flags[ids[v]] = 1;
}

__global__ void __launch_bounds__(LD_THREADS)
ld_iota_kernel(int32_t n, int32_t* __restrict__ out) {
  const int32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < n) out[v] = v;
}

// rmap[v] = compact id of v's refined community; the aggregate's membership = compact id of v's community
__global__ void __launch_bounds__(LD_THREADS)
ld_rmap_kernel(int32_t n, const int32_t* __restrict__ refined, const int32_t* __restrict__ rid, const int32_t* __restrict__ comm,
               const int32_t* __restrict__ cid, int32_t* __restrict__ rmap, int32_t* __restrict__ comm_next) {
  const int32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  const int32_t r = rid[refined[v]];
  rmap[v] = r;
  comm_next[r] = cid[comm[v]];   // every member of r writes the same value
}

__global__ void __launch_bounds__(LD_THREADS)
ld_compose_kernel(int32_t n, const int32_t* __restrict__ map, int32_t* __restrict__ x) {
  const int32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < n) x[v] = map[x[v]];
}

// the aggregate's CSR from the reduced (r_u, r_v) keys: row counts and column ids
__global__ void __launch_bounds__(LD_THREADS)
ld_agg_csr_kernel(const u64* __restrict__ ukeys, int32_t m, int shift, int32_t* __restrict__ rowcnt, int32_t* __restrict__ colidx) {
  const int32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= m) return;
  atomicAdd(&rowcnt[ukeys[s] >> shift], 1);
  colidx[s] = (int32_t)(ukeys[s] & ((1ull << shift) - 1));
}

// sort key of community c: decreasing size, then smallest member; empty communities last
__global__ void __launch_bounds__(LD_THREADS)
ld_order_key_kernel(int32_t n, const int32_t* __restrict__ size, const int32_t* __restrict__ minv, u64* __restrict__ keys,
                    u64* __restrict__ vals, int32_t* __restrict__ ncomm) {
  const int32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n) return;
  keys[c] = size[c] ? ((u64)(n - size[c]) << 32) | (u64)minv[c] : ~0ull;
  vals[c] = (u64)c;
  if (size[c]) atomicAdd(ncomm, 1);
}

__global__ void __launch_bounds__(LD_THREADS)
ld_rank_kernel(int32_t n, const u64* __restrict__ vals, const int32_t* __restrict__ ncomm, int32_t* __restrict__ lab_of) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < *ncomm) lab_of[vals[i]] = i;
}

__global__ void __launch_bounds__(LD_THREADS)
ld_relabel_kernel(int32_t n, const int32_t* __restrict__ lab_of, const int32_t* __restrict__ memb, int32_t* __restrict__ labels,
                  const int32_t* __restrict__ prev, int32_t* __restrict__ ndiff) {
  const int32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  const int32_t l = lab_of[memb[v]];
  labels[v] = l;
  if (l != prev[v]) atomicAdd(ndiff, 1);
}

// Σ_c K_c² in fp64 by one block in a fixed order (deterministic)
__global__ void __launch_bounds__(1024)
ld_sumsq_kernel(int32_t n, const u64* __restrict__ K, double* __restrict__ out) {
  __shared__ double part[32];
  double s = 0.0;
  for (int32_t c = threadIdx.x; c < n; c += blockDim.x) {
    const double k = (double)K[c];
    s += k * k;
  }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = threadIdx.x < (blockDim.x >> 5) ? part[threadIdx.x] : 0.0;
    s = warp_sum(s);
    if (threadIdx.x == 0) *out = s;
  }
}

// ---- workspace ---------------------------------------------------------------------------------------------------------------
struct Graph {
  const int32_t* rowptr;
  const int32_t* colidx;
  const u64* qw;
  int32_t n;
  int64_t m;
};

struct Work {
  // edges (E = max(nnz, n, 1) items)
  u64 *qw0, *qw[2], *keys_in, *keys_out, *vals_in, *vals_out, *ukeys, *agg;
  int32_t *colidx[2];
  // vertices (n + 1 items)
  int32_t *rowptr[2], *comm[2], *kept, *refined, *target, *bestc, *size, *minv, *targeted, *flags, *pos, *rank, *list, *rmap, *node2agg,
      *memb, *prev, *want, *lab_of, *counts;
  u64 *kq0, *kq[2], *K, *own, *best, *Kt, *wout, *wS;
  double* gain;
  uint8_t *pend, *moved;
  // scalars
  int32_t* ints;     // [0] runs, [1] moves / proposals, [2] communities, [3] differing labels, [4] bad input
  u64* totals;       // [0] W, [1] internal weight
  unsigned* maxw;
  double* sumsq;
  void* temp;
  size_t temp_bytes;
};

struct Carver {
  char* base;
  size_t off = 0;
  template <typename T>
  T* take(size_t count) {
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += align_up(sizeof(T) * (count ? count : 1), 256);
    return p;
  }
};

size_t cub_temp_bytes(int32_t n, int64_t E) {
  size_t a = 0, b = 0, c = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, a, (const u64*)nullptr, (u64*)nullptr, (const u64*)nullptr, (u64*)nullptr, (int)E, 0, 64);
  cub::DeviceReduce::ReduceByKey(nullptr, b, (const u64*)nullptr, (u64*)nullptr, (const u64*)nullptr, (u64*)nullptr, (int32_t*)nullptr,
                                 U64Sum(), (int)E);
  cub::DeviceScan::ExclusiveSum(nullptr, c, (const int32_t*)nullptr, (int32_t*)nullptr, n + 1);
  size_t d = 0;
  cub::DeviceScan::ExclusiveSumByKey(nullptr, d, (const u64*)nullptr, (const u64*)nullptr, (u64*)nullptr, n, U64Eq());
  return std::max(std::max(a, b), std::max(c, d));
}

size_t carve(Work& w, char* base, int32_t n, int64_t nnz) {
  const int64_t E = std::max<int64_t>(std::max<int64_t>(nnz, n), 1);
  const size_t V = (size_t)n + 1;
  Carver cv{base};
  w.qw0 = cv.take<u64>(E);
  for (int i = 0; i < 2; ++i) {
    w.qw[i] = cv.take<u64>(E);
    w.colidx[i] = cv.take<int32_t>(E);
    w.rowptr[i] = cv.take<int32_t>(V);
    w.comm[i] = cv.take<int32_t>(V);
    w.kq[i] = cv.take<u64>(V);
  }
  w.keys_in = cv.take<u64>(E);
  w.keys_out = cv.take<u64>(E);
  w.vals_in = cv.take<u64>(E);
  w.vals_out = cv.take<u64>(E);
  w.ukeys = cv.take<u64>(E);
  w.agg = cv.take<u64>(E);
  int32_t** iv[] = {&w.kept, &w.refined, &w.target, &w.bestc, &w.size, &w.minv, &w.targeted, &w.flags, &w.pos, &w.rank, &w.list, &w.rmap,
                    &w.node2agg, &w.memb, &w.prev, &w.want, &w.lab_of, &w.counts};
  for (auto p : iv) *p = cv.take<int32_t>(V);
  u64** uv[] = {&w.kq0, &w.K, &w.own, &w.best, &w.Kt, &w.wout, &w.wS};
  for (auto p : uv) *p = cv.take<u64>(V);
  w.gain = cv.take<double>(V);
  w.pend = cv.take<uint8_t>(V);
  w.moved = cv.take<uint8_t>(V);
  w.ints = cv.take<int32_t>(8);
  w.totals = cv.take<u64>(4);
  w.maxw = cv.take<unsigned>(1);
  w.sumsq = cv.take<double>(1);
  w.temp_bytes = cub_temp_bytes(n, E);
  w.temp = cv.take<char>(w.temp_bytes);
  return cv.off;
}

int bits_for(int32_t n) {   // bits to hold 0..n-1
  int b = 1;
  while (b < 31 && (1ll << b) < n) ++b;
  return b;
}

inline unsigned grid(int64_t items) { return (unsigned)std::max<int64_t>(ceil_div<int64_t>(items, LD_THREADS), 1); }
inline unsigned warp_grid(int64_t rows) { return grid(rows * 32); }

template <typename T>
int fetch(const T* dev, T* host, cudaStream_t st) {
  B2_CHECK_CUDA(cudaMemcpyAsync(host, dev, sizeof(T), cudaMemcpyDeviceToHost, st));
  B2_CHECK_CUDA(cudaStreamSynchronize(st));
  return B2_OK;
}

#define LD_TRY(expr)                     \
  do {                                   \
    const int _rc = (expr);              \
    if (_rc != B2_OK) return _rc;        \
  } while (0)

// Sorted, reduced (hi << shift | lab) keys of the selected rows' edges: ukeys / agg (or agg_out) with *runs on the host.
int group_edges(Work& w, const Graph& G, const uint8_t* sel, int selbit, const int32_t* hi, const int32_t* lab, const int32_t* same,
                int skip_self, int shift, u64* agg_out, int32_t* runs, cudaStream_t st) {
  const int32_t n = G.n;
  ld_gather_kernel<false><<<warp_grid(n), LD_THREADS, 0, st>>>(G.rowptr, G.colidx, G.qw, n, sel, selbit, hi, lab, same, skip_self,
                                                              shift, w.counts, nullptr, nullptr, nullptr);
  B2_CHECK_LAUNCH("ld_gather_kernel<count>");
  B2_CHECK_CUDA(cudaMemsetAsync(w.counts + n, 0, sizeof(int32_t), st));
  size_t tb = w.temp_bytes;
  B2_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, tb, w.counts, w.pos, n + 1, st));
  int32_t total = 0;
  LD_TRY(fetch(w.pos + n, &total, st));
  *runs = 0;
  if (total == 0) return B2_OK;
  ld_gather_kernel<true><<<warp_grid(n), LD_THREADS, 0, st>>>(G.rowptr, G.colidx, G.qw, n, sel, selbit, hi, lab, same, skip_self,
                                                             shift, nullptr, w.pos, w.keys_in, w.vals_in);
  B2_CHECK_LAUNCH("ld_gather_kernel<fill>");
  tb = w.temp_bytes;
  B2_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(w.temp, tb, w.keys_in, w.keys_out, w.vals_in, w.vals_out, total, 0, 2 * shift, st));
  tb = w.temp_bytes;
  B2_CHECK_CUDA(cub::DeviceReduce::ReduceByKey(w.temp, tb, w.keys_out, w.ukeys, w.vals_out, agg_out ? agg_out : w.agg, w.ints,
                                               U64Sum(), total, st));
  return fetch(w.ints, runs, st);
}

// K, size of the communities of `lab` (n ids), zeroed first
int community_sums(Work& w, int32_t n, const int32_t* lab, const u64* kq, cudaStream_t st) {
  B2_CHECK_CUDA(cudaMemsetAsync(w.K, 0, sizeof(u64) * n, st));
  B2_CHECK_CUDA(cudaMemsetAsync(w.size, 0, sizeof(int32_t) * n, st));
  ld_group_kernel<<<grid(n), LD_THREADS, 0, st>>>(n, lab, kq, w.K, w.size, nullptr);
  B2_CHECK_LAUNCH("ld_group_kernel");
  return B2_OK;
}

// one local-moving phase on G from membership comm; *moved_any = 1 if a vertex moved
int local_moving(Work& w, const Graph& G, int32_t* comm, const u64* kq, double g, double eps, int* moved_any, cudaStream_t st) {
  const int32_t n = G.n;
  const int shift = bits_for(n);
  B2_CHECK_CUDA(cudaMemsetAsync(w.pend, 3, n, st));
  LD_TRY(community_sums(w, n, comm, kq, st));
  int quiet = 0;
  for (int sweep = 0, dir = 0; sweep < LD_MAX_SWEEPS && quiet < 2; ++sweep, dir ^= 1) {
    const int selbit = 1 << dir;
    int32_t runs = 0;
    LD_TRY(group_edges(w, G, w.pend, selbit, nullptr, comm, nullptr, 1, shift, nullptr, &runs, st));
    B2_CHECK_CUDA(cudaMemsetAsync(w.own, 0, sizeof(u64) * n, st));
    B2_CHECK_CUDA(cudaMemsetAsync(w.best, 0, sizeof(u64) * n, st));
    B2_CHECK_CUDA(cudaMemsetAsync(w.bestc, 0x7f, sizeof(int32_t) * n, st));
    if (runs > 0) {
      ld_own_kernel<<<grid(runs), LD_THREADS, 0, st>>>(w.ukeys, w.agg, w.ints, shift, comm, w.own);
      B2_CHECK_LAUNCH("ld_own_kernel");
      ld_move_gain_kernel<0><<<grid(runs), LD_THREADS, 0, st>>>(w.ukeys, w.agg, w.ints, shift, comm, kq, w.K, w.own, g, eps, dir,
                                                                w.best, w.bestc);
      B2_CHECK_LAUNCH("ld_move_gain_kernel<0>");
      ld_move_gain_kernel<1><<<grid(runs), LD_THREADS, 0, st>>>(w.ukeys, w.agg, w.ints, shift, comm, kq, w.K, w.own, g, eps, dir,
                                                                w.best, w.bestc);
      B2_CHECK_LAUNCH("ld_move_gain_kernel<1>");
    }
    ld_move_decide_kernel<<<grid(n), LD_THREADS, 0, st>>>(n, w.pend, selbit, comm, kq, w.K, w.size, w.own, w.best, w.bestc, g, eps,
                                                          w.target, w.want, w.gain);
    B2_CHECK_LAUNCH("ld_move_decide_kernel");
    // empty ids (ascending) for the vertices that leave for an empty community (ascending)
    ld_flag_kernel<<<grid(n + 1), LD_THREADS, 0, st>>>(n, w.size, w.flags);
    B2_CHECK_LAUNCH("ld_flag_kernel");
    size_t tb = w.temp_bytes;
    B2_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, tb, w.flags, w.pos, n + 1, st));
    B2_CHECK_CUDA(cudaMemsetAsync(w.want + n, 0, sizeof(int32_t), st));
    tb = w.temp_bytes;
    B2_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, tb, w.want, w.rank, n + 1, st));
    ld_empty_list_kernel<<<grid(n), LD_THREADS, 0, st>>>(n, w.size, w.pos, w.list);
    B2_CHECK_LAUNCH("ld_empty_list_kernel");
    B2_CHECK_CUDA(cudaMemsetAsync(w.ints + 1, 0, 2 * sizeof(int32_t), st));
    ld_take_empty_kernel<<<grid(n), LD_THREADS, 0, st>>>(n, w.pos, w.want, w.rank, w.list, w.target, w.pend, w.ints + 2);
    B2_CHECK_LAUNCH("ld_take_empty_kernel");
    // strength of the earlier movers into each target (arrived → Kt) and out of each community (departed → wout)
    u64* before[2] = {w.wout, w.Kt};
    for (int by_target = 0; by_target < 2; ++by_target) {
      ld_mover_key_kernel<<<grid(n), LD_THREADS, 0, st>>>(n, w.target, comm, by_target, w.keys_in, w.vals_in);
      B2_CHECK_LAUNCH("ld_mover_key_kernel");
      tb = w.temp_bytes;
      B2_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(w.temp, tb, w.keys_in, w.keys_out, w.vals_in, w.vals_out, n, 0, 33, st));
      ld_mover_strength_kernel<<<grid(n), LD_THREADS, 0, st>>>(n, w.vals_out, kq, w.agg);
      B2_CHECK_LAUNCH("ld_mover_strength_kernel");
      tb = w.temp_bytes;
      B2_CHECK_CUDA(cub::DeviceScan::ExclusiveSumByKey(w.temp, tb, w.keys_out, w.agg, w.ukeys, n, U64Eq(), st));
      ld_mover_scatter_kernel<<<grid(n), LD_THREADS, 0, st>>>(n, w.keys_out, w.vals_out, w.ukeys, before[by_target]);
      B2_CHECK_LAUNCH("ld_mover_scatter_kernel");
    }
    ld_mover_check_kernel<<<warp_grid(n), LD_THREADS, 0, st>>>(G.rowptr, G.colidx, G.qw, n, comm, w.target, w.gain, kq, w.Kt, w.wout,
                                                               g, eps, w.kept, w.pend, w.ints + 2);
    B2_CHECK_LAUNCH("ld_mover_check_kernel");
    ld_apply_kernel<<<grid(n), LD_THREADS, 0, st>>>(n, w.kept, comm, w.moved, w.ints + 1);
    B2_CHECK_LAUNCH("ld_apply_kernel");
    int32_t counts[2] = {0, 0};   // moves, moves dropped or deferred (those vertices stay pending)
    B2_CHECK_CUDA(cudaMemcpyAsync(counts, w.ints + 1, sizeof(counts), cudaMemcpyDeviceToHost, st));
    B2_CHECK_CUDA(cudaStreamSynchronize(st));
    const int32_t moves = counts[0];
    if (moves == 0 && counts[1] == 0) {
      ++quiet;
      continue;
    }
    quiet = 0;
    *moved_any = 1;
    ld_activate_kernel<<<warp_grid(n), LD_THREADS, 0, st>>>(G.rowptr, G.colidx, n, w.moved, w.pend);
    B2_CHECK_LAUNCH("ld_activate_kernel");
    LD_TRY(community_sums(w, n, comm, kq, st));
  }
  return B2_OK;
}

// refine the partition comm of G (w.K holds its community strengths) into w.refined
int refine(Work& w, const Graph& G, const int32_t* comm, const u64* kq, double g, cudaStream_t st) {
  const int32_t n = G.n;
  const int shift = bits_for(n);
  ld_iota_kernel<<<grid(n), LD_THREADS, 0, st>>>(n, w.refined);
  B2_CHECK_LAUNCH("ld_iota_kernel");
  ld_rowsum_kernel<<<warp_grid(n), LD_THREADS, 0, st>>>(G.rowptr, G.colidx, G.qw, n, comm, nullptr, 1, w.wS, nullptr, nullptr);
  B2_CHECK_LAUNCH("ld_rowsum_kernel<wS>");
  int quiet = 0;
  for (int dir = 0; quiet < 2; dir ^= 1) {
    B2_CHECK_CUDA(cudaMemsetAsync(w.Kt, 0, sizeof(u64) * n, st));
    B2_CHECK_CUDA(cudaMemsetAsync(w.wout, 0, sizeof(u64) * n, st));
    B2_CHECK_CUDA(cudaMemsetAsync(w.minv, 0, sizeof(int32_t) * n, st));   // sub-community sizes
    ld_group_kernel<<<grid(n), LD_THREADS, 0, st>>>(n, w.refined, kq, w.Kt, w.minv, nullptr);
    B2_CHECK_LAUNCH("ld_group_kernel<refined>");
    ld_rowsum_kernel<<<warp_grid(n), LD_THREADS, 0, st>>>(G.rowptr, G.colidx, G.qw, n, comm, w.refined, 1, w.wout, w.refined, nullptr);
    B2_CHECK_LAUNCH("ld_rowsum_kernel<wout>");
    ld_refine_sel_kernel<<<grid(n), LD_THREADS, 0, st>>>(n, comm, w.refined, w.minv, kq, w.K, w.wS, g, w.pend);
    B2_CHECK_LAUNCH("ld_refine_sel_kernel");
    int32_t runs = 0;
    LD_TRY(group_edges(w, G, w.pend, 1, nullptr, w.refined, comm, 1, shift, nullptr, &runs, st));
    B2_CHECK_CUDA(cudaMemsetAsync(w.best, 0, sizeof(u64) * n, st));
    B2_CHECK_CUDA(cudaMemsetAsync(w.bestc, 0x7f, sizeof(int32_t) * n, st));
    B2_CHECK_CUDA(cudaMemsetAsync(w.targeted, 0, sizeof(int32_t) * n, st));
    B2_CHECK_CUDA(cudaMemsetAsync(w.ints + 1, 0, sizeof(int32_t), st));
    if (runs > 0) {
      ld_refine_gain_kernel<0><<<grid(runs), LD_THREADS, 0, st>>>(w.ukeys, w.agg, w.ints, shift, comm, kq, w.K, w.Kt, w.wout, g, dir,
                                                                  w.best, w.bestc);
      B2_CHECK_LAUNCH("ld_refine_gain_kernel<0>");
      ld_refine_gain_kernel<1><<<grid(runs), LD_THREADS, 0, st>>>(w.ukeys, w.agg, w.ints, shift, comm, kq, w.K, w.Kt, w.wout, g, dir,
                                                                  w.best, w.bestc);
      B2_CHECK_LAUNCH("ld_refine_gain_kernel<1>");
    }
    ld_refine_decide_kernel<<<grid(n), LD_THREADS, 0, st>>>(n, w.pend, w.best, w.bestc, w.target, w.targeted, w.ints + 1);
    B2_CHECK_LAUNCH("ld_refine_decide_kernel");
    int32_t props = 0;
    LD_TRY(fetch(w.ints + 1, &props, st));
    if (props == 0) {
      ++quiet;
      continue;
    }
    quiet = 0;
    ld_refine_apply_kernel<<<grid(n), LD_THREADS, 0, st>>>(n, w.target, w.targeted, w.refined);
    B2_CHECK_LAUNCH("ld_refine_apply_kernel");
  }
  return B2_OK;
}

// compact ids of the values present in ids[0..n): out[x] for x present, *count on the host
int compact_ids(Work& w, int32_t n, const int32_t* ids, int32_t* out, int32_t* count, cudaStream_t st) {
  B2_CHECK_CUDA(cudaMemsetAsync(w.flags, 0, sizeof(int32_t) * ((size_t)n + 1), st));
  ld_mark_kernel<<<grid(n), LD_THREADS, 0, st>>>(n, ids, w.flags);
  B2_CHECK_LAUNCH("ld_mark_kernel");
  size_t tb = w.temp_bytes;
  B2_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, tb, w.flags, out, n + 1, st));
  return fetch(out + n, count, st);
}

// labels (n0) numbered by decreasing size, ties by smallest member, from membership w.memb; *ndiff = labels changed vs w.prev
int canonical_labels(Work& w, int32_t n0, int32_t* labels, int32_t* ncomm, int32_t* ndiff, cudaStream_t st) {
  B2_CHECK_CUDA(cudaMemsetAsync(w.size, 0, sizeof(int32_t) * n0, st));
  B2_CHECK_CUDA(cudaMemsetAsync(w.minv, 0x7f, sizeof(int32_t) * n0, st));
  B2_CHECK_CUDA(cudaMemsetAsync(w.ints + 2, 0, 2 * sizeof(int32_t), st));
  ld_group_kernel<<<grid(n0), LD_THREADS, 0, st>>>(n0, w.memb, nullptr, nullptr, w.size, w.minv);
  B2_CHECK_LAUNCH("ld_group_kernel<labels>");
  ld_order_key_kernel<<<grid(n0), LD_THREADS, 0, st>>>(n0, w.size, w.minv, w.keys_in, w.vals_in, w.ints + 2);
  B2_CHECK_LAUNCH("ld_order_key_kernel");
  size_t tb = w.temp_bytes;
  B2_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(w.temp, tb, w.keys_in, w.keys_out, w.vals_in, w.vals_out, n0, 0, 64, st));
  ld_rank_kernel<<<grid(n0), LD_THREADS, 0, st>>>(n0, w.vals_out, w.ints + 2, w.lab_of);
  B2_CHECK_LAUNCH("ld_rank_kernel");
  ld_relabel_kernel<<<grid(n0), LD_THREADS, 0, st>>>(n0, w.lab_of, w.memb, labels, w.prev, w.ints + 3);
  B2_CHECK_LAUNCH("ld_relabel_kernel");
  LD_TRY(fetch(w.ints + 2, ncomm, st));
  return fetch(w.ints + 3, ndiff, st);
}

// one Leiden iteration on the level-0 graph G0 from membership w.memb (ids < n0); leaves the new membership in w.memb
int iteration(Work& w, const Graph& G0, double gamma, double W, int* levels, int* moved0, cudaStream_t st) {
  const int32_t n0 = G0.n;
  const double g = gamma / W, eps = LD_EPS * W;
  Graph G = G0;
  const u64* kq = w.kq0;
  int cur = 0;   // this level's membership is w.comm[cur]
  B2_CHECK_CUDA(cudaMemcpyAsync(w.comm[0], w.memb, sizeof(int32_t) * n0, cudaMemcpyDeviceToDevice, st));
  ld_iota_kernel<<<grid(n0), LD_THREADS, 0, st>>>(n0, w.node2agg);
  B2_CHECK_LAUNCH("ld_iota_kernel<node2agg>");
  *levels = 0;
  for (;;) {
    ++*levels;
    int32_t* comm = w.comm[cur];
    int moved = 0;
    LD_TRY(local_moving(w, G, comm, kq, g, eps, &moved, st));
    if (*levels == 1) *moved0 = moved;
    LD_TRY(refine(w, G, comm, kq, g, st));
    int32_t n2 = 0, nc = 0;
    LD_TRY(compact_ids(w, G.n, w.refined, w.list, &n2, st));
    if (n2 >= G.n) break;   // aggregation would not reduce the vertex count
    LD_TRY(compact_ids(w, G.n, comm, w.rank, &nc, st));
    const int nxt = cur ^ 1;
    ld_rmap_kernel<<<grid(G.n), LD_THREADS, 0, st>>>(G.n, w.refined, w.list, comm, w.rank, w.rmap, w.comm[nxt]);
    B2_CHECK_LAUNCH("ld_rmap_kernel");
    ld_compose_kernel<<<grid(n0), LD_THREADS, 0, st>>>(n0, w.rmap, w.node2agg);
    B2_CHECK_LAUNCH("ld_compose_kernel");
    // the aggregate, into the graph buffers the current level does not use (level 0 reads the caller's CSR and qw0)
    const int buf = G.qw == w.qw[0] ? 1 : 0;
    const int shift2 = bits_for(n2);
    int32_t m2 = 0;
    LD_TRY(group_edges(w, G, nullptr, 0, w.rmap, w.rmap, nullptr, 0, shift2, w.qw[buf], &m2, st));
    B2_CHECK_CUDA(cudaMemsetAsync(w.counts, 0, sizeof(int32_t) * ((size_t)n2 + 1), st));
    if (m2 > 0) {
      ld_agg_csr_kernel<<<grid(m2), LD_THREADS, 0, st>>>(w.ukeys, m2, shift2, w.counts, w.colidx[buf]);
      B2_CHECK_LAUNCH("ld_agg_csr_kernel");
    }
    size_t tb = w.temp_bytes;
    B2_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(w.temp, tb, w.counts, w.rowptr[buf], n2 + 1, st));
    G = Graph{w.rowptr[buf], w.colidx[buf], w.qw[buf], n2, m2};
    // the aggregate's strengths, self-loops included (= the sums of its members' strengths)
    ld_rowsum_kernel<<<warp_grid(n2), LD_THREADS, 0, st>>>(G.rowptr, G.colidx, G.qw, n2, nullptr, nullptr, 0, w.kq[buf], nullptr,
                                                           nullptr);
    B2_CHECK_LAUNCH("ld_rowsum_kernel<strength>");
    kq = w.kq[buf];
    cur = nxt;
  }
  // membership of the level-0 vertices
  B2_CHECK_CUDA(cudaMemcpyAsync(w.memb, w.node2agg, sizeof(int32_t) * n0, cudaMemcpyDeviceToDevice, st));
  ld_compose_kernel<<<grid(n0), LD_THREADS, 0, st>>>(n0, w.comm[cur], w.memb);
  B2_CHECK_LAUNCH("ld_compose_kernel<membership>");
  return B2_OK;
}

}  // namespace
}  // namespace b2

using namespace b2;

extern "C" size_t b2_leiden_workspace_bytes(int32_t n, int64_t nnz) {
  if (n <= 0 || nnz < 0 || nnz > INT32_MAX) return 0;
  Work w;
  return carve(w, nullptr, n, nnz);
}

extern "C" int b2_leiden_f32(const int32_t* rowptr, const int32_t* colidx, const float* vals, int32_t n, int64_t nnz, double resolution,
                             int max_iterations, int32_t* labels_out, int32_t* n_comm_out, double* quality_out, int32_t* info_out,
                             void* workspace, size_t workspace_bytes, void* stream) {
  B2_REQUIRE(rowptr && colidx && labels_out && n_comm_out && quality_out && workspace, "b2_leiden_f32: null pointer");
  B2_REQUIRE(n > 0 && nnz >= 0 && nnz <= INT32_MAX, "b2_leiden_f32: need n > 0 and 0 <= nnz < 2^31 (n=%d, nnz=%lld)", n, (long long)nnz);
  B2_REQUIRE(resolution >= 0.0 && resolution < HUGE_VAL, "b2_leiden_f32: resolution must be finite and non-negative (got %g)",
             resolution);
  B2_REQUIRE(max_iterations == -1 || max_iterations > 0, "b2_leiden_f32: max_iterations must be -1 or positive (got %d)",
             max_iterations);
  B2_REQUIRE(workspace_bytes >= b2_leiden_workspace_bytes(n, nnz), "b2_leiden_f32: workspace too small (%zu < %zu bytes)",
             workspace_bytes, b2_leiden_workspace_bytes(n, nnz));
  cudaStream_t st = as_stream(stream);
  Work w;
  carve(w, reinterpret_cast<char*>(workspace), n, nnz);

  // input checks, and the fixed-point scale from the largest weight
  B2_CHECK_CUDA(cudaMemsetAsync(w.maxw, 0, sizeof(unsigned), st));
  B2_CHECK_CUDA(cudaMemsetAsync(w.ints + 4, 0, sizeof(int32_t), st));
  const unsigned cg = grid_blocks(std::max<int64_t>(nnz, n + 1), LD_THREADS, 8);
  ld_check_kernel<<<cg, LD_THREADS, 0, st>>>(rowptr, colidx, vals, n, nnz, w.maxw, w.ints + 4);
  B2_CHECK_LAUNCH("ld_check_kernel");
  int32_t bad = 0;
  unsigned maxw_bits = 0;
  LD_TRY(fetch(w.ints + 4, &bad, st));
  LD_TRY(fetch(w.maxw, &maxw_bits, st));
  B2_REQUIRE(!(bad & 1), "b2_leiden_f32: rowptr / colidx do not form a CSR of n=%d rows and nnz=%lld columns in [0, n)", n,
             (long long)nnz);
  B2_REQUIRE(!(bad & 2), "b2_leiden_f32: vals must be finite and non-negative");
  float maxw;
  memcpy(&maxw, &maxw_bits, sizeof(maxw));
  if (info_out) info_out[0] = info_out[1] = 0;

  u64 Wq = 0;
  if (nnz > 0 && maxw > 0.f) {
    int ex = 0;
    frexp((double)maxw * (double)nnz, &ex);   // nnz·max(w) < 2^ex
    const double scale = ldexp(1.0, 61 - ex);
    ld_quantize_kernel<<<cg, LD_THREADS, 0, st>>>(vals, nnz, scale, w.qw0);
    B2_CHECK_LAUNCH("ld_quantize_kernel");
    B2_CHECK_CUDA(cudaMemsetAsync(w.totals, 0, sizeof(u64), st));
    ld_rowsum_kernel<<<warp_grid(n), LD_THREADS, 0, st>>>(rowptr, colidx, w.qw0, n, nullptr, nullptr, 0, w.kq0, nullptr, w.totals);
    B2_CHECK_LAUNCH("ld_rowsum_kernel<strength>");
    LD_TRY(fetch(w.totals, &Wq, st));
  }
  if (Wq == 0) {   // no weight: every vertex is its own community
    ld_iota_kernel<<<grid(n), LD_THREADS, 0, st>>>(n, labels_out);
    B2_CHECK_LAUNCH("ld_iota_kernel<labels>");
    B2_CHECK_CUDA(cudaStreamSynchronize(st));
    *n_comm_out = n;
    *quality_out = 0.0;
    return B2_OK;
  }

  const Graph G0{rowptr, colidx, w.qw0, n, nnz};
  const double W = (double)Wq;
  const int cap = max_iterations > 0 ? max_iterations : LD_MAX_ITERATIONS;
  ld_iota_kernel<<<grid(n), LD_THREADS, 0, st>>>(n, w.memb);
  B2_CHECK_LAUNCH("ld_iota_kernel<membership>");
  B2_CHECK_CUDA(cudaMemsetAsync(w.prev, 0xff, sizeof(int32_t) * n, st));   // -1: the first iteration always counts as a change
  int32_t ncomm = 0;
  for (int it = 0; it < cap; ++it) {
    int levels = 0, moved0 = 0;
    LD_TRY(iteration(w, G0, resolution, W, &levels, &moved0, st));
    int32_t ndiff = 0;
    LD_TRY(canonical_labels(w, n, labels_out, &ncomm, &ndiff, st));
    if (info_out) {
      info_out[0] = it + 1;
      info_out[1] = std::max(info_out[1], levels);
    }
    if (ndiff == 0 && !moved0) break;   // no vertex of the input graph moved: the labels are node-optimal
    B2_CHECK_CUDA(cudaMemcpyAsync(w.prev, labels_out, sizeof(int32_t) * n, cudaMemcpyDeviceToDevice, st));
    B2_CHECK_CUDA(cudaMemcpyAsync(w.memb, labels_out, sizeof(int32_t) * n, cudaMemcpyDeviceToDevice, st));
  }

  // Q / W = e_in / W − γ·Σ_c K_c² / W², all in fixed-point units
  B2_CHECK_CUDA(cudaMemsetAsync(w.totals + 1, 0, sizeof(u64), st));
  ld_rowsum_kernel<<<warp_grid(n), LD_THREADS, 0, st>>>(rowptr, colidx, w.qw0, n, labels_out, nullptr, 0, nullptr, nullptr, w.totals + 1);
  B2_CHECK_LAUNCH("ld_rowsum_kernel<internal>");
  B2_CHECK_CUDA(cudaMemsetAsync(w.K, 0, sizeof(u64) * n, st));
  ld_group_kernel<<<grid(n), LD_THREADS, 0, st>>>(n, labels_out, w.kq0, w.K, nullptr, nullptr);
  B2_CHECK_LAUNCH("ld_group_kernel<quality>");
  ld_sumsq_kernel<<<1, 1024, 0, st>>>(ncomm, w.K, w.sumsq);
  B2_CHECK_LAUNCH("ld_sumsq_kernel");
  u64 ein = 0;
  double sumsq = 0.0;
  LD_TRY(fetch(w.totals + 1, &ein, st));
  LD_TRY(fetch(w.sumsq, &sumsq, st));
  *n_comm_out = ncomm;
  *quality_out = (double)ein / W - resolution * sumsq / (W * W);
  return B2_OK;
}
