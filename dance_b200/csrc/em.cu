// scGNN EM-iteration stages (SURVEY §8f row 3): the pieces between two Feature-AE / Graph-AE rounds.
//   * KMeans on the graph embedding (Lloyd iterations; the reference calls sklearn KMeans, scgnn2.py:186)
//   * the cell-type / graph regulariser of the Cluster-AE WITHOUT the reference's two dense N×N matrices
//     (normalize_cell_cell_matrix of the adjacency and of the same-cluster indicator, scgnn2.py:716-752): the loss only takes
//     `(M @ mse).sum()` (scgnn2.py:1323-1326) = Σ_j colsum_j(M)·mse_j, i.e. per-cell weights
//   * loss_function_graph(regularizer_type="Celltype") value + gradient (scgnn2.py:1316-1326) and the L1 term of
//     train_handler (scgnn2.py:1268-1274)
//   * Louvain community detection on the symmetric kNN graph (host C++, CSR in / labels out; the reference goes through
//     networkx → dense matrix → igraph.community_multilevel, scgnn2.py:193-215)
#include "common.cuh"

#include <algorithm>
#include <numeric>
#include <vector>

namespace b2 {
namespace {

// ---- KMeans ---------------------------------------------------------------------------------------------------------
// one thread per point, centroids staged in shared memory; accumulates the new centroid sums (fp64 atomics) in the same pass
__global__ void __launch_bounds__(256)
kmeans_assign_kernel(const float* __restrict__ X, int64_t ldx, int32_t n, int32_t d, const float* __restrict__ C, int32_t k,
                     int32_t* __restrict__ labels, double* __restrict__ sums, int32_t* __restrict__ counts, int32_t* __restrict__ changed,
                     double* __restrict__ inertia) {
  extern __shared__ float sc[];   // [k, d]
  for (int t = threadIdx.x; t < k * d; t += blockDim.x) sc[t] = C[t];
  __syncthreads();
  double in_local = 0.0;
  int ch_local = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float* x = X + i * ldx;
    float best = 3.4e38f;
    int bi = 0;
    for (int c = 0; c < k; ++c) {
      float s = 0.f;
      for (int j = 0; j < d; ++j) { const float df = x[j] - sc[c * d + j]; s = fmaf(df, df, s); }
      if (s < best) { best = s; bi = c; }     // ties → lowest index
    }
    if (labels[i] != bi) { ++ch_local; labels[i] = bi; }
    in_local += (double)best;
    if (sums) {
      for (int j = 0; j < d; ++j) atomicAdd(sums + (size_t)bi * d + j, (double)x[j]);
      atomicAdd(counts + bi, 1);
    }
  }
  in_local = warp_sum(in_local);
  if ((threadIdx.x & 31) == 0) {
    if (inertia) atomicAdd(inertia, in_local);
  }
  if (ch_local) atomicAdd(changed, ch_local);
}

// C ← sums / counts (empty clusters keep their centre); shift2[0] += ‖C_new − C_old‖²
__global__ void kmeans_update_kernel(float* __restrict__ C, const double* __restrict__ sums, const int32_t* __restrict__ counts, int32_t k,
                                     int32_t d, double* __restrict__ shift2) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= k * d) return;
  const int c = t / d;
  if (counts[c] > 0) {
    const float nv = (float)(sums[t] / (double)counts[c]);
    const double df = (double)nv - (double)C[t];
    atomicAdd(shift2, df * df);
    C[t] = nv;
  }
}

__global__ void kmeans_changed_kernel(const int32_t* changed, double* stats) { stats[2] = (double)changed[0]; }

// ---- cell-type / graph regulariser weights -----------------------------------------------------------------------------------
// graph_celltype_regu_handler (scgnn2.py:716-730) calls normalize_cell_cell_matrix on `sp.csr_matrix.todense(adj)`, i.e. on an
// np.matrix, for which `avg_mtx * x` is a MATRIX product: adjdense[i, j] = Σ_k (1/deg_i)·adj[k, j] = deg_j / deg_i — a dense
// rank-one matrix, whatever the edges are (App. B-style quirk; it defines parity).  The Cluster-AE of cluster c takes
// (adjdense[c][:, c] @ mse).sum() = Σ_{j∈c} w_j·mse_j  with  w_j = deg_j · Σ_{i∈c} 1/deg_i.  Two passes over the degrees, no N×N.
// pattern = A + I (CSR of the normalised adjacency) or A: deg = row length without the diagonal entry.
__device__ __forceinline__ int32_t plain_degree(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx, int64_t i) {
  int32_t deg = rowptr[i + 1] - rowptr[i];
  for (int32_t q = rowptr[i]; q < rowptr[i + 1]; ++q) deg -= (colidx[q] == (int32_t)i) ? 1 : 0;
  return deg;
}
__global__ void __launch_bounds__(256)
cluster_inv_degree_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx, const int32_t* __restrict__ labels,
                          int32_t n, int32_t n_clusters, double* __restrict__ sums) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int32_t deg = plain_degree(rowptr, colidx, i), c = labels[i];
    if (deg > 0 && c >= 0 && c < n_clusters) atomicAdd(sums + c, 1.0 / (double)deg);
  }
}
__global__ void __launch_bounds__(256)
graph_regu_weights_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx, const int32_t* __restrict__ labels,
                          int32_t n, int32_t n_clusters, const double* __restrict__ sums, float* __restrict__ w) {
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
    const int32_t c = labels[j];
    w[j] = (c >= 0 && c < n_clusters) ? (float)((double)plain_degree(rowptr, colidx, j) * sums[c]) : 0.f;
  }
}

// The same weights for a weighted, directed adj (graph_AE_retain_weights returns W, scgnn2.py:659-670): adjdense[i, j] =
// colsum_j / rowsum_i, so w_j = colsum_j · Σ_{i∈cluster(j)} 1/rowsum_i; a row with zero sum is masked (np.ma) and adds 0.
// Diagonal entries are skipped as above.  Pass 1: rowsum_i in column order, colsum_j by fp64 atomics, Σ 1/rowsum per cluster.
__global__ void __launch_bounds__(256)
weighted_sums_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx, const double* __restrict__ vals,
                     const int32_t* __restrict__ labels, int32_t n, int32_t n_clusters, double* __restrict__ colsum,
                     double* __restrict__ sums) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    double r = 0.0;
    for (int32_t q = rowptr[i]; q < rowptr[i + 1]; ++q) {
      const int32_t j = colidx[q];
      if (j == (int32_t)i) continue;
      r += vals[q];
      atomicAdd(colsum + j, vals[q]);
    }
    const int32_t c = labels[i];
    if (r != 0.0 && c >= 0 && c < n_clusters) atomicAdd(sums + c, 1.0 / r);
  }
}
__global__ void __launch_bounds__(256)
weighted_regu_weights_kernel(const int32_t* __restrict__ labels, int32_t n, int32_t n_clusters, const double* __restrict__ colsum,
                             const double* __restrict__ sums, float* __restrict__ w) {
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
    const int32_t c = labels[j];
    w[j] = (c >= 0 && c < n_clusters) ? (float)(colsum[j] * sums[c]) : 0.f;
  }
}

// ---- loss_function_graph("Celltype") --------------------------------------------------------------------------------------
// pass 1: acc[0] += Σ_j roww_j Σ_g (r−x)²,  acc[1] += Σ_{xd≠0} (xd − r)²      (fp64)
__global__ void __launch_bounds__(256)
celltype_reduce_kernel(const float* __restrict__ recon, const float* __restrict__ target, const float* __restrict__ xdrop,
                       const float* __restrict__ roww, int64_t rows, int32_t cols, int32_t cols_orig, double* __restrict__ acc) {
  double a = 0.0, b = 0.0;
  const int64_t total = rows * cols;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / cols;
    const int g = (int)(t % cols);
    const float r = recon[t], d = r - target[t];
    a += (double)(roww[i] * d * d);
    if (g < cols_orig) {
      const float xd = xdrop[i * cols_orig + g];
      if (xd != 0.f) { const float v = xd - r; b += (double)(v * v); }
    }
  }
  a = warp_sum(a); b = warp_sum(b);
  if ((threadIdx.x & 31) == 0) { atomicAdd(acc, a); atomicAdd(acc + 1, b); }
}

// pass 2: grad = 2·roww_j·(r−x) − [xd≠0]·(xd−r)/‖·‖, masked by the decoder's final ReLU; loss_out += acc[0] + sqrt(acc[1])
__global__ void __launch_bounds__(256)
celltype_grad_kernel(const float* __restrict__ recon, const float* __restrict__ target, const float* __restrict__ xdrop,
                     const float* __restrict__ roww, int64_t rows, int32_t cols, int32_t cols_orig, const double* __restrict__ acc,
                     int relu_mask, float* __restrict__ grad, float* __restrict__ loss_out) {
  const double nrm = sqrt(acc[1]);
  const float inv = nrm > 0.0 ? (float)(1.0 / nrm) : 0.f;
  const int64_t total = rows * cols;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = t / cols;
    const int g = (int)(t % cols);
    const float r = recon[t];
    float gr = 2.f * roww[i] * (r - target[t]);
    if (g < cols_orig) {
      const float xd = xdrop[i * cols_orig + g];
      if (xd != 0.f) gr -= (xd - r) * inv;
    }
    if (relu_mask && !(r > 0.f)) gr = 0.f;
    grad[t] = gr;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0 && loss_out) atomicAdd(loss_out, (float)(acc[0] + nrm));
}

// grad += coef·sign(p);  l1_out[0] += coef·Σ|p|
__global__ void __launch_bounds__(256)
l1_grad_kernel(const float* __restrict__ p, float* __restrict__ grad, int64_t n, float coef, float* __restrict__ l1_out) {
  double a = 0.0;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    const float v = p[t];
    a += (double)fabsf(v);
    grad[t] += coef * (v > 0.f ? 1.f : (v < 0.f ? -1.f : 0.f));     // torch: d|p|/dp = sign(p), 0 at 0
  }
  a = warp_sum(a);
  if ((threadIdx.x & 31) == 0 && l1_out) atomicAdd(l1_out, (float)(a * coef));
}

}  // namespace
}  // namespace b2

extern "C" size_t b2_kmeans_workspace_bytes(int32_t k, int32_t d) {
  return b2::align_up((size_t)k * d * sizeof(double), 256) + b2::align_up((size_t)k * sizeof(int32_t), 256) + 256;
}

// One Lloyd iteration: labels ← nearest centre (ties → lowest index), then (update != 0) centres ← cluster means.
// stats (device, 3 doubles): [0] inertia with the OLD centres, [1] ‖ΔC‖², [2] number of labels that changed (as double).
extern "C" int b2_kmeans_step_f32(const float* X, int64_t ldx, int32_t n, int32_t d, float* C, int32_t k, int32_t* labels, int update,
                                  double* stats, void* workspace, size_t workspace_bytes, void* stream) {
  using namespace b2;
  B2_REQUIRE(X && C && labels && stats, "b2_kmeans_step_f32: null pointer");
  B2_REQUIRE(n > 0 && d > 0 && k > 0 && ldx >= d, "b2_kmeans_step_f32: bad shape n=%d d=%d k=%d", n, d, k);
  B2_REQUIRE((size_t)k * d * sizeof(float) <= 96 * 1024, "b2_kmeans_step_f32: k·d = %d centroid floats exceed shared memory", k * d);
  B2_REQUIRE(workspace && workspace_bytes >= b2_kmeans_workspace_bytes(k, d), "b2_kmeans_step_f32: workspace too small");
  cudaStream_t st = as_stream(stream);
  char* w = reinterpret_cast<char*>(workspace);
  double* sums = reinterpret_cast<double*>(w);
  int32_t* counts = reinterpret_cast<int32_t*>(w + align_up((size_t)k * d * sizeof(double), 256));
  int32_t* changed = reinterpret_cast<int32_t*>(w + align_up((size_t)k * d * sizeof(double), 256) + align_up((size_t)k * sizeof(int32_t), 256));
  B2_CHECK_CUDA(cudaMemsetAsync(workspace, 0, b2_kmeans_workspace_bytes(k, d), st));
  B2_CHECK_CUDA(cudaMemsetAsync(stats, 0, 3 * sizeof(double), st));
  const size_t smem = (size_t)k * d * sizeof(float);
  const int rc = allow_dynamic_smem((const void*)kmeans_assign_kernel, smem);
  if (rc != B2_OK) return rc;
  kmeans_assign_kernel<<<grid_blocks(n, 256), 256, smem, st>>>(X, ldx, n, d, C, k, labels, update ? sums : nullptr, counts, changed, stats);
  B2_CHECK_LAUNCH("kmeans_assign_kernel");
  if (update) {
    kmeans_update_kernel<<<ceil_div(k * d, 128), 128, 0, st>>>(C, sums, counts, k, d, stats + 1);
    B2_CHECK_LAUNCH("kmeans_update_kernel");
  }
  kmeans_changed_kernel<<<1, 1, 0, st>>>(changed, stats);
  B2_CHECK_LAUNCH("kmeans_changed");
  return B2_OK;
}

extern "C" int b2_graph_regu_weights_f32(const int32_t* rowptr, const int32_t* colidx, const int32_t* labels, int32_t n, int32_t n_clusters,
                                         double* cluster_sums, float* w, void* stream) {
  using namespace b2;
  B2_REQUIRE(rowptr && colidx && labels && w && cluster_sums && n_clusters > 0, "b2_graph_regu_weights_f32: bad arguments");
  if (n <= 0) return B2_OK;
  cudaStream_t st = as_stream(stream);
  B2_CHECK_CUDA(cudaMemsetAsync(cluster_sums, 0, sizeof(double) * (size_t)n_clusters, st));
  cluster_inv_degree_kernel<<<grid_blocks(n, 256), 256, 0, st>>>(rowptr, colidx, labels, n, n_clusters, cluster_sums);
  B2_CHECK_LAUNCH("cluster_inv_degree_kernel");
  graph_regu_weights_kernel<<<grid_blocks(n, 256), 256, 0, st>>>(rowptr, colidx, labels, n, n_clusters, cluster_sums, w);
  B2_CHECK_LAUNCH("graph_regu_weights_kernel");
  return B2_OK;
}

extern "C" int b2_graph_regu_weights_weighted_f32(const int32_t* rowptr, const int32_t* colidx, const double* vals, const int32_t* labels,
                                                  int32_t n, int32_t n_clusters, double* scratch, float* w, void* stream) {
  using namespace b2;
  B2_REQUIRE(rowptr && colidx && vals && labels && w && scratch && n_clusters > 0, "b2_graph_regu_weights_weighted_f32: bad arguments");
  if (n <= 0) return B2_OK;
  cudaStream_t st = as_stream(stream);
  double* colsum = scratch;
  double* sums = scratch + n;
  B2_CHECK_CUDA(cudaMemsetAsync(scratch, 0, sizeof(double) * ((size_t)n + n_clusters), st));
  weighted_sums_kernel<<<grid_blocks(n, 256), 256, 0, st>>>(rowptr, colidx, vals, labels, n, n_clusters, colsum, sums);
  B2_CHECK_LAUNCH("weighted_sums_kernel");
  weighted_regu_weights_kernel<<<grid_blocks(n, 256), 256, 0, st>>>(labels, n, n_clusters, colsum, sums, w);
  B2_CHECK_LAUNCH("weighted_regu_weights_kernel");
  return B2_OK;
}

extern "C" int b2_celltype_loss_grad_f32(const float* recon, const float* target, const float* x_dropout, const float* row_weight,
                                         int64_t rows, int32_t cols, int32_t cols_orig, int relu_mask, float* grad, float* loss_out,
                                         double* scratch2, void* stream) {
  using namespace b2;
  B2_REQUIRE(recon && target && x_dropout && row_weight && grad && scratch2, "b2_celltype_loss_grad_f32: null pointer");
  B2_REQUIRE(rows >= 0 && cols > 0 && cols_orig > 0 && cols_orig <= cols, "b2_celltype_loss_grad_f32: bad shape");
  if (rows == 0) return B2_OK;
  cudaStream_t st = as_stream(stream);
  B2_CHECK_CUDA(cudaMemsetAsync(scratch2, 0, 2 * sizeof(double), st));
  const unsigned g = grid_blocks(rows * cols, 1024);
  celltype_reduce_kernel<<<g, 256, 0, st>>>(recon, target, x_dropout, row_weight, rows, cols, cols_orig, scratch2);
  B2_CHECK_LAUNCH("celltype_reduce_kernel");
  celltype_grad_kernel<<<g, 256, 0, st>>>(recon, target, x_dropout, row_weight, rows, cols, cols_orig, scratch2, relu_mask, grad, loss_out);
  B2_CHECK_LAUNCH("celltype_grad_kernel");
  return B2_OK;
}

extern "C" int b2_l1_grad_add_f32(const float* param, float* grad, int64_t n, float coef, float* l1_out, void* stream) {
  using namespace b2;
  B2_REQUIRE(param && grad, "b2_l1_grad_add_f32: null pointer");
  if (n <= 0) return B2_OK;
  l1_grad_kernel<<<grid_blocks(n, 1024), 256, 0, as_stream(stream)>>>(param, grad, n, coef, l1_out);
  B2_CHECK_LAUNCH("l1_grad_kernel");
  return B2_OK;
}

// ---- Louvain (host) ---------------------------------------------------------------------------------------------------------
// Multilevel modularity optimisation (Blondel et al. 2008) on a symmetric weighted CSR held in HOST memory (every undirected
// edge stored in both directions, no self loops at level 0).  Nodes are visited in index order, ties keep the current /
// lowest-numbered community — deterministic.  Returns the number of communities; labels_out[i] ∈ [0, n_comm).
extern "C" int b2_louvain_csr_host(const int64_t* rowptr, const int32_t* colidx, const double* weights, int32_t n, int32_t* labels_out,
                                   int32_t* n_comm_out, double* modularity_out, int max_levels, double min_gain) {
  using namespace b2;
  B2_REQUIRE(rowptr && colidx && labels_out && n_comm_out, "b2_louvain_csr_host: null pointer");
  B2_REQUIRE(n >= 0, "b2_louvain_csr_host: negative n");
  if (n == 0) { *n_comm_out = 0; return B2_OK; }
  if (max_levels <= 0) max_levels = 64;
  std::vector<int64_t> rp(rowptr, rowptr + n + 1);
  std::vector<int32_t> ci(colidx, colidx + rowptr[n]);
  std::vector<double> wv(rp[n]);
  for (int64_t e = 0; e < rp[n]; ++e) wv[e] = weights ? weights[e] : 1.0;
  std::vector<int32_t> node2comm(n);            // original node → current super-node
  std::iota(node2comm.begin(), node2comm.end(), 0);
  int32_t cur_n = n;
  double mod = 0.0;
  for (int level = 0; level < max_levels; ++level) {
    std::vector<double> k(cur_n, 0.0), self(cur_n, 0.0);
    double m2 = 0.0;
    for (int32_t i = 0; i < cur_n; ++i) {
      for (int64_t e = rp[i]; e < rp[i + 1]; ++e) { k[i] += wv[e]; if (ci[e] == i) self[i] += wv[e]; }
      m2 += k[i];
    }
    if (m2 <= 0.0) break;
    std::vector<int32_t> comm(cur_n);
    std::iota(comm.begin(), comm.end(), 0);
    std::vector<double> tot(k), neigh_w(cur_n, -1.0);
    std::vector<int32_t> neigh_c;
    neigh_c.reserve(64);
    bool any_move = false;
    for (int sweep = 0; sweep < 100; ++sweep) {
      int64_t moves = 0;
      for (int32_t i = 0; i < cur_n; ++i) {
        const int32_t ci_old = comm[i];
        neigh_c.clear();
        neigh_w[ci_old] = 0.0;
        neigh_c.push_back(ci_old);
        for (int64_t e = rp[i]; e < rp[i + 1]; ++e) {
          const int32_t j = ci[e];
          if (j == i) continue;
          const int32_t cj = comm[j];
          if (neigh_w[cj] < 0.0) { neigh_w[cj] = 0.0; neigh_c.push_back(cj); }
          neigh_w[cj] += wv[e];
        }
        tot[ci_old] -= k[i];
        int32_t best = ci_old;
        double best_gain = neigh_w[ci_old] - tot[ci_old] * k[i] / m2;
        for (int32_t c : neigh_c) {
          const double gain = neigh_w[c] - tot[c] * k[i] / m2;
          if (gain > best_gain) { best_gain = gain; best = c; }   // ties keep the current community
        }
        tot[best] += k[i];
        comm[i] = best;
        if (best != ci_old) ++moves;
        for (int32_t c : neigh_c) neigh_w[c] = -1.0;
      }
      if (moves == 0) break;
      any_move = true;
    }
    // modularity of this level's partition
    {
      std::vector<double> in(cur_n, 0.0), tt(cur_n, 0.0);
      for (int32_t i = 0; i < cur_n; ++i) {
        tt[comm[i]] += k[i];
        for (int64_t e = rp[i]; e < rp[i + 1]; ++e) if (comm[ci[e]] == comm[i]) in[comm[i]] += wv[e];
      }
      double q = 0.0;
      for (int32_t c = 0; c < cur_n; ++c) if (tt[c] > 0.0) q += in[c] / m2 - (tt[c] / m2) * (tt[c] / m2);
      if (!any_move || (level > 0 && q - mod < min_gain)) break;   // this level does not improve the partition: keep the previous one
      mod = q;
    }
    // renumber communities in order of first appearance and aggregate
    std::vector<int32_t> renum(cur_n, -1);
    int32_t nc = 0;
    for (int32_t i = 0; i < cur_n; ++i) { if (renum[comm[i]] < 0) renum[comm[i]] = nc++; comm[i] = renum[comm[i]]; }
    for (int32_t v = 0; v < n; ++v) node2comm[v] = comm[node2comm[v]];
    if (nc == cur_n) break;
    std::vector<std::vector<int32_t>> members(nc);
    for (int32_t i = 0; i < cur_n; ++i) members[comm[i]].push_back(i);
    std::vector<int64_t> nrp(nc + 1, 0);
    std::vector<int32_t> nci;
    std::vector<double> nwv;
    std::vector<double> accw(nc, 0.0);
    std::vector<char> seen(nc, 0);
    std::vector<int32_t> touched;
    for (int32_t c = 0; c < nc; ++c) {
      touched.clear();
      for (int32_t i : members[c])
        for (int64_t e = rp[i]; e < rp[i + 1]; ++e) {
          const int32_t cj = comm[ci[e]];
          if (!seen[cj]) { seen[cj] = 1; touched.push_back(cj); }
          accw[cj] += wv[e];
        }
      std::sort(touched.begin(), touched.end());
      for (int32_t cj : touched) { nci.push_back(cj); nwv.push_back(accw[cj]); accw[cj] = 0.0; seen[cj] = 0; }
      nrp[c + 1] = (int64_t)nci.size();
    }
    rp.swap(nrp); ci.swap(nci); wv.swap(nwv);
    cur_n = nc;
  }
  // final renumbering by first appearance over the original nodes
  std::vector<int32_t> renum(n, -1);
  int32_t nc = 0;
  for (int32_t v = 0; v < n; ++v) { if (renum[node2comm[v]] < 0) renum[node2comm[v]] = nc++; labels_out[v] = renum[node2comm[v]]; }
  *n_comm_out = nc;
  if (modularity_out) *modularity_out = mod;
  return B2_OK;
}
