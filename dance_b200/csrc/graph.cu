// Graph assembly on device: CSR transpose and the scGNN kNN-graph pipeline
//   feature2adj (reference scgnn2.py:650-672): union-symmetrise the directed
//   kNN lists into a 0/1 adjacency, drop the diagonal;
//   preprocess_graph (scgnn2.py:1191-1198): Â = D^-1/2 (A + I) D^-1/2;
//   and with retain_weights (scgnn2.py:659-670) the weighted, directed W = 1/(d + 1e-16), for which
//   Â = ((W + I)·Dm)ᵀ·Dm is asymmetric: both orientations of W + I are built.
// Sort / unique / scan primitives come from CUB (header-only part of the CUDA
// toolkit); everything specific to the path is hand-written here.
#include "common.cuh"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_select.cuh>

namespace b2 {

struct WsCarver {
  char* base;
  size_t off = 0;
  size_t cap;
  WsCarver(void* p, size_t c) : base(reinterpret_cast<char*>(p)), cap(c) {}
  template <typename T>
  T* take(size_t n) {
    off = align_up(off, 256);
    T* r = reinterpret_cast<T*>(base + off);
    off += n * sizeof(T);
    return r;
  }
  bool ok() const { return off <= cap; }
};

__global__ void iota_kernel(int32_t* out, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = (int32_t)i;
}

// first position p in sorted[0,n) with sorted[p] >= key
template <typename T>
__device__ __forceinline__ int64_t lower_bound_dev(const T* sorted, int64_t n, T key) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (sorted[mid] < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__global__ void rowptr_from_sorted_i32(const int32_t* sorted_keys, int64_t nnz, int32_t n_rows, int32_t* rowptr) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r <= n_rows; r += (int64_t)gridDim.x * blockDim.x)
    rowptr[r] = (int32_t)lower_bound_dev<int32_t>(sorted_keys, nnz, (int32_t)r);
}

__global__ void transpose_fill_kernel(const int32_t* rowptr, const float* vals, const int32_t* perm, int32_t n_rows,
                                      int64_t nnz, int32_t* t_colidx, float* t_vals) {
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < nnz; p += (int64_t)gridDim.x * blockDim.x) {
    const int32_t e = perm[p];
    // source row of entry e: last r with rowptr[r] <= e
    int32_t lo = 0, hi = n_rows;
    while (lo < hi) {
      const int32_t mid = (lo + hi) >> 1;
      if (rowptr[mid + 1] <= e) lo = mid + 1; else hi = mid;
    }
    t_colidx[p] = lo;
    if (t_vals) t_vals[p] = vals ? vals[e] : 1.f;
  }
}

static int bits_for(int64_t n) {
  int b = 1;
  while ((1ll << b) < n && b < 62) ++b;
  return b;
}

// ---- kNN graph ------------------------------------------------------------

__global__ void knn_edge_keys_kernel(const int32_t* knn_idx, int32_t n, int32_t k, uint64_t* keys) {
  const int64_t total = (int64_t)n * k;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total + n; t += (int64_t)gridDim.x * blockDim.x) {
    if (t < total) {
      const uint64_t i = (uint64_t)(t / k);
      const uint64_t j = (uint64_t)knn_idx[t];
      keys[2 * t] = (i << 32) | j;       // i -> j
      keys[2 * t + 1] = (j << 32) | i;   // j -> i   (nx.from_dict_of_lists builds an undirected graph)
    } else {
      const uint64_t i = (uint64_t)(t - total);
      keys[2 * total + i] = (i << 32) | i;  // + I  (preprocess_graph adds sp.eye)
    }
  }
}

__global__ void knn_rowptr_kernel(const uint64_t* ukeys, const int32_t* num_unique, int32_t n, int32_t* rowptr) {
  const int64_t m = *num_unique;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r <= n; r += (int64_t)gridDim.x * blockDim.x)
    rowptr[r] = (int32_t)lower_bound_dev<uint64_t>(ukeys, m, ((uint64_t)r) << 32);
}

__global__ void knn_fill_kernel(const uint64_t* ukeys, const int32_t* rowptr, int32_t n, int32_t* colidx,
                                float* vals_norm) {
  // one thread per row keeps colidx/vals writes contiguous per row; rows are short (<= 2k+1 on average)
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    const int32_t s = rowptr[r], e = rowptr[r + 1];
    const double di = 1.0 / sqrt((double)(e - s));  // rowsum of (A+I) = number of entries (all ones)
    for (int32_t p = s; p < e; ++p) {
      const int32_t j = (int32_t)(ukeys[p] & 0xffffffffull);
      colidx[p] = j;
      const double dj = 1.0 / sqrt((double)(rowptr[j + 1] - rowptr[j]));
      vals_norm[p] = (float)(dj * di);  // (A_ · D^-1/2)ᵀ · D^-1/2, evaluated in fp64 then cast (scgnn2.py:1196,1205)
    }
  }
}

// ---- weighted, directed kNN graph (graph_AE_retain_weights) ----------------------------------------------------------------
// feature2adj with retain_weights (scgnn2.py:659-670): W[i, j] = 1/(d_ij + 1e-16) for the k listed neighbours of i, directed;
// adj_train = W without its diagonal.  L = adj_train + I, stored twice: by source row (L) and by target row (Lᵀ).  Entry t < n·k
// is the t-th kNN slot (a slot naming its own row is the dropped diagonal), entry n·k + i the unit diagonal of row i.  The sort
// key is (row << 32 | column); a dropped slot gets the key (n << 32), past every real row.
__global__ void knn_weighted_keys_kernel(const int32_t* knn_idx, int32_t n, int32_t k, bool by_target, uint64_t* keys, int32_t* slots,
                                         int32_t* bad_index) {
  const int64_t total = (int64_t)n * k;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total + n; t += (int64_t)gridDim.x * blockDim.x) {
    uint64_t key;
    if (t < total) {
      const uint64_t i = (uint64_t)(t / k);
      const int32_t jj = knn_idx[t];
      if (jj < 0 || jj >= n) { atomicExch(bad_index, 1); key = (uint64_t)n << 32; }
      else {
        const uint64_t j = (uint64_t)jj;
        key = j == i ? (uint64_t)n << 32 : (by_target ? (j << 32) | i : (i << 32) | j);
      }
    } else {
      const uint64_t i = (uint64_t)(t - total);
      key = (i << 32) | i;
    }
    keys[t] = key;
    slots[t] = (int32_t)t;
  }
}

// rowptr[n] = the number of kept entries: the dropped slots sort after row n − 1
__global__ void knn_weighted_rowptr_kernel(const uint64_t* keys, int64_t total, int32_t n, int32_t* rowptr) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r <= n; r += (int64_t)gridDim.x * blockDim.x)
    rowptr[r] = (int32_t)lower_bound_dev<uint64_t>(keys, total, ((uint64_t)r) << 32);
}

// a neighbour listed twice in one row would make two entries of one (row, column)
__global__ void sorted_keys_duplicate_kernel(const uint64_t* keys, const int32_t* rowptr, int32_t n, int32_t* dup) {
  const int64_t nnz = rowptr[n];
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p + 1 < nnz; p += (int64_t)gridDim.x * blockDim.x)
    if (keys[p] == keys[p + 1]) atomicExch(dup, 1);
}

__device__ __forceinline__ double slot_weight(const double* knn_dist, int64_t total, int32_t slot) {
  return slot < total ? 1.0 / (knn_dist[slot] + 1e-16) : 1.0;   // scgnn2.py:686; the + I entries are 1
}

// r_i = Σ_j adj_[i, j] over row i of L in column order (rowsum of adj_train + I, scgnn2.py:1194), dm_i = r_i^-1/2;
// w_row_i = the same row without the diagonal (its share of ΣW)
__global__ void knn_weighted_rowsum_kernel(const int32_t* rowptr, const uint64_t* keys, const int32_t* slots, const double* knn_dist,
                                           int32_t n, int32_t k, double* dm, double* w_row) {
  const int64_t total = (int64_t)n * k;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    double r = 0.0, w = 0.0;
    for (int32_t p = rowptr[i]; p < rowptr[i + 1]; ++p) {
      const double v = slot_weight(knn_dist, total, slots[p]);
      r += v;
      if ((int64_t)(keys[p] & 0xffffffffull) != i) w += v;
    }
    dm[i] = 1.0 / sqrt(r);
    w_row[i] = w;
  }
}

// Fill one orientation.  L (by_target = false): row i, entries j, y = adj_[i, j], norm = Âᵀ[i, j] = adj_[i, j]·dm_j·dm_i.
// Lᵀ (by_target = true): row a, entries b, y = adj_[b, a], norm = Â[a, b] = adj_[b, a]·dm_a·dm_b.  Â = (adj_·Dm)ᵀ·Dm
// (scgnn2.py:1196): the products are taken in that order in fp64 and cast to fp32 once.
__global__ void knn_weighted_fill_kernel(const int32_t* rowptr, const uint64_t* keys, const int32_t* slots, const double* knn_dist,
                                         const double* dm, int32_t n, int32_t k, bool by_target, int32_t* colidx, float* y,
                                         float* norm) {
  const int64_t total = (int64_t)n * k;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    const double dr = dm[r];
    for (int32_t p = rowptr[r]; p < rowptr[r + 1]; ++p) {
      const int32_t c = (int32_t)(keys[p] & 0xffffffffull);
      const double v = slot_weight(knn_dist, total, slots[p]);
      colidx[p] = c;
      y[p] = (float)v;
      // adj_[src, dst]·dm_dst·dm_src with (src, dst) = (r, c) for L and (c, r) for Lᵀ
      norm[p] = (float)(by_target ? (v * dr) * dm[c] : (v * dm[c]) * dr);
    }
  }
}

}  // namespace b2

using namespace b2;

extern "C" size_t b2_csr_transpose_workspace_bytes(int32_t n_rows, int32_t n_cols, int64_t nnz) {
  size_t temp = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, temp, (const int32_t*)nullptr, (int32_t*)nullptr,
                                  (const int32_t*)nullptr, (int32_t*)nullptr, (int)nnz);
  return align_up(temp, 256) + 3 * align_up((size_t)nnz * 4, 256) + 1024;
}

extern "C" int b2_csr_transpose(const int32_t* rowptr, const int32_t* colidx, const float* vals, int32_t n_rows,
                                int32_t n_cols, int64_t nnz, int32_t* t_rowptr, int32_t* t_colidx, float* t_vals,
                                int32_t* perm_out, void* workspace, size_t workspace_bytes, void* stream) {
  B2_REQUIRE(rowptr && t_rowptr, "b2_csr_transpose: null pointer");
  B2_REQUIRE(nnz >= 0 && nnz < (1ll << 31), "b2_csr_transpose: nnz out of range");
  cudaStream_t st = as_stream(stream);
  if (nnz == 0) {   // an edgeless matrix: colidx / t_colidx may have no storage
    B2_CHECK_CUDA(cudaMemsetAsync(t_rowptr, 0, sizeof(int32_t) * ((size_t)n_cols + 1), st));
    return B2_OK;
  }
  B2_REQUIRE(colidx && t_colidx, "b2_csr_transpose: null pointer");
  B2_REQUIRE(workspace && workspace_bytes >= b2_csr_transpose_workspace_bytes(n_rows, n_cols, nnz),
             "b2_csr_transpose: workspace too small");
  WsCarver ws(workspace, workspace_bytes);
  int32_t* keys_out = ws.take<int32_t>(nnz);
  int32_t* iota = ws.take<int32_t>(nnz);
  int32_t* perm = perm_out ? perm_out : ws.take<int32_t>(nnz);
  size_t temp = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, temp, colidx, keys_out, iota, perm, (int)nnz);
  void* d_temp = ws.take<char>(temp);
  if (!ws.ok()) { set_error("b2_csr_transpose: workspace carve overflow"); return B2_ERR_WORKSPACE; }
  iota_kernel<<<grid_blocks(nnz, 256, 32), 256, 0, st>>>(iota, nnz);
  B2_CHECK_LAUNCH("iota_kernel");
  // stable LSD radix sort: equal columns keep source (row-major) order → deterministic transpose
  B2_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(d_temp, temp, colidx, keys_out, iota, perm, (int)nnz, 0,
                                                bits_for((int64_t)n_cols + 1), st));
  rowptr_from_sorted_i32<<<grid_blocks((int64_t)n_cols + 1, 256, 32), 256, 0, st>>>(keys_out, nnz, n_cols, t_rowptr);
  B2_CHECK_LAUNCH("rowptr_from_sorted_i32");
  transpose_fill_kernel<<<grid_blocks(nnz, 256, 32), 256, 0, st>>>(rowptr, vals, perm, n_rows, nnz, t_colidx, t_vals);
  B2_CHECK_LAUNCH("transpose_fill_kernel");
  return B2_OK;
}

extern "C" size_t b2_knn_graph_workspace_bytes(int32_t n, int32_t k) {
  const int64_t total = 2ll * n * k + n;
  size_t t1 = 0, t2 = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, t1, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int)total);
  cub::DeviceSelect::Unique(nullptr, t2, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int32_t*)nullptr, (int)total);
  const size_t temp = t1 > t2 ? t1 : t2;
  return align_up(temp, 256) + 2 * align_up((size_t)total * 8, 256) + 2048;
}

extern "C" int b2_knn_graph_build(const int32_t* knn_idx, int32_t n, int32_t k, int32_t* rowptr, int32_t* colidx,
                                  float* vals_norm, int64_t capacity, int64_t* nnz_out_host, void* workspace,
                                  size_t workspace_bytes, void* stream) {
  B2_REQUIRE(knn_idx && rowptr && colidx && vals_norm && nnz_out_host, "b2_knn_graph_build: null pointer");
  B2_REQUIRE(n > 0 && k > 0, "b2_knn_graph_build: n and k must be positive");
  const int64_t total = 2ll * n * k + n;
  B2_REQUIRE(total < (1ll << 31), "b2_knn_graph_build: 2nk+n must be < 2^31");
  B2_REQUIRE(workspace && workspace_bytes >= b2_knn_graph_workspace_bytes(n, k),
             "b2_knn_graph_build: workspace too small");
  cudaStream_t st = as_stream(stream);
  WsCarver ws(workspace, workspace_bytes);
  uint64_t* keys = ws.take<uint64_t>(total);
  uint64_t* keys2 = ws.take<uint64_t>(total);
  int32_t* d_num = ws.take<int32_t>(4);
  size_t t1 = 0, t2 = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, t1, keys, keys2, (int)total);
  cub::DeviceSelect::Unique(nullptr, t2, keys2, keys, d_num, (int)total);
  size_t temp = t1 > t2 ? t1 : t2;
  void* d_temp = ws.take<char>(temp);
  if (!ws.ok()) { set_error("b2_knn_graph_build: workspace carve overflow"); return B2_ERR_WORKSPACE; }

  knn_edge_keys_kernel<<<grid_blocks((int64_t)n * k + n, 256, 32), 256, 0, st>>>(knn_idx, n, k, keys);
  B2_CHECK_LAUNCH("knn_edge_keys_kernel");
  B2_CHECK_CUDA(cub::DeviceRadixSort::SortKeys(d_temp, temp, keys, keys2, (int)total, 0, 32 + bits_for(n), st));
  B2_CHECK_CUDA(cub::DeviceSelect::Unique(d_temp, temp, keys2, keys, d_num, (int)total, st));
  int32_t h_num = 0;
  B2_CHECK_CUDA(cudaMemcpyAsync(&h_num, d_num, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  B2_CHECK_CUDA(cudaStreamSynchronize(st));
  *nnz_out_host = h_num;
  if ((int64_t)h_num > capacity) {
    set_error("b2_knn_graph_build: capacity %lld < nnz %d", (long long)capacity, h_num);
    return B2_ERR_WORKSPACE;
  }
  knn_rowptr_kernel<<<grid_blocks((int64_t)n + 1, 256, 32), 256, 0, st>>>(keys, d_num, n, rowptr);
  B2_CHECK_LAUNCH("knn_rowptr_kernel");
  knn_fill_kernel<<<grid_blocks(n, 256, 32), 256, 0, st>>>(keys, rowptr, n, colidx, vals_norm);
  B2_CHECK_LAUNCH("knn_fill_kernel");
  return B2_OK;
}

extern "C" size_t b2_knn_graph_weighted_workspace_bytes(int32_t n, int32_t k) {
  const int64_t total = (int64_t)n * k + n;
  size_t t1 = 0, t2 = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, t1, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int32_t*)nullptr,
                                  (int32_t*)nullptr, (int)total);
  cub::DeviceReduce::Sum(nullptr, t2, (const double*)nullptr, (double*)nullptr, n);
  const size_t temp = t1 > t2 ? t1 : t2;
  return align_up(temp, 256) + 2 * align_up((size_t)total * 8, 256) + 2 * align_up((size_t)total * 4, 256) +
         2 * align_up((size_t)n * 8, 256) + 4096;
}

extern "C" int b2_knn_graph_weighted_build(const int32_t* knn_idx, const double* knn_dist, int32_t n, int32_t k, int32_t* rowptr,
                                           int32_t* colidx, float* y, float* norm_t, int32_t* t_rowptr, int32_t* t_colidx, float* t_y,
                                           float* norm, double* sum_w, int64_t capacity, int64_t* nnz_out_host, void* workspace,
                                           size_t workspace_bytes, void* stream) {
  B2_REQUIRE(knn_idx && knn_dist && rowptr && colidx && y && norm_t && t_rowptr && t_colidx && t_y && norm && sum_w && nnz_out_host,
             "b2_knn_graph_weighted_build: null pointer");
  B2_REQUIRE(n > 0 && k > 0, "b2_knn_graph_weighted_build: n and k must be positive");
  const int64_t total = (int64_t)n * k + n;
  B2_REQUIRE(total < (1ll << 31), "b2_knn_graph_weighted_build: nk+n must be < 2^31");
  B2_REQUIRE(capacity >= total, "b2_knn_graph_weighted_build: capacity %lld < n*(k+1) = %lld", (long long)capacity, (long long)total);
  B2_REQUIRE(workspace && workspace_bytes >= b2_knn_graph_weighted_workspace_bytes(n, k),
             "b2_knn_graph_weighted_build: workspace too small");
  cudaStream_t st = as_stream(stream);
  WsCarver ws(workspace, workspace_bytes);
  uint64_t* keys = ws.take<uint64_t>(total);
  uint64_t* keys_sorted = ws.take<uint64_t>(total);
  int32_t* slots = ws.take<int32_t>(total);
  int32_t* slots_sorted = ws.take<int32_t>(total);
  double* dm = ws.take<double>(n);
  double* w_row = ws.take<double>(n);
  int32_t* flags = ws.take<int32_t>(2);   // [0] an index out of range, [1] a neighbour listed twice
  size_t t1 = 0, t2 = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, t1, keys, keys_sorted, slots, slots_sorted, (int)total);
  cub::DeviceReduce::Sum(nullptr, t2, w_row, sum_w, n);
  size_t temp = t1 > t2 ? t1 : t2;
  void* d_temp = ws.take<char>(temp);
  if (!ws.ok()) { set_error("b2_knn_graph_weighted_build: workspace carve overflow"); return B2_ERR_WORKSPACE; }
  B2_CHECK_CUDA(cudaMemsetAsync(flags, 0, 2 * sizeof(int32_t), st));
  const int key_bits = 32 + bits_for((int64_t)n + 1);
  for (int pass = 0; pass < 2; ++pass) {   // 0: L by source row, 1: Lᵀ by target row
    const bool by_target = pass == 1;
    int32_t* rp = by_target ? t_rowptr : rowptr;
    knn_weighted_keys_kernel<<<grid_blocks(total, 256, 32), 256, 0, st>>>(knn_idx, n, k, by_target, keys, slots, flags);
    B2_CHECK_LAUNCH("knn_weighted_keys_kernel");
    // LSD radix sort is stable, but every kept key is distinct, so the order within a row is the column order alone
    B2_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(d_temp, temp, keys, keys_sorted, slots, slots_sorted, (int)total, 0, key_bits, st));
    knn_weighted_rowptr_kernel<<<grid_blocks((int64_t)n + 1, 256, 32), 256, 0, st>>>(keys_sorted, total, n, rp);
    B2_CHECK_LAUNCH("knn_weighted_rowptr_kernel");
    sorted_keys_duplicate_kernel<<<grid_blocks(total, 256, 32), 256, 0, st>>>(keys_sorted, rp, n, flags + 1);
    B2_CHECK_LAUNCH("sorted_keys_duplicate_kernel");
    if (!by_target) {
      knn_weighted_rowsum_kernel<<<grid_blocks(n, 256, 32), 256, 0, st>>>(rp, keys_sorted, slots_sorted, knn_dist, n, k, dm, w_row);
      B2_CHECK_LAUNCH("knn_weighted_rowsum_kernel");
      B2_CHECK_CUDA(cub::DeviceReduce::Sum(d_temp, temp, w_row, sum_w, n, st));   // ΣW = adj_train.sum() (scgnn2.py:567)
    }
    knn_weighted_fill_kernel<<<grid_blocks(n, 256, 32), 256, 0, st>>>(rp, keys_sorted, slots_sorted, knn_dist, dm, n, k, by_target,
                                                                      by_target ? t_colidx : colidx, by_target ? t_y : y,
                                                                      by_target ? norm : norm_t);
    B2_CHECK_LAUNCH("knn_weighted_fill_kernel");
  }
  int32_t h_flags[2] = {0, 0}, h_nnz[2] = {0, 0};
  B2_CHECK_CUDA(cudaMemcpyAsync(h_flags, flags, 2 * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  B2_CHECK_CUDA(cudaMemcpyAsync(&h_nnz[0], rowptr + n, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  B2_CHECK_CUDA(cudaMemcpyAsync(&h_nnz[1], t_rowptr + n, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  B2_CHECK_CUDA(cudaStreamSynchronize(st));
  *nnz_out_host = h_nnz[0];
  if (h_flags[0]) { set_error("b2_knn_graph_weighted_build: knn_idx holds an index outside [0, %d)", n); return B2_ERR_INVALID; }
  if (h_flags[1]) { set_error("b2_knn_graph_weighted_build: a row of knn_idx lists the same neighbour twice"); return B2_ERR_INVALID; }
  if (h_nnz[0] != h_nnz[1]) { set_error("b2_knn_graph_weighted_build: internal error (nnz %d vs %d)", h_nnz[0], h_nnz[1]); return B2_ERR_INVALID; }
  return B2_OK;
}
