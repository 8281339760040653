// Issue cost of single wgmma instructions on sm_90a, for the small-N shapes of the decoder's gradient products.
//
// One CTA per SM, one or two warpgroups per CTA.  Each warpgroup issues REPS batches of BATCH wgmmas of one shape (round-robin
// into NACC accumulators, so that consecutive instructions do not depend on each other), one commit and one wait per batch,
// and times the whole loop with clock64.  Operands: K-major, 128-byte swizzle (the decoder's layout); A from shared memory
// (SS) or from registers (RS).  Prints one line per shape:
//   <dtype> <form> <n> <warpgroups> <clocks per wgmma per warpgroup> <clocks per wgmma per SM> <SM clock MHz>
// Built and run by benchmarks/wgmma_rate.py; not part of the library.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <algorithm>
#include <vector>

constexpr int BATCH = 32, NACC = 4, REPS = 4096;

__device__ __forceinline__ uint64_t desc_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

#define D8(o) "+f"(d[o + 0]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), "+f"(d[o + 6]), "+f"(d[o + 7])
#define R8 "%0, %1, %2, %3, %4, %5, %6, %7"
#define R16 R8 ", %8, %9, %10, %11, %12, %13, %14, %15"
#define R32 R16 ", %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"

// tf32 m64nNk8 and f16 m64nNk16, fp32 accumulators, scale-d = 1
#define WGMMA_SS(NAME, SHAPE, TYPE, REGS, NR, TAIL, ...)                                                                 \
  __device__ __forceinline__ void NAME(float (&d)[NR], uint64_t a, uint64_t b) {                                        \
    asm volatile("wgmma.mma_async.sync.aligned." SHAPE ".f32." TYPE "." TYPE " {" REGS "}, %" #NR ", %" NR_PLUS1_##NR \
                 ", 1, 1, 1" TAIL ";\n" : __VA_ARGS__ : "l"(a), "l"(b));                                               \
  }
#define NR_PLUS1_8 "9"
#define NR_PLUS1_16 "17"
#define NR_PLUS1_32 "33"
#define WGMMA_RS(NAME, SHAPE, TYPE, REGS, NR, TAIL, ...)                                                                 \
  __device__ __forceinline__ void NAME(float (&d)[NR], const uint32_t (&a)[4], uint64_t b) {                            \
    asm volatile("wgmma.mma_async.sync.aligned." SHAPE ".f32." TYPE "." TYPE " {" REGS "}, {%" #NR ", %" NR_PLUS1_##NR \
                 ", %" NR_PLUS2_##NR ", %" NR_PLUS3_##NR "}, %" NR_PLUS4_##NR ", 1, 1, 1" TAIL ";\n"                    \
                 : __VA_ARGS__ : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b));                                  \
  }
#define NR_PLUS2_8 "10"
#define NR_PLUS3_8 "11"
#define NR_PLUS4_8 "12"
#define NR_PLUS2_16 "18"
#define NR_PLUS3_16 "19"
#define NR_PLUS4_16 "20"
#define NR_PLUS2_32 "34"
#define NR_PLUS3_32 "35"
#define NR_PLUS4_32 "36"

// tf32 takes no transpose immediates; f16 SS takes trans-a and trans-b, f16 RS trans-b only (0: K-major)
WGMMA_SS(tf32_ss_16, "m64n16k8", "tf32", R8, 8, "", D8(0))
WGMMA_SS(tf32_ss_32, "m64n32k8", "tf32", R16, 16, "", D8(0), D8(8))
WGMMA_SS(tf32_ss_64, "m64n64k8", "tf32", R32, 32, "", D8(0), D8(8), D8(16), D8(24))
WGMMA_SS(f16_ss_16, "m64n16k16", "f16", R8, 8, ", 0, 0", D8(0))
WGMMA_SS(f16_ss_32, "m64n32k16", "f16", R16, 16, ", 0, 0", D8(0), D8(8))
WGMMA_SS(f16_ss_64, "m64n64k16", "f16", R32, 32, ", 0, 0", D8(0), D8(8), D8(16), D8(24))
WGMMA_RS(tf32_rs_16, "m64n16k8", "tf32", R8, 8, "", D8(0))
WGMMA_RS(tf32_rs_32, "m64n32k8", "tf32", R16, 16, "", D8(0), D8(8))
WGMMA_RS(tf32_rs_64, "m64n64k8", "tf32", R32, 32, "", D8(0), D8(8), D8(16), D8(24))
WGMMA_RS(f16_rs_16, "m64n16k16", "f16", R8, 8, ", 0", D8(0))
WGMMA_RS(f16_rs_32, "m64n32k16", "f16", R16, 16, ", 0", D8(0), D8(8))
WGMMA_RS(f16_rs_64, "m64n64k16", "f16", R32, 32, ", 0", D8(0), D8(8), D8(16), D8(24))

template <bool F16, bool RS, int N>
__device__ __forceinline__ void mma(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t ad, uint64_t bd) {
#define PICK(P, A) \
  if constexpr (N == 16) P##_16(d, A, bd); else if constexpr (N == 32) P##_32(d, A, bd); else P##_64(d, A, bd);
  if constexpr (F16 && RS) { PICK(f16_rs, a) }
  else if constexpr (RS) { PICK(tf32_rs, a) }
  else if constexpr (F16) { PICK(f16_ss, ad) }
  else { PICK(tf32_ss, ad) }
#undef PICK
}

template <bool F16, bool RS, int N>
__global__ void __launch_bounds__(256, 1) rate_kernel(int wgs, long long* clocks, float* sink) {
  __shared__ __align__(1024) uint32_t buf[2 * 64 * 32];   // A: 64 rows x 128 B, B: 64 rows x 128 B
  const int tid = threadIdx.x;
  for (int i = tid; i < 2 * 64 * 32; i += blockDim.x) buf[i] = F16 ? 0x3C003C00u >> (i & 1) : 0x3F800000u >> (i & 1);
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  if (tid >= 128 * wgs) return;
  const uint32_t base = (uint32_t)__cvta_generic_to_shared(buf);
  const uint64_t ad = desc_sw128(base), bd = desc_sw128(base + 64 * 128);
  uint32_t a[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) a[i] = buf[(tid * 4 + i) & 4095];
  float acc[NACC][N / 2];
#pragma unroll
  for (int k = 0; k < NACC; ++k)
#pragma unroll
    for (int v = 0; v < N / 2; ++v) acc[k][v] = 0.f;
  asm volatile("bar.sync 1, %0;" ::"r"(128 * wgs) : "memory");
  const long long t0 = clock64();
#pragma unroll 1
  for (int r = 0; r < REPS; ++r) {
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
    for (int b = 0; b < BATCH; ++b) mma<F16, RS, N>(acc[b % NACC], a, ad, bd);
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
  }
  const long long t1 = clock64();
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < NACC; ++k)
#pragma unroll
    for (int v = 0; v < N / 2; ++v) s += acc[k][v];
  if (s == 12345.f) sink[tid] = s;   // keeps the products live
  if ((tid & 127) == 0) clocks[blockIdx.x * 2 + tid / 128] = t1 - t0;
}

template <bool F16, bool RS, int N>
static void run(int sms, int wgs, long long* clocks, float* sink) {
  auto k = rate_kernel<F16, RS, N>;
  for (int it = 0; it < 2; ++it) k<<<sms, 128 * wgs>>>(wgs, clocks, sink);   // warm-up
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  cudaEventRecord(e0);
  k<<<sms, 128 * wgs>>>(wgs, clocks, sink);
  cudaEventRecord(e1);
  cudaError_t err = cudaEventSynchronize(e1);
  if (err != cudaSuccess) { fprintf(stderr, "CUDA error: %s\n", cudaGetErrorString(err)); exit(1); }
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e0, e1);
  std::vector<long long> h(2 * sms);
  cudaMemcpy(h.data(), clocks, sizeof(long long) * 2 * sms, cudaMemcpyDeviceToHost);
  std::vector<long long> c;
  for (int b = 0; b < sms; ++b)
    for (int w = 0; w < wgs; ++w) c.push_back(h[2 * b + w]);
  std::sort(c.begin(), c.end());
  const double med = (double)c[c.size() / 2];
  const double per_wg = med / ((double)REPS * BATCH);
  printf("%s %s %d %d %.3f %.3f %.0f\n", F16 ? "f16" : "tf32", RS ? "rs" : "ss", N, wgs, per_wg, per_wg / wgs,
         med / (ms * 1e3));
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
}

template <bool F16, bool RS>
static void shapes(int sms, long long* clocks, float* sink) {
  for (int wgs = 1; wgs <= 2; ++wgs) {
    run<F16, RS, 16>(sms, wgs, clocks, sink);
    run<F16, RS, 32>(sms, wgs, clocks, sink);
    run<F16, RS, 64>(sms, wgs, clocks, sink);
  }
}

int main() {
  int sms = 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0) != cudaSuccess || sms == 0) {
    fprintf(stderr, "no CUDA device\n");
    return 1;
  }
  long long* clocks;
  float* sink;
  cudaMalloc(&clocks, sizeof(long long) * 2 * sms);
  cudaMalloc(&sink, sizeof(float) * 256);
  shapes<false, false>(sms, clocks, sink);
  shapes<false, true>(sms, clocks, sink);
  shapes<true, false>(sms, clocks, sink);
  shapes<true, true>(sms, clocks, sink);
  cudaFree(clocks);
  cudaFree(sink);
  return 0;
}
