// Error plumbing + device queries for the C-ABI.
#include "common.cuh"

#include <string.h>

#include <atomic>
#include <mutex>
#include <unordered_map>

namespace b2 {

static thread_local char g_err[512] = "";
long long g_launch_count = 0;

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what) {
  set_error("CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
  return B2_ERR_CUDA;
}

// Per-device caches (sm_count, allow_dynamic_smem) hold devices 0 .. CACHED_DEVICES - 1; a device past them is queried, or
// opted in, on every call.
constexpr int CACHED_DEVICES = 16;
static bool cached_device(int dev) { return dev >= 0 && dev < CACHED_DEVICES; }

int sm_count() {
  static std::atomic<int> cached[CACHED_DEVICES];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 148;
  if (cached_device(dev)) {
    const int n = cached[dev].load(std::memory_order_relaxed);
    if (n > 0) return n;
  }
  int n = 0;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 148;
  if (cached_device(dev)) cached[dev].store(n, std::memory_order_relaxed);
  return n;
}

int allow_dynamic_smem(const void* kernel, size_t bytes) {
  if (bytes <= 48 * 1024) return B2_OK;
  int dev = 0;
  B2_CHECK_CUDA(cudaGetDevice(&dev));
  static std::mutex mu;
  static std::unordered_map<const void*, size_t> allowed[CACHED_DEVICES];   // per device: kernel → largest size opted into
  std::lock_guard<std::mutex> lock(mu);
  if (cached_device(dev)) {
    const auto it = allowed[dev].find(kernel);
    if (it != allowed[dev].end() && it->second >= bytes) return B2_OK;
  }
  B2_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  if (cached_device(dev)) allowed[dev][kernel] = bytes;
  return B2_OK;
}

const char* last_error() { return g_err; }

// kernel-path selectors (b2_set_path): every selectable path computes the same result, the switch exists for A/B tests
static int g_path[B2_PATH_COUNT] = {0, 0, 0};
int path_mode(int which) { return (which >= 0 && which < B2_PATH_COUNT) ? g_path[which] : 0; }

// scheduling knobs of the tensor-core decoder (b2_set_tuning): they move work in time, never change a result
static int g_tune[B2_TUNE_COUNT] = {0};
int tuning(int which) { return (which >= 0 && which < B2_TUNE_COUNT) ? g_tune[which] : 0; }

}  // namespace b2

extern "C" {

const char* b2_last_error(void) { return b2::last_error(); }

int b2_version(void) { return 101; }

int64_t b2_launch_count(void) { return (int64_t)b2::g_launch_count; }

int b2_set_path(int which, int mode) {
  B2_REQUIRE(which >= 0 && which < B2_PATH_COUNT, "b2_set_path: unknown selector %d", which);
  const bool ok = which == B2_PATH_GAE_DECODER ? mode >= 0 && mode <= 2 : mode == 0 || mode == 1;
  B2_REQUIRE(ok, "b2_set_path: mode %d out of range for selector %d", mode, which);
  b2::g_path[which] = mode;
  return B2_OK;
}

int b2_get_path(int which) { return b2::path_mode(which); }

int b2_set_tuning(int which, int value) {
  B2_REQUIRE(which >= 0 && which < B2_TUNE_COUNT, "b2_set_tuning: unknown knob %d", which);
  B2_REQUIRE(value >= 0 && value <= 1000000, "b2_set_tuning: value %d out of range", value);
  b2::g_tune[which] = value;
  return B2_OK;
}

int b2_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  int dev = 0;
  B2_CHECK_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp p;
  B2_CHECK_CUDA(cudaGetDeviceProperties(&p, dev));
  if (sm_count) *sm_count = p.multiProcessorCount;
  if (cc_major) *cc_major = p.major;
  if (cc_minor) *cc_minor = p.minor;
  return B2_OK;
}

}  // extern "C"
