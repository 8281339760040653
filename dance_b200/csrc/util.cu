// Error plumbing + device queries for the C-ABI.
#include "common.cuh"

#include <string.h>

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

int sm_count() {
  static int cached[16] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 148;
  if (dev < 0 || dev >= 16) dev = 0;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 148;
    cached[dev] = n;
  }
  return cached[dev];
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

int b2_version(void) { return 100; }

int64_t b2_launch_count(void) { return (int64_t)b2::g_launch_count; }

int b2_set_path(int which, int mode) {
  B2_REQUIRE(which >= 0 && which < B2_PATH_COUNT, "b2_set_path: unknown selector %d", which);
  B2_REQUIRE(mode >= 0 && mode <= (which == B2_PATH_GAE_DECODER ? 2 : 1), "b2_set_path: mode %d out of range for selector %d", mode, which);
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
