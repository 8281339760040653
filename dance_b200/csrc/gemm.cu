// b2_gemm_f32 dispatcher: tensor-core wgmma (TF32 / 3xTF32 / BF16) kernel when the shape qualifies,
// CUDA-core fp32 kernel otherwise (or when B2_PREC_FP32_SIMT is requested).
#include "common.cuh"

namespace b2 {
int gemm_simt(const float* A, int64_t lda, int transA, const float* B, int64_t ldb, int transB, float* C,
              int64_t ldc, int M, int N, int K, const float* bias, int act, const float* mask, int64_t ldmask,
              float beta, cudaStream_t st);
// returns B2_ERR_UNSUPPORTED (without setting an error) when the shape/alignment does not qualify
int gemm_tc(const float* A, int64_t lda, int transA, const float* B, int64_t ldb, int transB, float* C, int64_t ldc,
            int M, int N, int K, const float* bias, int act, const float* mask, int64_t ldmask, float beta,
            int precision, void* workspace, size_t workspace_bytes, cudaStream_t st);
size_t gemm_tc_workspace_bytes(int M, int N, int K, int transA, int transB, int precision);
}  // namespace b2

using namespace b2;

extern "C" size_t b2_gemm_workspace_bytes(int M, int N, int K, int transA, int transB, int precision) {
  if (precision == B2_PREC_FP32_SIMT) return 0;
  return gemm_tc_workspace_bytes(M, N, K, transA, transB, precision);
}

extern "C" int b2_gemm_f32(const float* A, int64_t lda, int transA, const float* B, int64_t ldb, int transB, float* C,
                           int64_t ldc, int M, int N, int K, const float* bias, int act, const float* mask,
                           int64_t ldmask, float beta, int precision, void* workspace, size_t workspace_bytes,
                           void* stream) {
  B2_REQUIRE(A && B && C, "b2_gemm_f32: null pointer");
  B2_REQUIRE(M >= 0 && N >= 0 && K >= 0, "b2_gemm_f32: negative shape");
  B2_REQUIRE(lda >= (transA ? M : K) && ldb >= (transB ? K : N) && ldc >= N, "b2_gemm_f32: leading dimension too small");
  B2_REQUIRE(!mask || ldmask >= N, "b2_gemm_f32: ldmask too small");
  B2_REQUIRE(precision == B2_PREC_FP32_SIMT || precision == B2_PREC_TF32X3 || precision == B2_PREC_TF32 ||
                 precision == B2_PREC_BF16,
             "b2_gemm_f32: unknown precision %d", precision);
  B2_REQUIRE(beta == 0.f || beta == 1.f, "b2_gemm_f32: beta must be 0 or 1");
  if (M == 0 || N == 0) return B2_OK;
  cudaStream_t st = as_stream(stream);
  if (precision != B2_PREC_FP32_SIMT) {
    const int rc = gemm_tc(A, lda, transA, B, ldb, transB, C, ldc, M, N, K, bias, act, mask, ldmask, beta, precision,
                           workspace, workspace_bytes, st);
    if (rc != B2_ERR_UNSUPPORTED) return rc;
  }
  return gemm_simt(A, lda, transA, B, ldb, transB, C, ldc, M, N, K, bias, act, mask, ldmask, beta, st);
}
