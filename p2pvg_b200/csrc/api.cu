// Library-wide state of libp2pvg_b200.so (include/p2pvg_b200.h): the thread-local error string, the GEMM implementation
// override and p2pvg_gemm's dispatch between the wgmma and CUDA-core kernels.  Every other entry point is defined in the
// file whose kernels it launches.
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

static thread_local char g_err[512] = "";

void p2pvg_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int p2pvg_check_launch(const char* what) {
  cudaError_t e = cudaPeekAtLastError();
  if (e != cudaSuccess) {
    p2pvg_set_error("%s: %s", what, cudaGetErrorString(e));
    (void)cudaGetLastError();
    return P2PVG_ERR_CUDA;
  }
  return P2PVG_OK;
}

static int g_gemm_impl = 0;  // 0 auto, 1 simt, 2 wgmma
int p2pvg_gemm_impl_forced() { return g_gemm_impl; }

extern "C" int p2pvg_version(void) { return 201; }
extern "C" const char* p2pvg_last_error(void) { return g_err; }
extern "C" int p2pvg_has_tc_gemm(void) { return p2pvg_gemm_tc_available(); }
extern "C" int p2pvg_set_gemm_impl(int impl) {
  if (impl < 0 || impl > 2) return P2PVG_ERR_BAD_ARG;
  g_gemm_impl = impl;
  return P2PVG_OK;
}

extern "C" int p2pvg_gemm(const void* A, int in_dtype, int a_mn, int64_t lda, const void* B, int b_mn, int64_t ldb, void* C,
                          int c_dtype, int64_t ldc, int M, int N, int K, int accumulate, const float* bias, const void* addend,
                          int64_t ldd, void* workspace, size_t ws_bytes, int flags, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  P2PVG_REQUIRE(A && B && C, P2PVG_ERR_BAD_ARG, "gemm: null operand");
  P2PVG_REQUIRE(M >= 0 && N >= 0 && K >= 0, P2PVG_ERR_BAD_ARG, "gemm: negative size");
  bool want_tc = (in_dtype == P2PVG_BF16) && g_gemm_impl != 1;
  // fp32 operands (LSTM / parity mode) always run on the CUDA cores; "forced wgmma" only makes the bf16 path
  // refuse to fall back when an operand is not TMA-compatible.
  if (want_tc)
    return p2pvg_gemm_tc(A, a_mn, lda, B, b_mn, ldb, C, c_dtype, ldc, M, N, K, accumulate, bias, addend, ldd, workspace, ws_bytes, st);
  if (in_dtype == P2PVG_F32 && (flags & P2PVG_GEMM_TF32) && g_gemm_impl != 1) {
    // documented dispatch (include/p2pvg_b200.h): TF32 tensor cores for K-major TMA-compatible operands, the exact
    // CUDA-core kernel otherwise -- unless the caller asked for an error instead
    int rc = P2PVG_ERR_UNSUPPORTED;
    if (!a_mn && !b_mn && K >= 32) rc = p2pvg_gemm_tf32(A, lda, B, ldb, C, c_dtype, ldc, M, N, K, accumulate, bias, addend, ldd, st);
    if (rc != P2PVG_ERR_UNSUPPORTED) return rc;
    if (flags & P2PVG_GEMM_TF32_REQUIRE) {
      p2pvg_set_error("gemm: fp32 operands not eligible for the TF32 tensor-core kernel (need K-major, K >= 32, 16-byte aligned bases / pitches): M=%d N=%d K=%d a_mn=%d b_mn=%d",
                      M, N, K, a_mn, b_mn);
      return P2PVG_ERR_UNSUPPORTED;
    }
  }
  return p2pvg_gemm_simt(A, in_dtype, a_mn, lda, B, b_mn, ldb, C, c_dtype, ldc, M, N, K, accumulate, bias, addend, ldd, workspace,
                         ws_bytes, st);
}
