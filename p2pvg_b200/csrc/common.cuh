// Shared helpers for the p2pvg_b200 sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>

// error codes, dtypes, activations and the extern "C" entry points every .cu file defines against
#include "../../include/p2pvg_b200.h"

// thread-local error string (C ABI: p2pvg_last_error)
void p2pvg_set_error(const char* fmt, ...);
int p2pvg_check_launch(const char* what);

#define P2PVG_REQUIRE(cond, code, ...)      \
  do {                                      \
    if (!(cond)) {                          \
      p2pvg_set_error(__VA_ARGS__);         \
      return (code);                        \
    }                                       \
  } while (0)

typedef __nv_bfloat16 bf16;

template <typename T> __device__ __forceinline__ float ld_f(const T* p);
template <> __device__ __forceinline__ float ld_f<float>(const float* p) { return *p; }
template <> __device__ __forceinline__ float ld_f<bf16>(const bf16* p) { return __bfloat162float(*p); }
template <typename T> __device__ __forceinline__ void st_f(T* p, float v);
template <> __device__ __forceinline__ void st_f<float>(float* p, float v) { *p = v; }
template <> __device__ __forceinline__ void st_f<bf16>(bf16* p, float v) { *p = __float2bfloat16_rn(v); }

// 4-wide vector access (16 B for float, 8 B for bf16).  Pointers must be aligned to the vector size.
struct f4 { float v[4]; };
template <typename T> __device__ __forceinline__ f4 ld_f4(const T* p);
template <> __device__ __forceinline__ f4 ld_f4<float>(const float* p) {
  float4 t = *reinterpret_cast<const float4*>(p);
  return f4{{t.x, t.y, t.z, t.w}};
}
template <> __device__ __forceinline__ f4 ld_f4<bf16>(const bf16* p) {
  uint2 t = *reinterpret_cast<const uint2*>(p);
  __nv_bfloat162 a = *reinterpret_cast<__nv_bfloat162*>(&t.x);
  __nv_bfloat162 b = *reinterpret_cast<__nv_bfloat162*>(&t.y);
  return f4{{__low2float(a), __high2float(a), __low2float(b), __high2float(b)}};
}
template <typename T> __device__ __forceinline__ void st_f4(T* p, const f4& x);
template <> __device__ __forceinline__ void st_f4<float>(float* p, const f4& x) {
  *reinterpret_cast<float4*>(p) = make_float4(x.v[0], x.v[1], x.v[2], x.v[3]);
}
template <> __device__ __forceinline__ void st_f4<bf16>(bf16* p, const f4& x) {
  __nv_bfloat162 a = __floats2bfloat162_rn(x.v[0], x.v[1]);
  __nv_bfloat162 b = __floats2bfloat162_rn(x.v[2], x.v[3]);
  uint2 t;
  t.x = *reinterpret_cast<uint32_t*>(&a);
  t.y = *reinterpret_cast<uint32_t*>(&b);
  *reinterpret_cast<uint2*>(p) = t;
}

// 16-byte vectors: 4 floats or 8 bf16.  VecN<T>::N elements per vector.
template <typename T> struct VecN;
template <> struct VecN<float> { static constexpr int N = 4; };
template <> struct VecN<bf16> { static constexpr int N = 8; };

__device__ __forceinline__ uint4 ld_raw16(const void* p) { return *reinterpret_cast<const uint4*>(p); }
__device__ __forceinline__ void st_raw16(void* p, uint4 v) { *reinterpret_cast<uint4*>(p) = v; }

template <typename T> __device__ __forceinline__ void unpack16(uint4 r, float* f);
template <> __device__ __forceinline__ void unpack16<float>(uint4 r, float* f) {
  f[0] = __uint_as_float(r.x); f[1] = __uint_as_float(r.y); f[2] = __uint_as_float(r.z); f[3] = __uint_as_float(r.w);
}
template <> __device__ __forceinline__ void unpack16<bf16>(uint4 r, float* f) {
  const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
  for (int i = 0; i < 4; i++) {  // bf16 -> fp32 is a 16-bit shift
    f[2 * i] = __uint_as_float(w[i] << 16);
    f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
  }
}
template <typename T> __device__ __forceinline__ uint4 pack16(const float* f);
template <> __device__ __forceinline__ uint4 pack16<float>(const float* f) {
  return make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]), __float_as_uint(f[3]));
}
template <> __device__ __forceinline__ uint4 pack16<bf16>(const float* f) {
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; i++) {
    __nv_bfloat162 p = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
    w[i] = *reinterpret_cast<uint32_t*>(&p);
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// Second pass of split-K (gemm_simt.cu, gemm_tc.cu, conv_gemm.cu), defined in gemm_tc.cu: C[M, N] = sum_z partial[z] + bias[n]
// + addend[m, n] + (accumulate ? C : 0), partial [splits][M][N] fp32, or [splits][N][M] when transposed; C and addend are
// c_dtype.  Deterministic: each element is summed by one thread in ascending z.
int p2pvg_splitk_reduce(const float* partial, int splits, void* C, int c_dtype, long long ldc, int M, int N, int accumulate,
                        const float* bias, const void* addend, long long ldd, int transposed, cudaStream_t st);

// The kernels behind p2pvg_gemm (api.cu).  gemm_simt.cu: CUDA cores, every dtype pair, exact fp32 accumulation.
int p2pvg_gemm_simt(const void* A, int in_dtype, int a_mn, long long lda, const void* B, int b_mn, long long ldb, void* C,
                    int c_dtype, long long ldc, int M, int N, int K, int accumulate, const float* bias, const void* addend,
                    long long ldd, void* workspace, size_t ws_bytes, cudaStream_t st);
// gemm_tc.cu: bf16 operands on wgmma; operands that are not TMA-compatible run on p2pvg_gemm_simt unless
// p2pvg_gemm_impl_forced() == 2 (P2PVG_ERR_UNSUPPORTED then).
int p2pvg_gemm_tc(const void* A, int a_mn, long long lda, const void* B, int b_mn, long long ldb, void* C, int c_dtype, long long ldc,
                  int M, int N, int K, int accumulate, const float* bias, const void* addend, long long ldd, void* workspace,
                  size_t ws_bytes, cudaStream_t st);
// gemm_tc.cu: K-major fp32 operands on wgmma .tf32; P2PVG_ERR_UNSUPPORTED when they are not TMA-compatible.
int p2pvg_gemm_tf32(const void* A, long long lda, const void* B, long long ldb, void* C, int c_dtype, long long ldc, int M, int N,
                    int K, int accumulate, const float* bias, const void* addend, long long ldd, cudaStream_t st);
int p2pvg_gemm_tc_available();
// p2pvg_set_gemm_impl's choice: 0 auto, 1 simt, 2 wgmma
int p2pvg_gemm_impl_forced();

// The thread-block-cluster LSTM scans behind p2pvg_lstm_scan_fwd / _bwd (lstm_scan.cu): clusters of 8 CTAs for the hidden
// sizes p2pvg_lstm_cluster_supported accepts (lstm_cluster.cu), clusters of 16 for R = 512 (lstm_cluster512.cu).
bool p2pvg_lstm_cluster_supported(int R);
int p2pvg_lstm_cluster_fwd(const float* pre, const float* whh, const float* bhh, float* gates, float* hs, float* cs, int S, int B,
                           int R, cudaStream_t st);
int p2pvg_lstm_cluster_bwd(const float* dhtop, const float* whh, const float* gates, const float* cs, float* dG, int S, int B, int R,
                           cudaStream_t st);
int p2pvg_lstm_cluster512_fwd(const float* pre, const float* whh, const float* bhh, float* gates, float* hs, float* cs, int S, int B,
                              cudaStream_t st);
int p2pvg_lstm_cluster512_bwd(const float* dhtop, const float* whh, const float* gates, const float* cs, float* dG, int S, int B,
                              cudaStream_t st);

#define DISPATCH_DTYPE(dt, T, ...)                                   \
  do {                                                               \
    if ((dt) == P2PVG_F32) { typedef float T; __VA_ARGS__; }         \
    else if ((dt) == P2PVG_BF16) { typedef bf16 T; __VA_ARGS__; }    \
    else { p2pvg_set_error("bad dtype %d", (int)(dt)); return P2PVG_ERR_BAD_ARG; } \
  } while (0)
