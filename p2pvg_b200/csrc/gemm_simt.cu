// CUDA-core GEMM (fp32 accumulate) used by the fp32 parity mode, by the LSTM path, and as the
// bisecting fallback for the wgmma GEMM (P2PVG_GEMM=simt).  Handles every shape / leading
// dimension / operand major-ness without alignment requirements.
//
//   C[M,N] = (accumulate ? C : 0) + opA(A) * opB(B) + bias[n] + addend[m,n]
//   a_mn = 0: A[m*lda + k] (K-major)       a_mn = 1: A[k*lda + m] (MN-major)
//   b_mn = 0: B[n*ldb + k] (K-major)       b_mn = 1: B[k*ldb + n] (MN-major)
#include "common.cuh"

namespace {

constexpr int BM = 64, BN = 64, BK = 16, PAD = 4;

template <typename TI, typename TO>
__global__ void __launch_bounds__(256) gemm_simt_kernel(const TI* __restrict__ A, int a_mn, long long lda,
                                                        const TI* __restrict__ B, int b_mn, long long ldb,
                                                        TO* __restrict__ C, long long ldc, int M, int N, int K,
                                                        int accumulate, const float* __restrict__ bias,
                                                        const TO* __restrict__ addend, long long ldd,
                                                        float* __restrict__ partial, int k_per_split) {
  __shared__ __align__(16) float As[BK][BM + PAD];
  __shared__ __align__(16) float Bs[BK][BN + PAD];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const long long m0 = (long long)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) acc[i][j] = 0.f;

  const int kbeg = blockIdx.z * k_per_split;
  const int kend = min(K, kbeg + k_per_split);
  K = kend;  // loads beyond this split's range read as zero
  for (int k0 = kbeg; k0 < kend; k0 += BK) {
    // ---- stage A tile (BM x BK) ----
#pragma unroll
    for (int i = 0; i < 4; i++) {
      int mm, kk;
      if (a_mn) { mm = tid & 63; kk = (tid >> 6) + 4 * i; }
      else      { kk = tid & 15; mm = (tid >> 4) + 16 * i; }
      long long gm = m0 + mm;
      int gk = k0 + kk;
      float v = 0.f;
      if (gm < M && gk < K) v = ld_f<TI>(a_mn ? &A[(long long)gk * lda + gm] : &A[gm * lda + gk]);
      As[kk][mm] = v;
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
      int nn, kk;
      if (b_mn) { nn = tid & 63; kk = (tid >> 6) + 4 * i; }
      else      { kk = tid & 15; nn = (tid >> 4) + 16 * i; }
      int gn = n0 + nn;
      int gk = k0 + kk;
      float v = 0.f;
      if (gn < N && gk < K) v = ld_f<TI>(b_mn ? &B[(long long)gk * ldb + gn] : &B[(long long)gn * ldb + gk]);
      Bs[kk][nn] = v;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; kk++) {
      float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
      float av[4] = {a.x, a.y, a.z, a.w};
      float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; i++) {
    long long gm = m0 + ty * 4 + i;
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      int gn = n0 + tx * 4 + j;
      if (gn >= N) continue;
      float v = acc[i][j];
      if (partial) {  // split-K: raw partial sums, finished by p2pvg_splitk_reduce
        partial[((long long)blockIdx.z * M + gm) * N + gn] = v;
        continue;
      }
      if (bias) v += bias[gn];
      if (addend) v += ld_f<TO>(&addend[gm * ldd + gn]);
      if (accumulate) v += ld_f<TO>(&C[gm * ldc + gn]);
      st_f<TO>(&C[gm * ldc + gn], v);
    }
  }
}

}  // namespace

int p2pvg_gemm_simt(const void* A, int in_dtype, int a_mn, long long lda, const void* B, int b_mn, long long ldb, void* C,
                    int c_dtype, long long ldc, int M, int N, int K, int accumulate, const float* bias,
                    const void* addend, long long ldd, void* workspace, size_t ws_bytes, cudaStream_t stream) {
  if (M <= 0 || N <= 0) return P2PVG_OK;
  dim3 grid(cdiv(M, BM), cdiv(N, BN));
  // split-K (deterministic two-pass) for small outputs with a long reduction, e.g. the Linear weight gradients
  int splits = 1, k_per_split = K > 0 ? K : 1;
  const long long tiles = (long long)grid.x * grid.y;
  if (tiles < 74 && K >= 2048 && workspace != nullptr) {
    long long want = (296 + tiles - 1) / tiles;
    long long maxs = K / 256;
    splits = (int)(want < maxs ? want : maxs);
    while (splits > 1 && (size_t)splits * M * N * sizeof(float) > ws_bytes) splits /= 2;
    if (splits < 1) splits = 1;
    k_per_split = ((cdiv(K, splits) + BK - 1) / BK) * BK;
    splits = cdiv(K, k_per_split);
  }
  grid.z = splits;
  float* partial = splits > 1 ? reinterpret_cast<float*>(workspace) : nullptr;
  P2PVG_REQUIRE(grid.y <= 65535, P2PVG_ERR_UNSUPPORTED, "gemm_simt: N=%d too large", N);
#define LAUNCH(TI, TO)                                                                                              \
  gemm_simt_kernel<TI, TO><<<grid, 256, 0, stream>>>((const TI*)A, a_mn, lda, (const TI*)B, b_mn, ldb, (TO*)C, ldc, \
                                                     M, N, K, accumulate, bias, (const TO*)addend, ldd, partial, k_per_split)
  if (in_dtype == P2PVG_F32 && c_dtype == P2PVG_F32) LAUNCH(float, float);
  else if (in_dtype == P2PVG_BF16 && c_dtype == P2PVG_F32) LAUNCH(bf16, float);
  else if (in_dtype == P2PVG_BF16 && c_dtype == P2PVG_BF16) LAUNCH(bf16, bf16);
  else if (in_dtype == P2PVG_F32 && c_dtype == P2PVG_BF16) LAUNCH(float, bf16);
  else {
    p2pvg_set_error("gemm_simt: bad dtypes %d/%d", in_dtype, c_dtype);
    return P2PVG_ERR_BAD_ARG;
  }
#undef LAUNCH
  if (splits > 1) return p2pvg_splitk_reduce(partial, splits, C, c_dtype, ldc, M, N, accumulate, bias, addend, ldd, 0, stream);
  return p2pvg_check_launch("gemm_simt");
}
