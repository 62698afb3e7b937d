// bf16 GEMM on the Hopper tensor cores (sm_90a): TMA (cp.async.bulk.tensor) stages 128B-swizzled operand tiles in
// shared memory, one warpgroup issues wgmma.mma_async (fp32 accumulator in registers) and hands each finished tile to
// four epilogue warps through a shared-memory staging buffer; they add bias / addend and store.
//
//   C[M,N] = (accumulate ? C : 0) + opA(A)*opB(B) + bias[n] + addend[m,n]          (same contract as gemm_simt)
//
// Operands may be K-major (row = m or n, contiguous along k) or MN-major (row = k, contiguous along m / n);
// MN-major tiles are what the weight-gradient GEMMs (reduction over pixels of NHWC tensors) need, so no
// transposed copies of activations are ever materialised.  Split-K (grid.z) with a deterministic second
// pass covers the weight gradients, whose output is tiny and whose reduction dimension is huge.
//
// The persistent, warp-specialised skeleton (warp roles, MMA loop, epilogue reads and stores) is tc_common.cuh, shared
// with conv_gemm.cu.
#include "tc_common.cuh"

namespace {

using namespace tc;

// ------------------------------------------------------------------ the kernel

// The persistent skeleton of tc_common.cuh.  A tile is (split z, m-tile, n-tile) with the n-tile fastest, so CTAs running at
// the same time share the A rows in L2.
template <typename TIn, int BN, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, void* __restrict__ Cv,
               int c_bf16, long long ldc, int M, int N, int K, int accumulate, const float* __restrict__ bias,
               const void* __restrict__ addend, long long ldd, float* __restrict__ partial, int kb_per_split, int splits) {
  using C_ = Cfg<BN>;
  constexpr int ELEM = sizeof(TIn);
  constexpr int BLOCK_K = ROW_BYTES / ELEM;  // elements of K per pipeline stage (K-major) / rows per stage (MN-major)
  constexpr bool TF32 = (ELEM == 4);
  static_assert(!(TF32 && (A_MN || B_MN)), "tf32 path supports K-major operands only");
  extern __shared__ uint8_t smem_raw[];
  const Smem sm = smem_setup<BN>(smem_raw);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_m = (M + BLOCK_M - 1) / BLOCK_M, tiles_n = (N + BN - 1) / BN;
  const int tiles_mn = tiles_m * tiles_n;
  const int num_tiles = tiles_mn * splits;
  const int nkb_total = (K + BLOCK_K - 1) / BLOCK_K;

  if (warp >= 8) {
    // ===================== TMA producer =====================
    regs_producer();
    if (warp == 8 && lane == 0) {
      uint32_t it = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const int z = (splits == 1) ? 0 : t / tiles_mn, r = t - z * tiles_mn;   // fast path: no integer division without split-K
        const int mt_ = (tiles_n == 1) ? r : r / tiles_n;
        const int m0 = mt_ * BLOCK_M, n0 = (r - mt_ * tiles_n) * BN;
        const int kb0 = z * kb_per_split, kb1 = min(kb0 + kb_per_split, nkb_total);
        for (int kb = kb0; kb < kb1; kb++, it++) {
          const int s = it % C_::STAGES;
          const uint32_t ph = (it / C_::STAGES) & 1;
          mbar_wait(&sm.empty_bar[s], ph ^ 1);
          uint8_t* sa = sm.ring + s * C_::STAGE_BYTES;
          uint8_t* sb = sa + A_STAGE_BYTES;
          mbar_expect_tx(&sm.full_bar[s], C_::STAGE_BYTES);
          const int k0 = kb * BLOCK_K;
          if (A_MN) {
            tma_load_2d(&tmA, &sm.full_bar[s], sa, m0, k0);
            tma_load_2d(&tmA, &sm.full_bar[s], sa + BLOCK_K * 128, m0 + 64, k0);
          } else {
            tma_load_2d(&tmA, &sm.full_bar[s], sa, k0, m0);
          }
          if (B_MN) {
#pragma unroll
            for (int j = 0; j < BN / 64; j++) tma_load_2d(&tmB, &sm.full_bar[s], sb + j * BLOCK_K * 128, n0 + 64 * j, k0);
          } else {
            tma_load_2d(&tmB, &sm.full_bar[s], sb, k0, n0);
          }
        }
      }
    }
  } else if (warp >= 4) {
    regs_worker();
    mma_loop<TF32, BN, A_MN, B_MN>(sm, num_tiles, tiles_mn, splits, kb_per_split, nkb_total, false);
  } else {
    // ===================== epilogue: staging buffer -> registers -> global =====================
    regs_worker();
    const bool split = (partial != nullptr);
    __shared__ float bias_s[2 * BN];
    uint32_t lt = 0;
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x, lt++) {
      const int z = (splits == 1) ? 0 : t / tiles_mn, r = t - z * tiles_mn;   // fast path: no integer division without split-K
      const int mt_ = (tiles_n == 1) ? r : r / tiles_n;
      const int m0 = mt_ * BLOCK_M, n0 = (r - mt_ * tiles_n) * BN;
      const uint32_t bsel = lt & 1;   // bias_s half of this tile
      const long long m = (long long)m0 + threadIdx.x;
      const bool row_ok = m < M;
      if (bias != nullptr && !split) {
        stage_cols<BN>(bias_s + bsel * BN, bias, n0, N);
        epi_bar_sync();
      }
      mbar_wait(sm.acc_full_bar, lt & 1);
#pragma unroll 1
      for (int pr = 0; pr < BN / 64; pr++) {
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const int c = pr * 2 + h;
          float f[32];
          read_chunk<BN>(sm, threadIdx.x, c, f);
          const int nbase = n0 + c * 32;
          if (!row_ok || nbase >= N) continue;
          const int ncols = N - nbase;
          if (split) {
            float* dst = partial + ((long long)z * M + m) * N + nbase;
            if (ncols >= 32 && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0)) {
#pragma unroll
              for (int j = 0; j < 32; j += 4) *reinterpret_cast<float4*>(dst + j) = make_float4(f[j], f[j + 1], f[j + 2], f[j + 3]);
            } else {
#pragma unroll
              for (int j = 0; j < 32; j++)
                if (j < ncols) dst[j] = f[j];
            }
            continue;
          }
          if (bias) add_staged32(f, bias_s + bsel * BN + c * 32);
          if (c_bf16) {
            if (addend) add_row32<bf16, true>(f, reinterpret_cast<const bf16*>(addend) + m * ldd + nbase, ncols);
            store_row32<bf16, true>(reinterpret_cast<bf16*>(Cv) + m * ldc + nbase, f, accumulate, ncols);
          } else {
            if (addend) add_row32<float, true>(f, reinterpret_cast<const float*>(addend) + m * ldd + nbase, ncols);
            store_row32<float, true>(reinterpret_cast<float*>(Cv) + m * ldc + nbase, f, accumulate, ncols);
          }
        }
      }
    }
  }
}

// second pass of split-K: C = sum_z partial[z] + bias + addend + (accumulate ? C : 0); transposed: the partials are [z][N][M]
// (conv kind 1 with swapped operand roles).  One thread sums one element in ascending z, whatever the grid.
template <typename TO>
__global__ void splitk_reduce_kernel(const float* __restrict__ partial, int splits, TO* __restrict__ C, long long ldc, int M, int N,
                                     int accumulate, const float* __restrict__ bias, const TO* __restrict__ addend, long long ldd,
                                     int transposed) {
  const long long total = (long long)M * N;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const long long m = idx / N;
    const int n = (int)(idx - m * N);
    const long long pidx = transposed ? (long long)n * M + m : idx;
    float acc = 0.f;
    for (int z = 0; z < splits; z++) acc += partial[(long long)z * total + pidx];
    if (bias) acc += bias[n];
    if (addend) acc += ld_f<TO>(&addend[m * ldd + n]);
    if (accumulate) acc += ld_f<TO>(&C[m * ldc + n]);
    st_f<TO>(&C[m * ldc + n], acc);
  }
}

// ------------------------------------------------------------------ host side
template <typename TIn, int BN, bool A_MN, bool B_MN>
int launch(const CUtensorMap& ta, const CUtensorMap& tb, void* C, int c_dtype, long long ldc, int M, int N, int K, int accumulate,
           const float* bias, const void* addend, long long ldd, float* partial, int splits, int kb_per_split, cudaStream_t st) {
  const long long num_tiles = (long long)cdiv(M, BLOCK_M) * cdiv(N, BN) * splits;
  return launch_persistent<gemm_tc_kernel<TIn, BN, A_MN, B_MN>, BN>(num_tiles, st, "gemm_tc", ta, tb, C, (int)(c_dtype == P2PVG_BF16), ldc,
                                                                    M, N, K, accumulate, bias, addend, ldd, partial, kb_per_split, splits);
}

}  // namespace

int p2pvg_gemm_tc_available() { return driver().encode != nullptr; }

int p2pvg_splitk_reduce(const float* partial, int splits, void* C, int c_dtype, long long ldc, int M, int N, int accumulate,
                        const float* bias, const void* addend, long long ldd, int transposed, cudaStream_t st) {
  const long long total = (long long)M * N;
  const int cap = driver().sms * 8;
  const int blocks = (int)((total + 255) / 256 > cap ? cap : (total + 255) / 256);
  if (c_dtype == P2PVG_BF16)
    splitk_reduce_kernel<bf16><<<blocks, 256, 0, st>>>(partial, splits, (bf16*)C, ldc, M, N, accumulate, bias, (const bf16*)addend, ldd,
                                                       transposed);
  else
    splitk_reduce_kernel<float><<<blocks, 256, 0, st>>>(partial, splits, (float*)C, ldc, M, N, accumulate, bias, (const float*)addend, ldd,
                                                        transposed);
  return p2pvg_check_launch("splitk_reduce");
}

static bool tc_operand_ok(const void* p, long long ld, int elem = 2) {
  return ((reinterpret_cast<uintptr_t>(p) & 15) == 0) && ((ld * elem) % 16 == 0);
}

// fp32 operands on the tensor cores at TF32 precision (K-major operands only).  Returns P2PVG_ERR_UNSUPPORTED when the
// operands are not TMA-compatible so that the caller can use the CUDA-core kernel instead.
int p2pvg_gemm_tf32(const void* A, long long lda, const void* B, long long ldb, void* C, int c_dtype, long long ldc, int M, int N,
                    int K, int accumulate, const float* bias, const void* addend, long long ldd, cudaStream_t st) {
  if (M <= 0 || N <= 0) return P2PVG_OK;
  if (!p2pvg_gemm_tc_available() || !tc_operand_ok(A, lda, 4) || !tc_operand_ok(B, ldb, 4) || K <= 0) return P2PVG_ERR_UNSUPPORTED;
  const int BN = (N > 64) ? 128 : 64;
  CUtensorMap ta, tb;
  int rc = map2d(&ta, A, K, M, lda, BLOCK_M, 4);
  if (rc) return rc;
  rc = map2d(&tb, B, K, N, ldb, BN, 4);
  if (rc) return rc;
  const int nkb = cdiv(K, 32);
  if (BN == 128) return launch<float, 128, false, false>(ta, tb, C, c_dtype, ldc, M, N, K, accumulate, bias, addend, ldd, nullptr, 1, nkb, st);
  return launch<float, 64, false, false>(ta, tb, C, c_dtype, ldc, M, N, K, accumulate, bias, addend, ldd, nullptr, 1, nkb, st);
}

int p2pvg_gemm_tc(const void* A, int a_mn, long long lda, const void* B, int b_mn, long long ldb, void* C, int c_dtype, long long ldc,
                  int M, int N, int K, int accumulate, const float* bias, const void* addend, long long ldd, void* workspace,
                  size_t ws_bytes, cudaStream_t st) {
  if (M <= 0 || N <= 0) return P2PVG_OK;
  if (!p2pvg_gemm_tc_available() || !tc_operand_ok(A, lda) || !tc_operand_ok(B, ldb) || K <= 0) {
    if (p2pvg_gemm_impl_forced() == 2) {
      p2pvg_set_error("gemm_tc: operands not TMA-compatible (A=%p lda=%lld B=%p ldb=%lld K=%d, driver=%d)", A, lda, B, ldb, K,
                      p2pvg_gemm_tc_available());
      return P2PVG_ERR_UNSUPPORTED;
    }
    return p2pvg_gemm_simt(A, P2PVG_BF16, a_mn, lda, B, b_mn, ldb, C, c_dtype, ldc, M, N, K, accumulate, bias, addend, ldd, workspace, ws_bytes, st);
  }
  const int BN = (N > 64) ? 128 : 64;
  CUtensorMap ta, tb;
  int rc;
  constexpr int BLOCK_K = 64;
  if (a_mn) rc = map2d(&ta, A, M, K, lda, BLOCK_K);
  else rc = map2d(&ta, A, K, M, lda, BLOCK_M);
  if (rc) return rc;
  if (b_mn) rc = map2d(&tb, B, N, K, ldb, BLOCK_K);
  else rc = map2d(&tb, B, K, N, ldb, BN);
  if (rc) return rc;

  // split-K when the output has too few tiles to fill the SMs and the reduction is long
  const int nkb = cdiv(K, BLOCK_K);
  const long long tiles = (long long)cdiv(M, BLOCK_M) * cdiv(N, BN);
  int splits = 1;
  if (tiles < 120 && nkb >= 16) {
    long long want = (2 * driver().sms + tiles - 1) / tiles;
    long long maxs = nkb / 8;
    splits = (int)(want < maxs ? want : maxs);
    if (splits < 1) splits = 1;
    size_t need = (size_t)splits * M * N * sizeof(float);
    while (splits > 1 && (workspace == nullptr || need > ws_bytes)) {
      splits /= 2;
      need = (size_t)splits * M * N * sizeof(float);
    }
  }
  int kb_per_split = cdiv(nkb, splits);
  splits = cdiv(nkb, kb_per_split);
  float* partial = splits > 1 ? reinterpret_cast<float*>(workspace) : nullptr;

#define GO(BN_, AM, BM)                                                                                                     \
  rc = launch<bf16, BN_, AM, BM>(ta, tb, C, c_dtype, ldc, M, N, K, accumulate, bias, addend, ldd, partial, splits, kb_per_split, st)
  if (BN == 128) {
    if (a_mn && b_mn) GO(128, true, true);
    else if (a_mn) GO(128, true, false);
    else if (b_mn) GO(128, false, true);
    else GO(128, false, false);
  } else {
    if (a_mn && b_mn) GO(64, true, true);
    else if (a_mn) GO(64, true, false);
    else if (b_mn) GO(64, false, true);
    else GO(64, false, false);
  }
#undef GO
  if (rc) return rc;
  if (splits > 1) return p2pvg_splitk_reduce(partial, splits, C, c_dtype, ldc, M, N, accumulate, bias, addend, ldd, 0, st);
  return P2PVG_OK;
}
