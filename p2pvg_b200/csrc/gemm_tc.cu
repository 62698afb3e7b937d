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
// Warp roles (384 threads): warps 0..3 = epilogue (one tile row per thread), warps 4..7 = the MMA warpgroup,
// warp 8 = TMA producer (warps 9..11 only complete its warpgroup).
#include <cuda.h>

#include <mutex>

#include "tc_common.cuh"

namespace {

constexpr int BLOCK_M = 128;
constexpr int ROW_BYTES = 128;  // one SWIZZLE_128B row: 64 bf16 or 32 fp32 (tf32) along the contiguous dimension
constexpr int A_STAGE_BYTES = BLOCK_M * ROW_BYTES;
constexpr int NUM_THREADS = 384;

template <int BN> struct Cfg {
  static constexpr int B_STAGE_BYTES = BN * ROW_BYTES;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int STAGES = (BN == 128) ? 4 : 7;
  static constexpr int ACC_LD = BN + 4;   // staging row pitch in floats: the row-per-thread float4 reads are conflict-free
  static constexpr int ACC_BYTES = BLOCK_M * ACC_LD * 4;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + ACC_BYTES + 1024 /*align slack*/ + 512 /*barriers*/;
};

// PTX wrappers (mbarrier / TMA / wgmma): tc_common.cuh, shared with conv_gemm.cu
using namespace tc;

// ------------------------------------------------------------------ the kernel

// Persistent: grid = min(#tiles, #SMs); every CTA walks tiles t = blockIdx.x, +gridDim.x, ...  A tile is
// (split z, m-tile, n-tile) with the n-tile fastest, so CTAs running at the same time share the A rows in L2.
// The MMA warpgroup accumulates tile i+1 in registers while the epilogue drains tile i from the staging buffer.
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
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* accs = reinterpret_cast<float*>(smem + C_::STAGES * C_::STAGE_BYTES);   // [BLOCK_M][ACC_LD] staging buffer
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + C_::STAGES * C_::STAGE_BYTES + C_::ACC_BYTES);
  uint64_t* empty_bar = full_bar + C_::STAGES;
  uint64_t* acc_full_bar = empty_bar + C_::STAGES;
  uint64_t* acc_empty_bar = acc_full_bar + 1;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_m = (M + BLOCK_M - 1) / BLOCK_M, tiles_n = (N + BN - 1) / BN;
  const int tiles_mn = tiles_m * tiles_n;
  const int num_tiles = tiles_mn * splits;
  const int nkb_total = (K + BLOCK_K - 1) / BLOCK_K;

  if (threadIdx.x == 0) {
    for (int s = 0; s < C_::STAGES; s++) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 128);   // every thread of the MMA warpgroup
    }
    mbar_init(acc_full_bar, 128);
    mbar_init(acc_empty_bar, 4);  // one arrival per epilogue warp
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

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
          mbar_wait(&empty_bar[s], ph ^ 1);
          uint8_t* sa = smem + s * C_::STAGE_BYTES;
          uint8_t* sb = sa + A_STAGE_BYTES;
          mbar_expect_tx(&full_bar[s], C_::STAGE_BYTES);
          const int k0 = kb * BLOCK_K;
          if (A_MN) {
            tma_load_2d(&tmA, &full_bar[s], sa, m0, k0);
            tma_load_2d(&tmA, &full_bar[s], sa + BLOCK_K * 128, m0 + 64, k0);
          } else {
            tma_load_2d(&tmA, &full_bar[s], sa, k0, m0);
          }
          if (B_MN) {
#pragma unroll
            for (int j = 0; j < BN / 64; j++) tma_load_2d(&tmB, &full_bar[s], sb + j * BLOCK_K * 128, n0 + 64 * j, k0);
          } else {
            tma_load_2d(&tmB, &full_bar[s], sb, k0, n0);
          }
        }
      }
    }
  } else if (warp >= 4) {
    // ===================== MMA warpgroup =====================
    regs_worker();
    const int wt = threadIdx.x - 128;
    const uint32_t smem0 = smem_u32(smem);
    const uint64_t da0 = A_MN ? make_desc(smem0, BLOCK_K * 128, 1024) : make_desc(smem0, 0, 1024);
    const uint64_t db0 = B_MN ? make_desc(smem0 + A_STAGE_BYTES, BLOCK_K * 128, 1024) : make_desc(smem0 + A_STAGE_BYTES, 0, 1024);
    float acc[2][BN / 2];
    uint32_t it = 0, lt = 0;
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x, lt++) {
      const int z = (splits == 1) ? 0 : t / tiles_mn;
      const int kb0 = z * kb_per_split, kb1 = min(kb0 + kb_per_split, nkb_total);
      int prev = -1;   // stage of the previous K block: released once its MMAs have completed
      for (int kb = kb0; kb < kb1; kb++, it++) {
        const int s = it % C_::STAGES;
        const uint32_t ph = (it / C_::STAGES) & 1;
        mbar_wait(&full_bar[s], ph);
        const uint64_t off = (uint64_t)((uint32_t)s * (uint32_t)(C_::STAGE_BYTES >> 4));
        fence_regs(acc[0]);
        fence_regs(acc[1]);
        wgmma_fence();
        wgmma_kblock<TF32, BN, A_MN, B_MN>(acc, da0 + off, db0 + off, kb == kb0);
        wgmma_commit();
        wgmma_wait<1>();
        fence_regs(acc[0]);
        fence_regs(acc[1]);
        if (prev >= 0) mbar_arrive(&empty_bar[prev]);
        prev = s;
      }
      wgmma_wait<0>();
      fence_regs(acc[0]);
      fence_regs(acc[1]);
      if (prev >= 0) mbar_arrive(&empty_bar[prev]);
      mbar_wait(acc_empty_bar, (lt & 1) ^ 1);   // the epilogue has drained the previous tile
      acc_to_smem<BN>(acc, accs, C_::ACC_LD, wt);
      mbar_arrive(acc_full_bar);
    }
  } else {
    // ===================== epilogue: staging buffer -> registers -> global =====================
    regs_worker();
    const int q = warp;  // rows [32 q, 32 q + 32) of the tile
    const bool split = (partial != nullptr);
    __shared__ float bias_s[2 * BN];
    uint32_t lt = 0;
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x, lt++) {
      const int z = (splits == 1) ? 0 : t / tiles_mn, r = t - z * tiles_mn;   // fast path: no integer division without split-K
      const int mt_ = (tiles_n == 1) ? r : r / tiles_n;
        const int m0 = mt_ * BLOCK_M, n0 = (r - mt_ * tiles_n) * BN;
      const uint32_t bsel = lt & 1;   // bias_s half of this tile
      const long long m = (long long)m0 + q * 32 + lane;
      const bool row_ok = m < M;
      // stage the bias slice of this tile in shared memory while the MMAs are still running
      if (bias != nullptr && !split) {
        for (int i = q * 32 + lane; i < BN; i += 128) bias_s[bsel * BN + i] = (n0 + i < N) ? bias[n0 + i] : 0.f;
        epi_bar_sync();
      }
      mbar_wait(acc_full_bar, lt & 1);
#pragma unroll 1
      for (int pr = 0; pr < BN / 64; pr++) {
#pragma unroll
        for (int h = 0; h < 2; h++) {
          // 32 columns at a time; after the last chunk is read the staging buffer goes back to the MMA warpgroup *before*
          // the global stores
          const int c = pr * 2 + h;
          uint32_t v[32];
          acc_row32(accs + (q * 32 + lane) * C_::ACC_LD + c * 32, v);
          if (c == BN / 32 - 1) {
            __syncwarp();
            if (lane == 0) mbar_arrive(acc_empty_bar);
          }
          const int nbase = n0 + c * 32;
          if (!row_ok || nbase >= N) continue;
          if (split) {
            float* dst = partial + ((long long)z * M + m) * N + nbase;
            if (nbase + 32 <= N && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0)) {
#pragma unroll
              for (int j = 0; j < 32; j += 4)
                *reinterpret_cast<float4*>(dst + j) = make_float4(__uint_as_float(v[j]), __uint_as_float(v[j + 1]), __uint_as_float(v[j + 2]), __uint_as_float(v[j + 3]));
            } else {
#pragma unroll
              for (int j = 0; j < 32; j++)
                if (nbase + j < N) dst[j] = __uint_as_float(v[j]);
            }
            continue;
          }
          float f[32];
#pragma unroll
          for (int j = 0; j < 32; j++) f[j] = __uint_as_float(v[j]);
          if (bias) {
            const float* bs = bias_s + bsel * BN + c * 32;
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
              const float4 b4 = *reinterpret_cast<const float4*>(bs + j);
              f[j] += b4.x; f[j + 1] += b4.y; f[j + 2] += b4.z; f[j + 3] += b4.w;
            }
          }
          if (c_bf16) {
            bf16* crow = reinterpret_cast<bf16*>(Cv) + m * ldc + nbase;
            if (addend) {
              const bf16* arow = reinterpret_cast<const bf16*>(addend) + m * ldd + nbase;
#pragma unroll
              for (int j = 0; j < 32; j++)
                if (nbase + j < N) f[j] += __bfloat162float(arow[j]);
            }
            if (accumulate) {
#pragma unroll
              for (int j = 0; j < 32; j++)
                if (nbase + j < N) f[j] += __bfloat162float(crow[j]);
            }
            const bool vec = (nbase + 32 <= N) && ((reinterpret_cast<uintptr_t>(crow) & 15) == 0);
            if (vec && (reinterpret_cast<uintptr_t>(crow) & 31) == 0) {
#pragma unroll
              for (int j = 0; j < 32; j += 16)
                st_global_256(crow + j, pack_bf16x2(f[j], f[j + 1]), pack_bf16x2(f[j + 2], f[j + 3]), pack_bf16x2(f[j + 4], f[j + 5]),
                              pack_bf16x2(f[j + 6], f[j + 7]), pack_bf16x2(f[j + 8], f[j + 9]), pack_bf16x2(f[j + 10], f[j + 11]),
                              pack_bf16x2(f[j + 12], f[j + 13]), pack_bf16x2(f[j + 14], f[j + 15]));
            } else if (vec) {
#pragma unroll
              for (int j = 0; j < 32; j += 8) {
                uint4 pk;
                pk.x = pack_bf16x2(f[j], f[j + 1]);
                pk.y = pack_bf16x2(f[j + 2], f[j + 3]);
                pk.z = pack_bf16x2(f[j + 4], f[j + 5]);
                pk.w = pack_bf16x2(f[j + 6], f[j + 7]);
                *reinterpret_cast<uint4*>(crow + j) = pk;
              }
            } else {
#pragma unroll
              for (int j = 0; j < 32; j++)
                if (nbase + j < N) crow[j] = __float2bfloat16_rn(f[j]);
            }
          } else {
            float* crow = reinterpret_cast<float*>(Cv) + m * ldc + nbase;
            if (addend) {
              const float* arow = reinterpret_cast<const float*>(addend) + m * ldd + nbase;
#pragma unroll
              for (int j = 0; j < 32; j++)
                if (nbase + j < N) f[j] += arow[j];
            }
            if (accumulate) {
#pragma unroll
              for (int j = 0; j < 32; j++)
                if (nbase + j < N) f[j] += crow[j];
            }
            const bool vec = (nbase + 32 <= N) && ((reinterpret_cast<uintptr_t>(crow) & 15) == 0);
            if (vec && (reinterpret_cast<uintptr_t>(crow) & 31) == 0) {
#pragma unroll
              for (int j = 0; j < 32; j += 8)
                st_global_256(crow + j, __float_as_uint(f[j]), __float_as_uint(f[j + 1]), __float_as_uint(f[j + 2]), __float_as_uint(f[j + 3]),
                              __float_as_uint(f[j + 4]), __float_as_uint(f[j + 5]), __float_as_uint(f[j + 6]), __float_as_uint(f[j + 7]));
            } else if (vec) {
#pragma unroll
              for (int j = 0; j < 32; j += 4) *reinterpret_cast<float4*>(crow + j) = make_float4(f[j], f[j + 1], f[j + 2], f[j + 3]);
            } else {
#pragma unroll
              for (int j = 0; j < 32; j++)
                if (nbase + j < N) crow[j] = f[j];
            }
          }
        }
      }
    }
  }
}

// second pass of split-K: C = sum_z partial[z] + bias + addend + (accumulate ? C : 0)
template <typename TO>
__global__ void splitk_reduce_kernel(const float* __restrict__ partial, int splits, TO* __restrict__ C, long long ldc, int M, int N,
                                     int accumulate, const float* __restrict__ bias, const TO* __restrict__ addend, long long ldd) {
  const long long total = (long long)M * N;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const long long m = idx / N;
    const int n = (int)(idx - m * N);
    float acc = 0.f;
    for (int z = 0; z < splits; z++) acc += partial[(long long)z * total + idx];
    if (bias) acc += bias[n];
    if (addend) acc += ld_f<TO>(&addend[m * ldd + n]);
    if (accumulate) acc += ld_f<TO>(&C[m * ldc + n]);
    st_f<TO>(&C[m * ldc + n], acc);
  }
}

// ------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;
std::once_flag g_once;
int g_attr_done[2][2][2][2] = {};

int g_num_sms = 132;

void resolve_driver() {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && sms > 0)
    g_num_sms = sms;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q);
  if (e == cudaSuccess && q == cudaDriverEntryPointSuccess) g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  (void)cudaGetLastError();
}

// 2-D bf16 tensor map: dim0 (contiguous) x dim1, row pitch ld elements, box (64 x box1), 128B swizzle, zero OOB fill
int make_map(CUtensorMap* map, const void* base, long long dim0, long long dim1, long long ld, int box1, int elem = 2) {
  cuuint64_t dims[2] = {(cuuint64_t)dim0, (cuuint64_t)dim1};
  cuuint64_t strides[1] = {(cuuint64_t)ld * elem};
  cuuint32_t box[2] = {(cuuint32_t)(ROW_BYTES / elem), (cuuint32_t)box1};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(map, elem == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    p2pvg_set_error("cuTensorMapEncodeTiled failed (%d): base=%p dims=(%lld,%lld) ld=%lld box1=%d", (int)r, base, dim0, dim1, ld, box1);
    return P2PVG_ERR_CUDA;
  }
  return P2PVG_OK;
}

template <typename TIn, int BN, bool A_MN, bool B_MN>
int launch(const CUtensorMap& ta, const CUtensorMap& tb, void* C, int c_dtype, long long ldc, int M, int N, int K, int accumulate,
           const float* bias, const void* addend, long long ldd, float* partial, int splits, int kb_per_split, cudaStream_t st) {
  auto kern = gemm_tc_kernel<TIn, BN, A_MN, B_MN>;
  int& done = g_attr_done[sizeof(TIn) == 4][BN == 128][A_MN][B_MN];
  if (!done) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<BN>::SMEM_BYTES);
    if (e != cudaSuccess) {
      p2pvg_set_error("gemm_tc: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
      return P2PVG_ERR_CUDA;
    }
    done = 1;
  }
  long long num_tiles = (long long)cdiv(M, BLOCK_M) * cdiv(N, BN) * splits;
  int grid = (int)(num_tiles < g_num_sms ? num_tiles : g_num_sms);
  kern<<<grid, NUM_THREADS, Cfg<BN>::SMEM_BYTES, st>>>(ta, tb, C, c_dtype == P2PVG_BF16, ldc, M, N, K, accumulate, bias, addend, ldd,
                                                      partial, kb_per_split, splits);
  return p2pvg_check_launch("gemm_tc");
}

}  // namespace

int p2pvg_gemm_tc_available() {
  std::call_once(g_once, resolve_driver);
  return g_encode != nullptr;
}

int p2pvg_gemm_simt(const void*, int, int, long long, const void*, int, long long, void*, int, long long, int, int, int, int,
                    const float*, const void*, long long, void*, size_t, cudaStream_t);

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
  int rc = make_map(&ta, A, K, M, lda, BLOCK_M, 4);
  if (rc) return rc;
  rc = make_map(&tb, B, K, N, ldb, BN, 4);
  if (rc) return rc;
  const int nkb = cdiv(K, 32);
  if (BN == 128) return launch<float, 128, false, false>(ta, tb, C, c_dtype, ldc, M, N, K, accumulate, bias, addend, ldd, nullptr, 1, nkb, st);
  return launch<float, 64, false, false>(ta, tb, C, c_dtype, ldc, M, N, K, accumulate, bias, addend, ldd, nullptr, 1, nkb, st);
}

int p2pvg_gemm_tc(const void* A, int a_mn, long long lda, const void* B, int b_mn, long long ldb, void* C, int c_dtype, long long ldc,
                  int M, int N, int K, int accumulate, const float* bias, const void* addend, long long ldd, void* workspace,
                  size_t ws_bytes, cudaStream_t st) {
  if (M <= 0 || N <= 0) return P2PVG_OK;
  extern int p2pvg_gemm_impl_forced();
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
  if (a_mn) rc = make_map(&ta, A, M, K, lda, BLOCK_K);
  else rc = make_map(&ta, A, K, M, lda, BLOCK_M);
  if (rc) return rc;
  if (b_mn) rc = make_map(&tb, B, N, K, ldb, BLOCK_K);
  else rc = make_map(&tb, B, K, N, ldb, BN);
  if (rc) return rc;

  // split-K when the output has too few tiles to fill the SMs and the reduction is long
  const int nkb = cdiv(K, BLOCK_K);
  const long long tiles = (long long)cdiv(M, BLOCK_M) * cdiv(N, BN);
  int splits = 1;
  if (tiles < 120 && nkb >= 16) {
    long long want = (2 * g_num_sms + tiles - 1) / tiles;
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
  if (splits > 1) {
    long long total = (long long)M * N;
    int blocks = (int)((total + 255) / 256 > g_num_sms * 8 ? g_num_sms * 8 : (total + 255) / 256);
    if (c_dtype == P2PVG_BF16)
      splitk_reduce_kernel<bf16><<<blocks, 256, 0, st>>>(partial, splits, (bf16*)C, ldc, M, N, accumulate, bias, (const bf16*)addend, ldd);
    else
      splitk_reduce_kernel<float><<<blocks, 256, 0, st>>>(partial, splits, (float*)C, ldc, M, N, accumulate, bias, (const float*)addend, ldd);
    return p2pvg_check_launch("splitk_reduce");
  }
  return P2PVG_OK;
}
