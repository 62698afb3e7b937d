// The persistent wgmma skeleton of the tensor-core GEMM (gemm_tc.cu) and the implicit-GEMM convolutions (conv_gemm.cu), sm_90a:
// the wgmma / TMA / mbarrier PTX wrappers, the tile configuration and shared-memory carve-up, the MMA warpgroup loop, the
// epilogue's staging-buffer reads and row stores, and the host side (driver entry point, SM count, tensor maps, launch).
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace tc {

// ------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* desc, uint64_t* bar, void* smem_dst, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(desc)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// ------------------------------------------------------------------ wgmma (sm_90a warpgroup MMA, accumulator in registers)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of accumulator registers across the asynchronous MMAs that own them
template <int N>
__device__ __forceinline__ void fence_regs(float (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; i++) asm volatile("" : "+f"(r[i])::"memory");
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_n64(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_n128(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d), "n"(TA), "n"(TB));
}
// D[64 x 256] (+)= A[64 x 16] . B[16 x 256]; 128 fp32 accumulators per thread
template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16_n256(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, %131, %132;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d), "n"(TA), "n"(TB));
}
__device__ __forceinline__ void wgmma_tf32_n64(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_tf32_n128(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(scale_d));
}
// one full 32-byte sector (32-byte aligned) as two 16-byte stores
__device__ __forceinline__ void st_global_256(void* p, uint32_t a, uint32_t b, uint32_t c, uint32_t d, uint32_t e, uint32_t f, uint32_t g,
                                              uint32_t h) {
  uint4* q = reinterpret_cast<uint4*>(p);
  q[0] = make_uint4(a, b, c, d);
  q[1] = make_uint4(e, f, g, h);
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
// register budget of a 384-thread CTA (3 warpgroups, 168 registers each at launch): the producer warpgroup gives most of its
// registers to the MMA and epilogue warpgroups (40 + 232 + 232 <= 3 x 168)
__device__ __forceinline__ void regs_producer() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;"); }
__device__ __forceinline__ void regs_worker() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;"); }
// named barrier among the four epilogue warps (barrier 0 is __syncthreads)
__device__ __forceinline__ void epi_bar_sync() { asm volatile("bar.sync 1, 128;" ::: "memory"); }

// wgmma shared-memory matrix descriptor of a SWIZZLE_128B tile (1024-byte aligned 8-row atoms).  K-major: rows of 128 B
// along k, sbo = 1024 between 8-row groups.  MN-major: rows of 128 B along m / n, lbo = stride between 64-element chunks
// along m / n, sbo = 1024 between groups of 8 k rows.
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;  // SWIZZLE_128B
  return d;
}

// One 128-byte K block of a BM x BN tile.  128 rows: for every MMA-K slice, one wgmma per 64-row half; the row halves of A
// are 8 KB apart in both majors (K-major: 64 rows of 128 B; MN-major: the second 64-wide m chunk).  256 x 64 (bf16,
// K-major A, MN-major B): the transposed product D^T[64 x 256] = B^T . A^T, one m64n256k16 per MMA-K slice with the B
// tile as the (M-major) A operand and the A tile as the (K-major) B operand.  Four m64n64k16 would read 16 KB of shared
// memory per k-slice where the one m64n256k16 reads 10 KB.  da / db describe k-slice 0 of the stage.  first: the first K
// block of the tile (overwrites the accumulator).
template <bool TF32, int BN, bool A_MN, bool B_MN, int BM>
__device__ __forceinline__ void wgmma_kblock(float (&acc)[BM / 64][BN / 2], uint64_t da, uint64_t db, bool first) {
  constexpr int UMMA_K = TF32 ? 8 : 16;
  constexpr int KSTEPS = 4;   // 128 B of K: 4 x k8 (tf32) or 4 x k16 (bf16)
  constexpr uint32_t A_STEP = (A_MN ? UMMA_K * 128 : 32) >> 4, B_STEP = (B_MN ? UMMA_K * 128 : 32) >> 4;
  if constexpr (BM == 256) {
    static_assert(!TF32 && BN == 64 && !A_MN && B_MN, "256-row tiles: bf16, K-major A, MN-major B, 64 columns");
#pragma unroll
    for (int k = 0; k < KSTEPS; k++)
      wgmma_bf16_n256<1, 0>(&acc[0][0], db + (uint64_t)(k * B_STEP), da + (uint64_t)(k * A_STEP), (first && k == 0) ? 0u : 1u);
  } else {
#pragma unroll
    for (int k = 0; k < KSTEPS; k++) {
      const uint32_t sc = (first && k == 0) ? 0u : 1u;
#pragma unroll
      for (int h = 0; h < BM / 64; h++) {
        const uint64_t a = da + (uint64_t)(h * (8192 >> 4) + k * A_STEP), b = db + (uint64_t)(k * B_STEP);
        if constexpr (TF32) {
          if constexpr (BN == 128) wgmma_tf32_n128(acc[h], a, b, sc);
          else wgmma_tf32_n64(acc[h], a, b, sc);
        } else {
          if constexpr (BN == 128) wgmma_bf16_n128<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc[h], a, b, sc);
          else wgmma_bf16_n64<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc[h], a, b, sc);
        }
      }
    }
  }
}

// Rows [128 hf, 128 hf + 128) of the MMA warpgroup's BM x BN accumulator (wgmma fragment layout) -> the row-major fp32
// staging buffer of 128 rows (row pitch ld floats) from which the epilogue warps read one tile row per thread.  t: thread
// index within the warpgroup.
template <int BN, int BM>
__device__ __forceinline__ void acc_to_smem(const float (&acc)[BM / 64][BN / 2], int hf, float* buf, int ld, int t) {
  const int w = t >> 5, l = t & 31;
  if constexpr (BM == 256) {
    // the transposed 64 x 256 accumulator (wgmma_kblock): fragment element 4 j + 2 i + e holds tile column
    // 16 w + (l >> 2) + 8 i of tile row 8 j + 2 (l & 3) + e.  Scalar stores; with ld = 68 the 32 lanes of one store hit
    // 32 different banks.
    const float* a = &acc[0][0];
    float* r0 = buf + (2 * (l & 3)) * ld + 16 * w + (l >> 2);
#pragma unroll
    for (int j = 0; j < 16; j++) {
      const int jj = 16 * hf + j;
#pragma unroll
      for (int e = 0; e < 2; e++) {
        r0[(8 * j + e) * ld] = a[4 * jj + e];
        r0[(8 * j + e) * ld + 8] = a[4 * jj + 2 + e];
      }
    }
  } else {
#pragma unroll
    for (int h = 0; h < 2; h++) {
      float* r0 = buf + (64 * h + 16 * w + (l >> 2)) * ld + 2 * (l & 3);
      const float* a = acc[2 * hf + h];
#pragma unroll
      for (int j = 0; j < BN / 8; j++) {
        *reinterpret_cast<float2*>(r0 + 8 * j) = make_float2(a[4 * j], a[4 * j + 1]);
        *reinterpret_cast<float2*>(r0 + 8 * ld + 8 * j) = make_float2(a[4 * j + 2], a[4 * j + 3]);
      }
    }
  }
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_load_4d(const CUtensorMap* desc, uint64_t* bar, void* smem_dst, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(desc)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// Thread-per-row epilogues hold one tile row per lane: column sums over the 32 rows of a warp by a transpose-reduce
// butterfly (16 + 8 + 4 + 2 + 1 = 31 shuffles for 32 columns instead of 5 per column).  Lane L returns the sum over the
// warp's lanes of v[L]; v is destroyed.  One template instance per stage: with a run-time stage loop the compiler did not
// unroll the inner loop fully, `v[j + off]` became a dynamic index and the arrays of the statistics epilogues lived in local
// memory (256-byte stack frame, 384 local loads / stores per 32-column chunk of a tile row).
template <int OFF>
__device__ __forceinline__ void colsum_stage(float (&v)[32], int lane) {
  const bool upper = (lane & OFF) != 0;
#pragma unroll
  for (int j = 0; j < OFF; j++) {
    const float send = upper ? v[j] : v[j + OFF];
    const float keep = upper ? v[j + OFF] : v[j];
    v[j] = keep + __shfl_xor_sync(0xffffffffu, send, OFF);
  }
  if constexpr (OFF > 1) colsum_stage<OFF / 2>(v, lane);
}
__device__ __forceinline__ float warp_colsum32(float (&v)[32], int lane) {
  colsum_stage<16>(v, lane);
  return v[0];
}
__device__ __forceinline__ float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// ------------------------------------------------------------------ the persistent skeleton
// 384 threads: warps 0..3 = epilogue (one tile row per thread), warps 4..7 = the MMA warpgroup, warp 8 = TMA producer (warps
// 9..11 only complete its warpgroup).  grid = min(#tiles, #SMs); every CTA walks tiles t = blockIdx.x, +gridDim.x, ...  The
// MMA warpgroup accumulates tile i+1 in registers while the epilogue drains tile i from the staging buffer.  Each kernel keeps
// its own TMA producer loop and tile decode, and what its epilogue does between reading a chunk and storing it.
constexpr int BLOCK_M = 128;
constexpr int ROW_BYTES = 128;  // one SWIZZLE_128B row: 64 bf16 or 32 fp32 (tf32) along the contiguous dimension
constexpr int A_STAGE_BYTES = BLOCK_M * ROW_BYTES;
constexpr int NUM_THREADS = 384;

// BM x BN tiles, BM = 128 (BN = 64 / 128) or 256 (BN = 64): one warpgroup holds the whole fp32 accumulator in registers
// (BM * BN / 128 per thread, at most 128).  The staging buffer always holds 128 rows: a 256-row tile is handed to the
// epilogue in two halves, which leaves room for 4 stages of 40 KB (a 256-row buffer would leave 3).
template <int BN, int BM = BLOCK_M> struct Cfg {
  static_assert(BM == 128 || (BM == 256 && BN == 64), "tile shapes: 128 x 64, 128 x 128, 256 x 64");
  static constexpr int A_STAGE_BYTES = BM * ROW_BYTES;
  static constexpr int B_STAGE_BYTES = BN * ROW_BYTES;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int STAGES = (BM == 256 || BN == 128) ? 4 : 7;
  static constexpr int ACC_LD = BN + 4;   // staging row pitch in floats: the row-per-thread float4 reads are conflict-free
  static constexpr int ACC_BYTES = BLOCK_M * ACC_LD * 4;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + ACC_BYTES + 1024 /*align slack*/ + 512 /*barriers*/;
};

// resident-weight mode (conv kind 0, BN = 64): weights at [0, 9 * 8 KB), A ring of 6 x 16 KB behind them
constexpr int BRES_B_BYTES = 9 * 64 * 128, BRES_STAGES = 6;
static_assert(BRES_B_BYTES + BRES_STAGES * A_STAGE_BYTES <= Cfg<64>::STAGES * Cfg<64>::STAGE_BYTES, "resident weights + A ring");

// the dynamic shared memory: operand stages, [BLOCK_M][ACC_LD] staging buffer, barriers
struct Smem {
  uint8_t* ring;
  float* accs;
  uint64_t *full_bar, *empty_bar, *acc_full_bar, *acc_empty_bar;
  uint64_t* bres_bar;   // the resident weights have landed (conv only)
};

template <int BN, int BM = BLOCK_M>
__device__ __forceinline__ Smem smem_setup(uint8_t* smem_raw) {
  using C_ = Cfg<BN, BM>;
  Smem s;
  s.ring = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  s.accs = reinterpret_cast<float*>(s.ring + C_::STAGES * C_::STAGE_BYTES);
  s.full_bar = reinterpret_cast<uint64_t*>(s.ring + C_::STAGES * C_::STAGE_BYTES + C_::ACC_BYTES);
  s.empty_bar = s.full_bar + C_::STAGES;
  s.acc_full_bar = s.empty_bar + C_::STAGES;
  s.acc_empty_bar = s.acc_full_bar + 1;
  s.bres_bar = s.acc_empty_bar + 1;
  if (threadIdx.x == 0) {
    for (int i = 0; i < C_::STAGES; i++) {
      mbar_init(&s.full_bar[i], 1);
      mbar_init(&s.empty_bar[i], 128);   // every thread of the MMA warpgroup
    }
    mbar_init(s.acc_full_bar, 128);
    mbar_init(s.acc_empty_bar, 4);       // one arrival per epilogue warp
    mbar_init(s.bres_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  return s;
}

// The MMA warpgroup: for each tile of this CTA, the K blocks of its split z, then the accumulator into the staging buffer,
// 128 rows at a time (a 256-row tile waits for the epilogue to drain its first half before it stages the second).
// bres: B is the resident weight tap kb and A streams through the BRES_STAGES ring (gemm_tc passes false).
template <bool TF32, int BN, bool A_MN, bool B_MN, int BM = BLOCK_M>
__device__ __forceinline__ void mma_loop(const Smem& sm, int num_tiles, int tiles_mn, int splits, int kb_per_split, int nkb_total,
                                         bool bres) {
  using C_ = Cfg<BN, BM>;
  static_assert(BM == 128 || !A_MN, "256-row tiles take a K-major A");
  const int wt = threadIdx.x - 128;
  const uint32_t smem0 = smem_u32(sm.ring);
  // MN-major: the 64-element chunks along m / n are 8 KB apart (MN-major operands are bf16)
  const uint64_t da0 = A_MN ? make_desc(smem0, 64 * 128, 1024) : make_desc(smem0, 0, 1024);
  const uint64_t db0 = B_MN ? make_desc(smem0 + C_::A_STAGE_BYTES, 64 * 128, 1024) : make_desc(smem0 + C_::A_STAGE_BYTES, 0, 1024);
  uint32_t it = 0, lh = 0;   // lh: staging-buffer hand-overs so far
  if (bres) mbar_wait(sm.bres_bar, 0);   // the resident weights have landed
  const uint64_t da0r = make_desc(smem0 + BRES_B_BYTES, 0, 1024), db0r = make_desc(smem0, 0, 1024);
  float acc[BM / 64][BN / 2];
  for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
    const int z = (splits == 1) ? 0 : t / tiles_mn;   // phases (conv kind 2) never split K
    const int kb0 = z * kb_per_split, kb1 = min(kb0 + kb_per_split, nkb_total);
    int prev = -1;   // stage of the previous K block: released once its MMAs have completed
    for (int kb = kb0; kb < kb1; kb++, it++) {
      // (both divisors are compile-time constants: no runtime division in the per-K-block path)
      const int s = bres ? (int)(it % BRES_STAGES) : (int)(it % C_::STAGES);
      const uint32_t par = (bres ? (it / BRES_STAGES) : (it / C_::STAGES)) & 1;
      mbar_wait(&sm.full_bar[s], par);
      // descriptors of stage 0 / k 0 are built once; the start-address field (bits 0-13, address >> 4) is advanced by
      // plain additions
      const uint64_t stage_off = (uint64_t)((uint32_t)s * (uint32_t)(C_::STAGE_BYTES >> 4));
      const uint64_t a_off = bres ? (uint64_t)((uint32_t)s * (uint32_t)(A_STAGE_BYTES >> 4)) : stage_off;
      const uint64_t b_off = bres ? (uint64_t)((uint32_t)kb * (uint32_t)((64 * 128) >> 4)) : stage_off;   // resident: tap kb
#pragma unroll
      for (int h = 0; h < BM / 64; h++) fence_regs(acc[h]);
      wgmma_fence();
      wgmma_kblock<TF32, BN, A_MN, B_MN, BM>(acc, (bres ? da0r : da0) + a_off, (bres ? db0r : db0) + b_off, kb == kb0);
      wgmma_commit();
      wgmma_wait<1>();
#pragma unroll
      for (int h = 0; h < BM / 64; h++) fence_regs(acc[h]);
      if (prev >= 0) mbar_arrive(&sm.empty_bar[prev]);
      prev = s;
    }
    wgmma_wait<0>();
#pragma unroll
    for (int h = 0; h < BM / 64; h++) fence_regs(acc[h]);
    if (prev >= 0) mbar_arrive(&sm.empty_bar[prev]);
#pragma unroll
    for (int hf = 0; hf < BM / 128; hf++, lh++) {
      mbar_wait(sm.acc_empty_bar, (lh & 1) ^ 1);   // the epilogue has drained the previous hand-over
      acc_to_smem<BN, BM>(acc, hf, sm.accs, C_::ACC_LD, wt);
      mbar_arrive(sm.acc_full_bar);
    }
  }
}

// Epilogue (threads 0..127): dst[i] = src[n0 + i] for i < BN (0 past N), staged while the MMAs are still running.  The
// caller double-buffers dst by tile parity and synchronises the epilogue warps before reading it.
template <int BN>
__device__ __forceinline__ void stage_cols(float* dst, const float* src, int n0, int N) {
  for (int i = threadIdx.x; i < BN; i += 128) dst[i] = (n0 + i < N) ? src[n0 + i] : 0.f;
}

// Epilogue: the staged accumulator columns [32 c, 32 c + 32) of tile row `row`.  After the tile's last chunk is read the
// staging buffer goes back to the MMA warpgroup *before* the caller's global stores.
template <int BN>
__device__ __forceinline__ void read_chunk(const Smem& sm, int row, int c, float (&f)[32]) {
  const float* src = sm.accs + row * Cfg<BN>::ACC_LD + c * 32;
#pragma unroll
  for (int j = 0; j < 32; j += 4) {
    const float4 x = *reinterpret_cast<const float4*>(src + j);
    f[j] = x.x; f[j + 1] = x.y; f[j + 2] = x.z; f[j + 3] = x.w;
  }
  if (c == BN / 32 - 1) {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(sm.acc_empty_bar);
  }
}

// f[0..31] += 32 columns staged by stage_cols
__device__ __forceinline__ void add_staged32(float (&f)[32], const float* s) {
#pragma unroll
  for (int j = 0; j < 32; j += 4) {
    const float4 b4 = *reinterpret_cast<const float4*>(s + j);
    f[j] += b4.x; f[j + 1] += b4.y; f[j + 2] += b4.z; f[j + 3] += b4.w;
  }
}

// f[j] += row[j] for the j < ncols (TAIL) or all 32 (!TAIL) columns
template <typename T, bool TAIL>
__device__ __forceinline__ void add_row32(float (&f)[32], const T* row, int ncols) {
#pragma unroll
  for (int j = 0; j < 32; j++)
    if (!TAIL || j < ncols) f[j] += ld_f<T>(row + j);
}

// One 32-column segment of an output row: (accumulate ? crow : 0) + f, stored as 256-bit stores when crow is 32-byte aligned,
// 128-bit stores otherwise.  TAIL (gemm_tc): fewer than 32 valid columns (ncols) or a row that is not 16-byte aligned is
// stored element by element; without TAIL all 32 columns are valid and crow is 16-byte aligned.
template <typename T, bool TAIL>
__device__ __forceinline__ void store_row32(T* crow, float (&f)[32], int accumulate, int ncols) {
  if (accumulate) add_row32<T, TAIL>(f, crow, ncols);
  const bool vec = !TAIL || (ncols >= 32 && (reinterpret_cast<uintptr_t>(crow) & 15) == 0);
  if (vec && (reinterpret_cast<uintptr_t>(crow) & 31) == 0) {
    if constexpr (sizeof(T) == 2) {
#pragma unroll
      for (int j = 0; j < 32; j += 16)
        st_global_256(crow + j, pack_bf16x2(f[j], f[j + 1]), pack_bf16x2(f[j + 2], f[j + 3]), pack_bf16x2(f[j + 4], f[j + 5]),
                      pack_bf16x2(f[j + 6], f[j + 7]), pack_bf16x2(f[j + 8], f[j + 9]), pack_bf16x2(f[j + 10], f[j + 11]),
                      pack_bf16x2(f[j + 12], f[j + 13]), pack_bf16x2(f[j + 14], f[j + 15]));
    } else {
#pragma unroll
      for (int j = 0; j < 32; j += 8)
        st_global_256(crow + j, __float_as_uint(f[j]), __float_as_uint(f[j + 1]), __float_as_uint(f[j + 2]), __float_as_uint(f[j + 3]),
                      __float_as_uint(f[j + 4]), __float_as_uint(f[j + 5]), __float_as_uint(f[j + 6]), __float_as_uint(f[j + 7]));
    }
  } else if (vec) {
    if constexpr (sizeof(T) == 2) {
#pragma unroll
      for (int j = 0; j < 32; j += 8)
        *reinterpret_cast<uint4*>(crow + j) =
            make_uint4(pack_bf16x2(f[j], f[j + 1]), pack_bf16x2(f[j + 2], f[j + 3]), pack_bf16x2(f[j + 4], f[j + 5]), pack_bf16x2(f[j + 6], f[j + 7]));
    } else {
#pragma unroll
      for (int j = 0; j < 32; j += 4) *reinterpret_cast<float4*>(crow + j) = make_float4(f[j], f[j + 1], f[j + 2], f[j + 3]);
    }
  } else {
#pragma unroll
    for (int j = 0; j < 32; j++)
      if (j < ncols) st_f<T>(crow + j, f[j]);
  }
}

// ------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
struct Driver {
  EncodeTiledFn encode = nullptr;   // cuTensorMapEncodeTiled; nullptr when the driver does not provide it
  int sms = 132;                    // SMs of the device that is current at the first call
};

// resolved once, on first use
inline const Driver& driver() {
  static const Driver d = [] {
    Driver r;
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && sms > 0)
      r.sms = sms;
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      r.encode = reinterpret_cast<EncodeTiledFn>(fn);
    (void)cudaGetLastError();
    return r;
  }();
  return d;
}

// 2-D tensor map of bf16 (elem 2) or fp32 (elem 4) elements: dim0 (contiguous) x dim1, row pitch ld elements, box
// (128 B x box1), 128B swizzle, zero OOB fill
inline int map2d(CUtensorMap* map, const void* base, long long dim0, long long dim1, long long ld, int box1, int elem = 2) {
  cuuint64_t dims[2] = {(cuuint64_t)dim0, (cuuint64_t)dim1};
  cuuint64_t strides[1] = {(cuuint64_t)ld * elem};
  cuuint32_t box[2] = {(cuuint32_t)(ROW_BYTES / elem), (cuuint32_t)box1};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = driver().encode(map, elem == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base),
                               dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    p2pvg_set_error("cuTensorMapEncodeTiled failed (%d): base=%p dims=(%lld,%lld) ld=%lld box1=%d", (int)r, base, dim0, dim1, ld, box1);
    return P2PVG_ERR_CUDA;
  }
  return P2PVG_OK;
}

// Launches KERN (a skeleton kernel with BM x BN tiles) on the persistent grid min(tiles, SMs).  The dynamic shared memory
// limit is raised on the first launch of each kernel instance.
template <auto KERN, int BN, int BM = BLOCK_M, typename... Args>
int launch_persistent(long long tiles, cudaStream_t st, const char* what, Args... args) {
  constexpr int SMEM_BYTES = Cfg<BN, BM>::SMEM_BYTES;
  static bool smem_attr_set = false;
  if (!smem_attr_set) {
    const cudaError_t e = cudaFuncSetAttribute(KERN, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (e != cudaSuccess) {
      p2pvg_set_error("%s: cudaFuncSetAttribute: %s", what, cudaGetErrorString(e));
      return P2PVG_ERR_CUDA;
    }
    smem_attr_set = true;
  }
  const int sms = driver().sms;
  KERN<<<(int)(tiles < sms ? tiles : sms), NUM_THREADS, SMEM_BYTES, st>>>(args...);
  return p2pvg_check_launch(what);
}

}  // namespace tc
