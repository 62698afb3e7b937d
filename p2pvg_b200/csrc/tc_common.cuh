// wgmma / TMA / mbarrier PTX wrappers shared by the tensor-core kernels (sm_90a).
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

// One 128-byte K block of a 128 x BN tile: for every MMA-K slice, one wgmma per 64-row half.  da / db describe k-slice 0 of
// the stage; the row halves of A are 8 KB apart in both majors (K-major: 64 rows of 128 B; MN-major: the second 64-wide m
// chunk).  first: the first K block of the tile (overwrites the accumulator).
template <bool TF32, int BN, bool A_MN, bool B_MN>
__device__ __forceinline__ void wgmma_kblock(float (&acc)[2][BN / 2], uint64_t da, uint64_t db, bool first) {
  constexpr int UMMA_K = TF32 ? 8 : 16;
  constexpr int KSTEPS = 4;   // 128 B of K: 4 x k8 (tf32) or 4 x k16 (bf16)
  constexpr uint32_t A_STEP = (A_MN ? UMMA_K * 128 : 32) >> 4, B_STEP = (B_MN ? UMMA_K * 128 : 32) >> 4;
#pragma unroll
  for (int k = 0; k < KSTEPS; k++) {
    const uint32_t sc = (first && k == 0) ? 0u : 1u;
#pragma unroll
    for (int h = 0; h < 2; h++) {
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

// The MMA warpgroup's 128 x BN accumulator (wgmma fragment layout) -> row-major fp32 staging buffer (row pitch ld floats)
// from which the epilogue warps read one tile row per thread.  t: thread index within the warpgroup.
template <int BN>
__device__ __forceinline__ void acc_to_smem(const float (&acc)[2][BN / 2], float* buf, int ld, int t) {
  const int w = t >> 5, l = t & 31;
#pragma unroll
  for (int h = 0; h < 2; h++) {
    float* r0 = buf + (64 * h + 16 * w + (l >> 2)) * ld + 2 * (l & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; j++) {
      *reinterpret_cast<float2*>(r0 + 8 * j) = make_float2(acc[h][4 * j], acc[h][4 * j + 1]);
      *reinterpret_cast<float2*>(r0 + 8 * ld + 8 * j) = make_float2(acc[h][4 * j + 2], acc[h][4 * j + 3]);
    }
  }
}
// 32 consecutive fp32 accumulator columns of one staged row
__device__ __forceinline__ void acc_row32(const float* src, uint32_t* v) {
#pragma unroll
  for (int j = 0; j < 32; j += 4) {
    const float4 x = *reinterpret_cast<const float4*>(src + j);
    v[j] = __float_as_uint(x.x); v[j + 1] = __float_as_uint(x.y); v[j + 2] = __float_as_uint(x.z); v[j + 3] = __float_as_uint(x.w);
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

}  // namespace tc
