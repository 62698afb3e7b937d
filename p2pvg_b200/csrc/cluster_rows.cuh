// Helpers of the row-slab cluster kernels (lstm_step.cu, pose_mlp.cu): a slab of up to NB batch rows sits in shared memory,
// every output unit is one warp streaming its weight row from L2 (lanes along K, coalesced), exact fp32 FFMA.
#pragma once
#include <cuda_runtime.h>

// acc[b] = sum_k w[k] * x[b * ldx + k] over the warp (lanes along k), result in every lane
template <int NB>
__device__ __forceinline__ void warp_dot(const float* __restrict__ w, const float* x, int ldx, int K, int nrows, int lane,
                                         float (&acc)[NB]) {
#pragma unroll
  for (int b = 0; b < NB; b++) acc[b] = 0.f;
  for (int k = lane; k < K; k += 32) {
    const float wk = __ldg(w + k);
#pragma unroll
    for (int b = 0; b < NB; b++)
      if (b < nrows) acc[b] = fmaf(wk, x[b * ldx + k], acc[b]);
  }
#pragma unroll
  for (int b = 0; b < NB; b++)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[b] += __shfl_xor_sync(0xffffffffu, acc[b], o);
}
