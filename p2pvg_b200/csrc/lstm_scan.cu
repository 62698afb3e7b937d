// Persistent LSTM-layer scans: ONE launch runs all timesteps of a layer's recurrence
//   forward :  gates_s = Pre_s + b_hh + h_{s-1} . W_hh^T ; (i,f,g,o) -> c_s, h_s            (nn.LSTMCell, models/lstm.py:41,89)
//   backward:  dh_s = dHtop_s + dG_{s+1} . W_hh ; cell pointwise backward -> dG_s, dc_{s-1}
// instead of two launches per step.  Work split: CTA = (block of 8 hidden units) x (block of 64 batch rows); the CTA keeps
// its slice of W_hh in shared memory for the whole sequence and its cell state / cell-state gradient in registers.  Steps
// are separated by a grid-wide barrier (monotonic counter in global memory; the kernel is launched cooperatively so all CTAs
// are co-resident).  State exchanged between CTAs (h_s, dG_s) goes through global memory / L2 with L1-bypassing loads.
// fp32 CUDA-core math: exact-fp32 recurrence in both precision modes.
#include <cooperative_groups.h>

#include "common.cuh"

namespace {

constexpr int UB = 8;    // hidden units per CTA  (-> 32 gate columns)
constexpr int RB = 64;   // batch rows per CTA
constexpr int NT = 256;  // threads
constexpr int PAD = 4;

__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ void grid_barrier(unsigned* counter, unsigned target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(counter, 1u);
    while (ld_acquire(counter) < target) { __nanosleep(32); }
  }
  __syncthreads();
}

// legacy warp-level tensor-core MMA (TF32 operands, fp32 accumulate): D[16x8] += A[16x8] . B[8x8]
__device__ __forceinline__ void mma_tf32(float* c, const uint32_t* a, const uint32_t* b) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
__device__ __forceinline__ uint32_t to_tf32(float x) {
  uint32_t r;
  asm volatile("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}

// ------------------------------------------------------------------------------------------------ forward
// TC = false: exact fp32 FFMA recurrence (parity mode).  TC = true: the h.W_hh^T product on the tensor cores (TF32).
template <bool TC>
__global__ void __launch_bounds__(NT, 1)
lstm_scan_fwd_kernel(const float* __restrict__ pre, const float* __restrict__ whh, const float* __restrict__ bhh,
                     float* __restrict__ gates, float* __restrict__ hs, float* __restrict__ cs, int S, int B, int R,
                     unsigned* __restrict__ counter) {
  extern __shared__ __align__(16) float sm[];
  const int LD = R + PAD;
  float* Ws = sm;                    // [32][LD]   rows: gate*8 + uu
  float* Hs = Ws + 32 * LD;          // [RB][LD]
  float* Gs = Hs + RB * LD;          // [RB][33]   gate pre-activations of this CTA
  const int nub = R / UB;
  const int ub = blockIdx.x % nub, rb = blockIdx.x / nub;
  const int u0 = ub * UB, r0 = rb * RB;
  const int tid = threadIdx.x;
  const unsigned nctas = gridDim.x;

  // resident W_hh slice: row (gate g, unit u0+uu) of W_hh[4R, R]
  for (int i = tid; i < 32 * (R / 4); i += NT) {
    const int row = i / (R / 4), k4 = i - row * (R / 4);
    const int g = row >> 3, uu = row & 7;
    const float4 v = *reinterpret_cast<const float4*>(whh + (long long)(g * R + u0 + uu) * R + k4 * 4);
    *reinterpret_cast<float4*>(Ws + row * LD + k4 * 4) = v;
  }
  // this thread's two (row, unit) cells for the pointwise part
  const int pr0 = tid >> 3, puu = tid & 7;     // rows pr0 and pr0+32
  float c_reg[2];
#pragma unroll
  for (int h = 0; h < 2; h++) {
    const int b = r0 + pr0 + 32 * h;
    c_reg[h] = (b < B) ? cs[(long long)b * R + u0 + puu] : 0.f;   // cs[0]
  }
  float bh[4];
#pragma unroll
  for (int g = 0; g < 4; g++) bh[g] = bhh[g * R + u0 + puu];
  // matmul thread tile: 4 rows x 2 cols
  const int tr = (tid >> 4) * 4, tc = (tid & 15) * 2;

  for (int s = 0; s < S; s++) {
    if (s > 0) grid_barrier(counter, nctas * (unsigned)s);   // h_s of every CTA is visible
    else __syncthreads();
    // stage h_{s-1} rows [r0, r0+RB) (L1 bypass: written by other SMs in the previous step)
    const float* hprev = hs + (long long)s * B * R;
    for (int i = tid; i < RB * (R / 4); i += NT) {
      const int row = i / (R / 4), k4 = i - row * (R / 4);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r0 + row < B) v = __ldcg(reinterpret_cast<const float4*>(hprev + (long long)(r0 + row) * R + k4 * 4));
      *reinterpret_cast<float4*>(Hs + row * LD + k4 * 4) = v;
    }
    __syncthreads();
    if (TC) {
      // 64x32 output = 4 (m16) x 4 (n8) MMA tiles; warp w: m-tile w>>1, n-tiles 2*(w&1)+{0,1}
      const int warp = tid >> 5, lane = tid & 31, gq = lane >> 2, tq = lane & 3;
      const int m0 = (warp >> 1) * 16, nb = (warp & 1) * 16;
      float c0[4] = {0.f, 0.f, 0.f, 0.f}, c1[4] = {0.f, 0.f, 0.f, 0.f};
      const float* ha = Hs + (m0 + gq) * LD + tq;
      const float* wb0 = Ws + (nb + gq) * LD + tq;
      const float* wb1 = wb0 + 8 * LD;
      for (int k = 0; k < R; k += 8) {
        uint32_t a[4], b0[2], b1[2];
        a[0] = to_tf32(ha[k]); a[1] = to_tf32(ha[8 * LD + k]); a[2] = to_tf32(ha[k + 4]); a[3] = to_tf32(ha[8 * LD + k + 4]);
        b0[0] = to_tf32(wb0[k]); b0[1] = to_tf32(wb0[k + 4]);
        b1[0] = to_tf32(wb1[k]); b1[1] = to_tf32(wb1[k + 4]);
        mma_tf32(c0, a, b0);
        mma_tf32(c1, a, b1);
      }
      Gs[(m0 + gq) * 33 + nb + 2 * tq] = c0[0];
      Gs[(m0 + gq) * 33 + nb + 2 * tq + 1] = c0[1];
      Gs[(m0 + gq + 8) * 33 + nb + 2 * tq] = c0[2];
      Gs[(m0 + gq + 8) * 33 + nb + 2 * tq + 1] = c0[3];
      Gs[(m0 + gq) * 33 + nb + 8 + 2 * tq] = c1[0];
      Gs[(m0 + gq) * 33 + nb + 8 + 2 * tq + 1] = c1[1];
      Gs[(m0 + gq + 8) * 33 + nb + 8 + 2 * tq] = c1[2];
      Gs[(m0 + gq + 8) * 33 + nb + 8 + 2 * tq + 1] = c1[3];
    } else {
    float acc[4][2];
#pragma unroll
    for (int i = 0; i < 4; i++) { acc[i][0] = 0.f; acc[i][1] = 0.f; }
    for (int k = 0; k < R; k += 4) {
      float4 a[4], w[2];
#pragma unroll
      for (int i = 0; i < 4; i++) a[i] = *reinterpret_cast<const float4*>(Hs + (tr + i) * LD + k);
#pragma unroll
      for (int j = 0; j < 2; j++) w[j] = *reinterpret_cast<const float4*>(Ws + (tc + j) * LD + k);
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 2; j++) {
          acc[i][j] = fmaf(a[i].x, w[j].x, acc[i][j]);
          acc[i][j] = fmaf(a[i].y, w[j].y, acc[i][j]);
          acc[i][j] = fmaf(a[i].z, w[j].z, acc[i][j]);
          acc[i][j] = fmaf(a[i].w, w[j].w, acc[i][j]);
        }
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
      Gs[(tr + i) * 33 + tc] = acc[i][0];
      Gs[(tr + i) * 33 + tc + 1] = acc[i][1];
    }
    }
    __syncthreads();
    // pointwise LSTM cell for (row, unit) = (pr0 + 32h, puu)
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int row = pr0 + 32 * h, b = r0 + row;
      if (b >= B) continue;
      const long long gbase = ((long long)s * B + b) * 4 * R + u0 + puu;
      float z[4];
#pragma unroll
      for (int g = 0; g < 4; g++) z[g] = Gs[row * 33 + g * 8 + puu] + pre[gbase + (long long)g * R] + bh[g];
      const float ig = sigmoidf_(z[0]), fg = sigmoidf_(z[1]), gg = tanhf(z[2]), og = sigmoidf_(z[3]);
      const float c = fg * c_reg[h] + ig * gg;
      c_reg[h] = c;
      gates[gbase] = ig;
      gates[gbase + R] = fg;
      gates[gbase + 2LL * R] = gg;
      gates[gbase + 3LL * R] = og;
      const long long o = ((long long)(s + 1) * B + b) * R + u0 + puu;
      cs[o] = c;
      hs[o] = og * tanhf(c);
    }
  }
}

// ------------------------------------------------------------------------------------------------ backward
template <bool TC>
__global__ void __launch_bounds__(NT, 1)
lstm_scan_bwd_kernel(const float* __restrict__ dhtop, const float* __restrict__ whh, const float* __restrict__ gates,
                     const float* __restrict__ cs, float* __restrict__ dG, int S, int B, int R, unsigned* __restrict__ counter) {
  extern __shared__ __align__(16) float sm[];
  const int K4 = 4 * R;
  const int KC = 256;                 // dG columns staged per chunk
  const int LDW = K4 + PAD, LDG = KC + PAD;
  float* Wt = sm;                     // [UB][LDW]   Wt[uu][q] = W_hh[q][u0+uu]
  float* Gc = Wt + UB * LDW;          // [RB][LDG]   chunk of dG_{s+1}
  float* Rs = Gc + RB * LDG;          // [2][RB][9]  TC: partial dh_rec of the two K halves
  const int nub = R / UB;
  const int ub = blockIdx.x % nub, rb = blockIdx.x / nub;
  const int u0 = ub * UB, r0 = rb * RB;
  const int tid = threadIdx.x;
  const unsigned nctas = gridDim.x;
  for (int i = tid; i < UB * K4; i += NT) {
    const int q = i / UB, uu = i - q * UB;
    Wt[uu * LDW + q] = whh[(long long)q * R + u0 + uu];
  }
  // thread -> 2 (row, unit) cells: rows pr0, pr0+32; unit puu
  const int pr0 = tid >> 3, puu = tid & 7;
  float dc_reg[2] = {0.f, 0.f};
  __syncthreads();

  for (int it = 0; it < S; it++) {
    const int s = S - 1 - it;
    float rec[2] = {0.f, 0.f};
    if (it > 0) {
      grid_barrier(counter, nctas * (unsigned)it);   // dG_{s+1} complete everywhere
      const float* gnext = dG + (long long)(s + 1) * B * K4;
      // TC: warp w -> m-tile (w&3), K half (w>>2); accumulates over all chunks in registers
      const int warp = tid >> 5, lane = tid & 31, gq = lane >> 2, tq = lane & 3;
      const int m0 = (warp & 3) * 16, kh = (warp >> 2) * 128;
      float cacc[4] = {0.f, 0.f, 0.f, 0.f};
      for (int kc = 0; kc < K4; kc += KC) {
        for (int i = tid; i < RB * (KC / 4); i += NT) {
          const int row = i / (KC / 4), k4 = i - row * (KC / 4);
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (r0 + row < B) v = __ldcg(reinterpret_cast<const float4*>(gnext + (long long)(r0 + row) * K4 + kc + k4 * 4));
          *reinterpret_cast<float4*>(Gc + row * LDG + k4 * 4) = v;
        }
        __syncthreads();
        if (TC) {
          const float* ga = Gc + (m0 + gq) * LDG + kh + tq;
          const float* wb = Wt + gq * LDW + kc + kh + tq;
#pragma unroll 4
          for (int k = 0; k < 128; k += 8) {
            uint32_t a[4], b[2];
            a[0] = to_tf32(ga[k]); a[1] = to_tf32(ga[8 * LDG + k]); a[2] = to_tf32(ga[k + 4]); a[3] = to_tf32(ga[8 * LDG + k + 4]);
            b[0] = to_tf32(wb[k]); b[1] = to_tf32(wb[k + 4]);
            mma_tf32(cacc, a, b);
          }
        } else {
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const float* grow = Gc + (pr0 + 32 * h) * LDG;
          const float* wrow = Wt + puu * LDW + kc;
          float a0 = 0.f, a1 = 0.f;
          for (int k = 0; k < KC; k += 8) {
            const float4 g0 = *reinterpret_cast<const float4*>(grow + k), g1 = *reinterpret_cast<const float4*>(grow + k + 4);
            const float4 w0 = *reinterpret_cast<const float4*>(wrow + k), w1 = *reinterpret_cast<const float4*>(wrow + k + 4);
            a0 = fmaf(g0.x, w0.x, a0); a0 = fmaf(g0.y, w0.y, a0); a0 = fmaf(g0.z, w0.z, a0); a0 = fmaf(g0.w, w0.w, a0);
            a1 = fmaf(g1.x, w1.x, a1); a1 = fmaf(g1.y, w1.y, a1); a1 = fmaf(g1.z, w1.z, a1); a1 = fmaf(g1.w, w1.w, a1);
          }
          rec[h] += a0 + a1;
        }
        }
        __syncthreads();
      }
      if (TC) {
        float* dst = Rs + (warp >> 2) * RB * 9;
        dst[(m0 + gq) * 9 + 2 * tq] = cacc[0];
        dst[(m0 + gq) * 9 + 2 * tq + 1] = cacc[1];
        dst[(m0 + gq + 8) * 9 + 2 * tq] = cacc[2];
        dst[(m0 + gq + 8) * 9 + 2 * tq + 1] = cacc[3];
        __syncthreads();
#pragma unroll
        for (int h = 0; h < 2; h++) rec[h] = Rs[(pr0 + 32 * h) * 9 + puu] + Rs[RB * 9 + (pr0 + 32 * h) * 9 + puu];
      }
    }
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int b = r0 + pr0 + 32 * h;
      if (b >= B) continue;
      const long long gbase = ((long long)s * B + b) * K4 + u0 + puu;
      const float ig = gates[gbase], fg = gates[gbase + R], gg = gates[gbase + 2LL * R], og = gates[gbase + 3LL * R];
      const long long o = ((long long)s * B + b) * R + u0 + puu;          // cs[s] = c_{s-1}, cs[s+1] = c_s
      const float cprev = cs[o], c = cs[o + (long long)B * R];
      const float dh = dhtop[o] + rec[h];
      const float tc = tanhf(c);
      const float dc = dh * og * (1.f - tc * tc) + dc_reg[h];
      dG[gbase] = dc * gg * ig * (1.f - ig);
      dG[gbase + R] = dc * cprev * fg * (1.f - fg);
      dG[gbase + 2LL * R] = dc * ig * (1.f - gg * gg);
      dG[gbase + 3LL * R] = dh * tc * og * (1.f - og);
      dc_reg[h] = dc * fg;
    }
  }
}

size_t g_fwd_attr = 0, g_bwd_attr = 0;  // largest dynamic shared memory size enabled so far

}  // namespace

static int cooperative_scan_fwd(const float* pre, const float* whh, const float* bhh, float* gates, float* hs, float* cs, int S, int B,
                                int R, int tf32, unsigned* counter, cudaStream_t st) {
  if (S <= 0 || B <= 0) return P2PVG_OK;
  P2PVG_REQUIRE(R % 8 == 0 && R % 4 == 0, P2PVG_ERR_UNSUPPORTED, "lstm_scan: hidden size %d must be a multiple of 8", R);
  const size_t smem = (size_t)(32 * (R + PAD) + RB * (R + PAD) + RB * 33) * sizeof(float);
  P2PVG_REQUIRE(smem <= 227 * 1024, P2PVG_ERR_UNSUPPORTED, "lstm_scan_fwd: hidden size %d needs %zu B of shared memory", R, smem);
  if (smem > g_fwd_attr) {
    cudaError_t e = cudaFuncSetAttribute(lstm_scan_fwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(lstm_scan_fwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { p2pvg_set_error("lstm_scan_fwd: %s", cudaGetErrorString(e)); return P2PVG_ERR_CUDA; }
    g_fwd_attr = smem;
  }
  const int grid = (R / UB) * cdiv(B, RB);
  void* args[] = {(void*)&pre, (void*)&whh, (void*)&bhh, (void*)&gates, (void*)&hs, (void*)&cs, (void*)&S, (void*)&B, (void*)&R, (void*)&counter};
  const void* kfn = tf32 ? (const void*)lstm_scan_fwd_kernel<true> : (const void*)lstm_scan_fwd_kernel<false>;
  cudaError_t e = cudaLaunchCooperativeKernel(kfn, dim3(grid), dim3(NT), args, smem, st);
  if (e != cudaSuccess) {
    p2pvg_set_error("lstm_scan_fwd: cooperative launch of %d CTAs failed: %s", grid, cudaGetErrorString(e));
    (void)cudaGetLastError();
    return P2PVG_ERR_CUDA;
  }
  return P2PVG_OK;
}

static int cooperative_scan_bwd(const float* dhtop, const float* whh, const float* gates, const float* cs, float* dG, int S, int B, int R,
                                int tf32, unsigned* counter, cudaStream_t st) {
  if (S <= 0 || B <= 0) return P2PVG_OK;
  P2PVG_REQUIRE(R % 64 == 0, P2PVG_ERR_UNSUPPORTED, "lstm_scan_bwd: hidden size %d must be a multiple of 64", R);
  const size_t smem = (size_t)(UB * (4 * R + PAD) + RB * (256 + PAD) + 2 * RB * 9) * sizeof(float);
  P2PVG_REQUIRE(smem <= 227 * 1024, P2PVG_ERR_UNSUPPORTED, "lstm_scan_bwd: hidden size %d needs %zu B of shared memory", R, smem);
  if (smem > g_bwd_attr) {
    cudaError_t e = cudaFuncSetAttribute(lstm_scan_bwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(lstm_scan_bwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { p2pvg_set_error("lstm_scan_bwd: %s", cudaGetErrorString(e)); return P2PVG_ERR_CUDA; }
    g_bwd_attr = smem;
  }
  const int grid = (R / UB) * cdiv(B, RB);
  void* args[] = {(void*)&dhtop, (void*)&whh, (void*)&gates, (void*)&cs, (void*)&dG, (void*)&S, (void*)&B, (void*)&R, (void*)&counter};
  const void* kfn = tf32 ? (const void*)lstm_scan_bwd_kernel<true> : (const void*)lstm_scan_bwd_kernel<false>;
  cudaError_t e = cudaLaunchCooperativeKernel(kfn, dim3(grid), dim3(NT), args, smem, st);
  if (e != cudaSuccess) {
    p2pvg_set_error("lstm_scan_bwd: cooperative launch of %d CTAs failed: %s", grid, cudaGetErrorString(e));
    (void)cudaGetLastError();
    return P2PVG_ERR_CUDA;
  }
  return P2PVG_OK;
}

// tensor-core mode: thread-block-cluster scans, clusters of 16 CTAs for R = 512 (BASELINE config 5, lstm_cluster512.cu) and of 8
// CTAs for R in {64,128,256} (lstm_cluster.cu); the exact-fp32 mode runs the cooperative-grid scans
extern "C" int p2pvg_lstm_scan_fwd(const float* pre, const float* whh, const float* bhh, float* gates, float* hs, float* cs, int S, int B,
                                   int R, int tf32, unsigned* counter, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (tf32 && R == 512) return p2pvg_lstm_cluster512_fwd(pre, whh, bhh, gates, hs, cs, S, B, st);
  if (tf32 && p2pvg_lstm_cluster_supported(R)) return p2pvg_lstm_cluster_fwd(pre, whh, bhh, gates, hs, cs, S, B, R, st);
  return cooperative_scan_fwd(pre, whh, bhh, gates, hs, cs, S, B, R, tf32, counter, st);
}

extern "C" int p2pvg_lstm_scan_bwd(const float* dhtop, const float* whh, const float* gates, const float* cs, float* dG, int S, int B, int R,
                                   int tf32, unsigned* counter, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (tf32 && R == 512) return p2pvg_lstm_cluster512_bwd(dhtop, whh, gates, cs, dG, S, B, st);
  if (tf32 && p2pvg_lstm_cluster_supported(R)) return p2pvg_lstm_cluster_bwd(dhtop, whh, gates, cs, dG, S, B, R, st);
  return cooperative_scan_bwd(dhtop, whh, gates, cs, dG, S, B, R, tf32, counter, st);
}
