// One timestep of one or two stand-alone LSTM modules (models/lstm.py:29-44, 83-94) in ONE launch: embed Linear, L x
// nn.LSTMCell and the head (Linear + tanh of `lstm`, or mu_net / logvar_net + reparameterize of `gaussian_lstm`).
//
// Clusters of 8 CTAs; a cluster owns a slab of up to SLAB batch rows, CTA rank r owns the hidden units [r R/8, (r+1) R/8)
// of the embed output and of every layer.  Each stage output (embed, every layer's h) is written by its owner CTA into a
// slice in its shared memory and gathered by all CTAs of the cluster through distributed shared memory between two cluster
// barriers.  Weights are streamed from L2 (one warp per output unit, lanes along K, coalesced); every product is an exact
// fp32 FFMA, the same arithmetic class as the CUDA-core GEMMs of the eager generation path.  blockIdx.y = module.
#include <cooperative_groups.h>

#include "cluster_rows.cuh"
#include "common.cuh"
#include "../../include/p2pvg_b200.h"

namespace cg = cooperative_groups;

namespace {

constexpr int CS = 8;        // CTAs per cluster
constexpr int SLAB = 8;      // batch rows per cluster
constexpr int NT = 256;      // threads per CTA
constexpr int NW = NT / 32;

// the module input row b: [ A[ia * rows + b, 0:ga] | Bm[ib * rows + b, 0:gb] | tuc | dt ], the counters of row b's group
__device__ __forceinline__ float in_elem(const p2pvg_lstm_step_module& m, int rows, int b, int k) {
  if (k < m.ga) return m.seg_a[((long long)m.idx_a[0] * rows + b) * m.ga + k];
  k -= m.ga;
  if (k < m.gb) return m.seg_b[((long long)m.idx_b[0] * rows + b) * m.gb + k];
  const int grp = m.counter_rows > 0 ? b / m.counter_rows : 0;
  return k == m.gb ? m.tuc[grp] : m.dt[grp];
}

// full[b][R] <- the slices [b][U] of all CTAs of the cluster
__device__ __forceinline__ void gather(cg::cluster_group& cl, float* slice, float* full, int U, int R, int nrows) {
  cl.sync();
  for (int i = threadIdx.x; i < CS * nrows * U; i += NT) {
    const int rank = i / (nrows * U), rem = i - rank * nrows * U, b = rem / U, u = rem - b * U;
    const float* src = cl.map_shared_rank(slice, rank);
    full[b * R + rank * U + u] = src[b * U + u];
  }
  cl.sync();   // no CTA may overwrite its slice while another one still reads it
}

__global__ void __cluster_dims__(CS, 1, 1) __launch_bounds__(NT, 1)
lstm_step_kernel(p2pvg_lstm_step_module m0, p2pvg_lstm_step_module m1, int rows, int R) {
  const p2pvg_lstm_step_module& m = blockIdx.y == 0 ? m0 : m1;
  cg::cluster_group cl = cg::this_cluster();
  const int rank = (int)cl.block_rank();
  const int b0 = (blockIdx.x / CS) * SLAB;
  const int nrows = min(SLAB, rows - b0);
  const int U = R / CS, u0 = rank * U;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int in_dim = m.ga + m.gb + 2;
  extern __shared__ float sm[];
  float* X = sm;                       // [SLAB][in_dim]   module input
  float* cur = X + SLAB * in_dim;      // [SLAB][R]        input of the current layer (embed output, then h of the layer below)
  float* hp = cur + SLAB * R;          // [SLAB][R]        h_{t-1} of the current layer
  float* slice = hp + SLAB * R;        // [SLAB][U]        this CTA's units of the stage output

  for (int i = threadIdx.x; i < nrows * in_dim; i += NT) {
    const int b = i / in_dim, k = i - b * in_dim;
    X[i] = in_elem(m, rows, b0 + b, k);
  }
  __syncthreads();
  float acc[SLAB], acc2[SLAB];
  // embed Linear
  for (int u = warp; u < U; u += NW) {
    warp_dot(m.w_embed + (long long)(u0 + u) * in_dim, X, in_dim, in_dim, nrows, lane, acc);
    if (lane == 0)
      for (int b = 0; b < nrows; b++) slice[b * U + u] = acc[b] + m.b_embed[u0 + u];
  }
  gather(cl, slice, cur, U, R, nrows);
  // L x LSTMCell: gates = x W_ih^T + b_ih + h W_hh^T + b_hh, order (i, f, g, o)
  for (int l = 0; l < m.layers; l++) {
    const float* const* wp = m.layer_w + 4 * l;     // w_ih, b_ih, w_hh, b_hh
    float* const* sp = m.state + 4 * l;             // h_in, c_in, h_out, c_out
    for (int i = threadIdx.x; i < nrows * R; i += NT) hp[i] = sp[0][(long long)b0 * R + i];
    cl.sync();   // every CTA holds h_in before any CTA writes h_out: the state may be updated in place
    for (int u = warp; u < U; u += NW) {
      float gt[4][SLAB];
#pragma unroll
      for (int q = 0; q < 4; q++) {
        const long long row = (long long)q * R + u0 + u;
        warp_dot(wp[0] + row * R, cur, R, R, nrows, lane, acc);
        warp_dot(wp[2] + row * R, hp, R, R, nrows, lane, acc2);
#pragma unroll
        for (int b = 0; b < SLAB; b++) gt[q][b] = (acc[b] + wp[1][row]) + (acc2[b] + wp[3][row]);
      }
      if (lane == 0) {
        for (int b = 0; b < nrows; b++) {
          const long long e = (long long)(b0 + b) * R + u0 + u;
          const float ig = sigmoidf_(gt[0][b]), fg = sigmoidf_(gt[1][b]), gg = tanhf(gt[2][b]), og = sigmoidf_(gt[3][b]);
          const float c = fg * sp[1][e] + ig * gg;
          const float h = og * tanhf(c);
          sp[3][e] = c;
          sp[2][e] = h;
          slice[b * U + u] = h;
        }
      }
    }
    gather(cl, slice, cur, U, R, nrows);   // also orders the h_in reads of this layer before any later overwrite
  }
  // head: outputs o split over the cluster (rank r takes o = r, r + 8, ...)
  if (m.head == P2PVG_LSTM_HEAD_LINEAR_TANH) {
    for (int o = rank + CS * warp; o < m.out_dim; o += CS * NW) {
      warp_dot(m.w_out + (long long)o * R, cur, R, R, nrows, lane, acc);
      if (lane == 0)
        for (int b = 0; b < nrows; b++) m.out[(long long)(b0 + b) * m.out_dim + o] = tanhf(acc[b] + m.b_out[o]);
    }
  } else {
    for (int o = rank + CS * warp; o < m.out_dim; o += CS * NW) {
      warp_dot(m.w_out + (long long)o * R, cur, R, R, nrows, lane, acc);
      warp_dot(m.w_out2 + (long long)o * R, cur, R, R, nrows, lane, acc2);
      if (lane == 0)
        for (int b = 0; b < nrows; b++) {
          const long long e = (long long)(b0 + b) * m.out_dim + o;
          const float mu = acc[b] + m.b_out[o], lv = acc2[b] + m.b_out2[o];
          if (m.mu) m.mu[e] = mu;
          if (m.logvar) m.logvar[e] = lv;
          m.out[e] = m.eps[e] * expf(0.5f * lv) + mu;   // reparameterize (models/lstm.py:76-81), as p2pvg_reparam_kl_fwd
        }
    }
  }
}

}  // namespace

int p2pvg_lstm_step_impl(const p2pvg_lstm_step_module* mods, int n_mods, int rows, int R, cudaStream_t st) {
  P2PVG_REQUIRE(mods != nullptr && (n_mods == 1 || n_mods == 2), P2PVG_ERR_BAD_ARG, "lstm_step: 1 or 2 modules");
  P2PVG_REQUIRE(R % CS == 0 && R >= 64 && R <= 512, P2PVG_ERR_UNSUPPORTED, "lstm_step: hidden size %d (64..512, multiple of 8)", R);
  int in_max = 0;
  for (int i = 0; i < n_mods; i++) {
    const p2pvg_lstm_step_module& m = mods[i];
    P2PVG_REQUIRE(m.layers >= 1 && m.layer_w && m.state && m.w_embed && m.b_embed && m.w_out && m.b_out && m.out, P2PVG_ERR_BAD_ARG,
                  "lstm_step: module %d incomplete", i);
    P2PVG_REQUIRE(m.seg_a && m.idx_a && m.ga >= 0 && m.gb >= 0 && (m.gb == 0 || (m.seg_b && m.idx_b)) && m.tuc && m.dt, P2PVG_ERR_BAD_ARG,
                  "lstm_step: module %d input segments", i);
    P2PVG_REQUIRE(m.head == P2PVG_LSTM_HEAD_LINEAR_TANH || (m.head == P2PVG_LSTM_HEAD_GAUSSIAN && m.w_out2 && m.b_out2 && m.eps),
                  P2PVG_ERR_BAD_ARG, "lstm_step: module %d head", i);
    P2PVG_REQUIRE(m.counter_rows >= 0, P2PVG_ERR_BAD_ARG, "lstm_step: module %d counter_rows %d (needs >= 0)", i, m.counter_rows);
    in_max = max(in_max, m.ga + m.gb + 2);
  }
  if (rows <= 0) return P2PVG_OK;
  const size_t smem = sizeof(float) * ((size_t)SLAB * in_max + 2 * (size_t)SLAB * R + (size_t)SLAB * (R / CS));
  static int attr_done = 0;
  if (smem > 48 * 1024 || !attr_done) {
    cudaError_t e = cudaFuncSetAttribute(lstm_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
    if (e != cudaSuccess) {
      p2pvg_set_error("lstm_step: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
      return P2PVG_ERR_CUDA;
    }
    attr_done = 1;
  }
  P2PVG_REQUIRE(smem <= 96 * 1024, P2PVG_ERR_UNSUPPORTED, "lstm_step: input too wide (%d)", in_max);
  dim3 grid(CS * ((rows + SLAB - 1) / SLAB), n_mods);
  lstm_step_kernel<<<grid, NT, smem, st>>>(mods[0], mods[n_mods - 1], rows, R);
  return p2pvg_check_launch("lstm_step");
}
