// One whole call of the h36m pose encoder or decoder (models/h36m_mlp.py:28-95) in ONE launch: two residual_linear blocks and
// the final Linear, as the eager path's GEMM / activation / accumulate / LayerNorm sequence computes them (infer.py).
//
// Clusters of 8 CTAs; a cluster owns a slab of up to SLAB rows, CTA rank r owns the output units [r n / 8, (r + 1) n / 8) of
// every Linear (n = 25 or 51 splits unevenly).  The owner of a unit pushes its value into the stage buffer of every CTA of the
// cluster through distributed shared memory; one cluster barrier per stage then makes the full row visible everywhere.  A unit's
// shortcut and long-path outputs have the same owner, so the residual add is local; after the push every CTA holds the whole
// pre-norm row and applies the LayerNorm itself.  Weights are streamed from L2 (one warp per output unit, lanes along K);
// every product is an exact fp32 FFMA, the arithmetic class of the eager path's exact fp32 GEMMs.
#include <cooperative_groups.h>

#include "cluster_rows.cuh"
#include "common.cuh"

namespace cg = cooperative_groups;

namespace {

constexpr int CS = 8;        // CTAs per cluster
constexpr int SLAB = 8;      // rows per cluster
constexpr int NT = 256;      // threads per CTA
constexpr int NW = NT / 32;
constexpr int POSE = 17 * 3;
constexpr float LN_EPS = 1e-5f;   // nn.LayerNorm default (models/h36m_mlp.py:43)
constexpr size_t SMEM_MAX = 227 * 1024;

// first unit of CTA rank r when n units are split over the cluster
__device__ __forceinline__ int unit0(int r, int n) { return r * n / CS; }

// acc[b] for a run-time b, without spilling acc to local memory
__device__ __forceinline__ float pick(const float (&acc)[SLAB], int b) {
  float v = acc[0];
#pragma unroll
  for (int i = 1; i < SLAB; i++)
    if (i == b) v = acc[i];
  return v;
}

// dst[b * ld + col] = f(acc[b], b) in every CTA of the cluster; lane t stores row t % SLAB into ranks t / SLAB and t / SLAB + 4
template <class F>
__device__ __forceinline__ void push(cg::cluster_group& cl, float* dst, int ld, int col, const float (&acc)[SLAB], int nrows,
                                     int lane, F f) {
  for (int t = lane; t < SLAB * CS; t += 32) {
    const int b = t % SLAB, r = t / SLAB;
    if (b < nrows) cl.map_shared_rank(dst, r)[b * ld + col] = f(pick(acc, b), b);
  }
}

// dst[b][0:nout] (local, pitch ldd) = residual_linear(src[b][0:nin]) (pitch lds) for the slab's rows.  P / Q: long-path
// stages [SLAB][nin / 2], Y: pre-norm rows [SLAB][nout], SC: this CTA's shortcut units [SLAB][nout].
__device__ void residual(cg::cluster_group& cl, const p2pvg_pose_residual& p, const float* src, int lds, int nin, int nout,
                         float* P, float* Q, float* Y, float* SC, float* dst, int ldd, int nrows, int rank) {
  const int half = nin / 2;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h0 = unit0(rank, half), nh = unit0(rank + 1, half) - h0;
  const int s0 = unit0(rank, nout), ns = unit0(rank + 1, nout) - s0;
  float acc[SLAB];
  // L1 (relu) everywhere, the shortcut (relu) kept locally
  for (int u = warp; u < nh + ns; u += NW) {
    if (u < nh) {
      const int o = h0 + u;
      warp_dot(p.w1 + (long long)o * nin, src, lds, nin, nrows, lane, acc);
      const float bias = __ldg(p.b1 + o);
      push(cl, P, half, o, acc, nrows, lane, [&](float v, int) { return fmaxf(v + bias, 0.f); });
    } else {
      const int o = s0 + u - nh;
      warp_dot(p.w_sc + (long long)o * nin, src, lds, nin, nrows, lane, acc);
      const float bias = __ldg(p.b_sc + o);
      if (lane < nrows) SC[lane * nout + o] = fmaxf(pick(acc, lane) + bias, 0.f);
    }
  }
  cl.sync();
  // L2 (relu)
  for (int u = warp; u < nh; u += NW) {
    const int o = h0 + u;
    warp_dot(p.w2 + (long long)o * half, P, half, half, nrows, lane, acc);
    const float bias = __ldg(p.b2 + o);
    push(cl, Q, half, o, acc, nrows, lane, [&](float v, int) { return fmaxf(v + bias, 0.f); });
  }
  cl.sync();
  // L3 (relu) + shortcut: the pre-norm row, everywhere
  for (int u = warp; u < ns; u += NW) {
    const int o = s0 + u;
    warp_dot(p.w3 + (long long)o * half, Q, half, half, nrows, lane, acc);
    const float bias = __ldg(p.b3 + o);
    push(cl, Y, nout, o, acc, nrows, lane, [&](float v, int b) { return SC[b * nout + o] + fmaxf(v + bias, 0.f); });
  }
  cl.sync();
  // LayerNorm of every row in every CTA (the arithmetic of layernorm_fwd_kernel, mlp.cu)
  for (int b = warp; b < nrows; b += NW) {
    const float* y = Y + b * nout;
    float s = 0.f;
    for (int c = lane; c < nout; c += 32) s += y[c];
    s = warp_sum(s);
    const float m = s / (float)nout;
    float v = 0.f;
    for (int c = lane; c < nout; c += 32) {
      const float d = y[c] - m;
      v = fmaf(d, d, v);
    }
    v = warp_sum(v);
    const float r = rsqrtf(v / (float)nout + LN_EPS);
    for (int c = lane; c < nout; c += 32) dst[b * ldd + c] = (y[c] - m) * r * __ldg(p.gamma + c) + __ldg(p.beta + c);
  }
  __syncthreads();
}

// this CTA's columns of the slab's rows x[b][0:n] (pitch ldx) -> out[(b0 + b) * n + c]
__device__ __forceinline__ void store_cols(const float* x, int ldx, int n, float* out, int b0, int nrows, int rank) {
  const int c0 = unit0(rank, n), nc = unit0(rank + 1, n) - c0;
  for (int i = threadIdx.x; i < nrows * nc; i += NT) {
    const int b = i / nc, c = c0 + i - b * nc;
    out[(long long)(b0 + b) * n + c] = x[b * ldx + c];
  }
}

__global__ void __cluster_dims__(CS, 1, 1) __launch_bounds__(NT, 1)
pose_mlp_kernel(p2pvg_pose_mlp_args a, int rows, int ldx, int hmax) {
  cg::cluster_group cl = cg::this_cluster();
  const int rank = (int)cl.block_rank();
  const int b0 = (blockIdx.x / CS) * SLAB;
  const int nrows = min(SLAB, rows - b0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = a.g;
  extern __shared__ float sm[];
  float* XA = sm;                   // [SLAB][ldx]  input; encoder h2 / decoder [d2 | skip1]
  float* XB = XA + SLAB * ldx;      // [SLAB][ldx]  encoder h1 / decoder [d1 | skip2]
  float* P = XB + SLAB * ldx;       // [SLAB][hmax] long-path stages
  float* Q = P + SLAB * hmax;
  float* Y = Q + SLAB * hmax;       // [SLAB][g]    pre-norm rows
  float* SC = Y + SLAB * g;         // [SLAB][g]    this CTA's shortcut units

  const int in_dim = a.decoder ? g : POSE;
  const float* in = a.src + ((long long)(a.src_idx ? a.src_idx[0] : 0) * rows + b0) * in_dim;
  for (int i = threadIdx.x; i < nrows * in_dim; i += NT) {
    const int b = i / in_dim, k = i - b * in_dim;
    XA[b * ldx + k] = in[(long long)b * in_dim + k];
  }
  if (a.decoder) {
    for (int i = threadIdx.x; i < nrows * g; i += NT) {
      const int b = i / g, k = i - b * g;
      const long long sr = (b0 + b) % a.nsrc;
      XB[b * ldx + g + k] = a.skip2[sr * g + k];
      XA[b * ldx + g + k] = a.skip1[sr * g + k];
    }
  }
  cl.sync();   // every CTA of the cluster runs (its shared memory may be written) and the slab is loaded
  float acc[SLAB];
  if (!a.decoder) {
    residual(cl, a.fc1, XA, ldx, POSE, g, P, Q, Y, SC, XB, ldx, nrows, rank);
    if (a.h1) store_cols(XB, ldx, g, a.h1, b0, nrows, rank);
    residual(cl, a.fc2, XB, ldx, g, g, P, Q, Y, SC, XA, ldx, nrows, rank);
    if (a.h2) store_cols(XA, ldx, g, a.h2, b0, nrows, rank);
    const int o0 = unit0(rank, g), no = unit0(rank + 1, g) - o0;
    for (int u = warp; u < no; u += NW) {
      const int o = o0 + u;
      warp_dot(a.w3 + (long long)o * g, XA, ldx, g, nrows, lane, acc);
      if (lane < nrows) a.out[(long long)(b0 + lane) * g + o] = tanhf(pick(acc, lane) + __ldg(a.b3 + o));
    }
  } else {
    residual(cl, a.fc1, XA, ldx, g, g, P, Q, Y, SC, XB, ldx, nrows, rank);
    residual(cl, a.fc2, XB, ldx, 2 * g, g, P, Q, Y, SC, XA, ldx, nrows, rank);
    const int o0 = unit0(rank, POSE), no = unit0(rank + 1, POSE) - o0;
    for (int u = warp; u < no; u += NW) {
      const int o = o0 + u;
      warp_dot(a.w3 + (long long)o * 2 * g, XA, ldx, 2 * g, nrows, lane, acc);
      if (lane < nrows) a.out[(long long)(b0 + lane) * POSE + o] = pick(acc, lane) + __ldg(a.b3 + o);
    }
  }
}

bool residual_complete(const p2pvg_pose_residual& p) {
  return p.w_sc && p.b_sc && p.w1 && p.b1 && p.w2 && p.b2 && p.w3 && p.b3 && p.gamma && p.beta;
}

}  // namespace

extern "C" int p2pvg_pose_mlp(const p2pvg_pose_mlp_args* args, int rows, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  P2PVG_REQUIRE(args != nullptr && rows >= 0, P2PVG_ERR_BAD_ARG, "pose_mlp: bad arguments");
  const p2pvg_pose_mlp_args& a = *args;
  P2PVG_REQUIRE(a.g >= 8, P2PVG_ERR_BAD_ARG, "pose_mlp: g = %d (>= 8)", a.g);
  P2PVG_REQUIRE(a.src && a.out && a.w3 && a.b3 && residual_complete(a.fc1) && residual_complete(a.fc2), P2PVG_ERR_BAD_ARG,
                "pose_mlp: NULL input, output or weight");
  P2PVG_REQUIRE(!a.decoder || (a.skip1 && a.skip2 && a.nsrc >= 1), P2PVG_ERR_BAD_ARG, "pose_mlp: decoder skips (nsrc %d)", a.nsrc);
  const int g = a.g;
  const int ldx = a.decoder ? 2 * g : max(POSE, g);
  const int hmax = a.decoder ? g : max(POSE / 2, g / 2);
  const size_t smem = sizeof(float) * SLAB * (2 * (size_t)ldx + 2 * (size_t)hmax + 2 * (size_t)g);
  P2PVG_REQUIRE(smem <= SMEM_MAX, P2PVG_ERR_UNSUPPORTED, "pose_mlp: g = %d needs %zu bytes of shared memory per CTA", g, smem);
  if (rows == 0) return P2PVG_OK;
  static size_t attr = 48 * 1024;
  if (smem > attr) {
    cudaError_t e = cudaFuncSetAttribute(pose_mlp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_MAX);
    if (e != cudaSuccess) {
      p2pvg_set_error("pose_mlp: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
      return P2PVG_ERR_CUDA;
    }
    attr = SMEM_MAX;
  }
  pose_mlp_kernel<<<CS * ((rows + SLAB - 1) / SLAB), NT, smem, st>>>(a, rows, ldx, hmax);
  return p2pvg_check_launch("pose_mlp");
}
