// Scores of generated frames and poses against the ground truth (include/p2pvg_b200.h): per pair MSE, PSNR and 7x7
// uniform-window SSIM for frames, MSE and MPJPE for poses.
//
// Frames: one CTA scores one pair in a single pass.  It walks the pair's channels in strips of FM_SH rows: each strip is
// loaded once (float4, the next strip's loads issued before this one is processed), the squared differences are summed
// from the registers that loaded them, and the strip goes to shared memory.  The five horizontal 7-tap sums (x, y, x^2,
// y^2, xy) of every strip row land in a ring of FM_RING rows; each window whose bottom row is in the strip then sums its 7
// ring rows and evaluates S.  Every window sum is a fresh 7 + 7 term sum (no running add-new / subtract-old sums, whose
// error grows with the row count).  Per-pixel arithmetic is fp32 on values shifted by the channel's first pixel (the
// variances are shift-invariant; the shift removes the cancellation of mean(x^2) - mean(x)^2 on flat or bright frames);
// each thread adds its squared differences and S values into fp64 in a fixed order and the CTA reduces those in a fixed
// order, so a pair's result does not depend on the launch it is part of.  Nothing but the result goes to global memory.
//
// Poses: one warp per pair, fp64 throughout.
#include "common.cuh"

#include <math.h>

#define FM_THREADS 128
#define FM_SH 8                      // input rows per strip
#define FM_RING 16                   // rows of horizontal sums kept: a power of two >= FM_SH + 6
#define FM_MAX_W 128                 // widest frame the shared-memory tiles cover
#define FM_VEC ((FM_SH * FM_MAX_W / 4 + FM_THREADS - 1) / FM_THREADS)   // float4 loads per thread and frame per strip
#define PM_THREADS 128

static_assert(FM_RING >= FM_SH + 6 && (FM_RING & (FM_RING - 1)) == 0, "ring must hold a window's 7 rows past a strip");

namespace {

// ring rows are padded to a multiple of 4 floats so that the horizontal phase stores 4 window sums as one float4
__host__ __device__ __forceinline__ int ring_stride(int W) { return W - 4; }   // (W - 6) rounded up to a multiple of 4

size_t frame_metrics_smem(int W) { return (size_t)(2 * FM_SH * W + 5 * FM_RING * ring_stride(W)) * sizeof(float); }

// Four consecutive 7-tap box sums o[k] = v[k] + ... + v[k + 6], each a fresh fixed-order sum of its own 7 terms; the terms
// v[3..6] that all four share are added once.
__device__ __forceinline__ void box7x4(const float (&v)[10], float (&o)[4]) {
  const float c = (v[3] + v[4]) + (v[5] + v[6]);
  const float l1 = v[1] + v[2], r2 = v[7] + v[8];
  o[0] = (v[0] + l1) + c;
  o[1] = (l1 + c) + v[7];
  o[2] = (v[2] + c) + r2;
  o[3] = c + (r2 + v[9]);
}

__global__ void __launch_bounds__(FM_THREADS) frame_metrics_kernel(const float* __restrict__ pred, const float* __restrict__ gt,
                                                                    const int32_t* __restrict__ pairs, int C, int H, int W,
                                                                    float c1, float c2, double range2, double* __restrict__ out) {
  extern __shared__ __align__(16) float sm[];
  __shared__ double red[2][FM_THREADS / 32];
  const int Wv = W - 6, Wp = ring_stride(W), W4 = W / 4, Wg = Wp / 4, tid = threadIdx.x;
  float* xs = sm;                      // [FM_SH][W] pred strip
  float* ys = xs + FM_SH * W;          // [FM_SH][W] gt strip
  float* hs = ys + FM_SH * W;          // [5][FM_RING][Wp] horizontal sums of x, y, x^2, y^2, xy
  const int qs = FM_RING * Wp;         // stride between the five quantities
  const size_t fsz = (size_t)C * H * W;
  const float4* P = reinterpret_cast<const float4*>(pred + (size_t)pairs[2 * blockIdx.x] * fsz);
  const float4* G = reinterpret_cast<const float4*>(gt + (size_t)pairs[2 * blockIdx.x + 1] * fsz);
  const int nsc = (H + FM_SH - 1) / FM_SH, nstrip = C * nsc;

  float4 rx[FM_VEC], ry[FM_VEC];
  auto load = [&](int t) {
    const int c = t / nsc, r0 = (t - c * nsc) * FM_SH, n4 = min(FM_SH, H - r0) * W4;
    const size_t base = ((size_t)c * H + r0) * W4;
#pragma unroll
    for (int u = 0; u < FM_VEC; ++u) {
      const int i = tid + u * FM_THREADS;
      if (i < n4) {
        rx[u] = __ldcs(P + base + i);   // generated frames are read once
        ry[u] = __ldg(G + base + i);    // ground truth: the samples of one frame follow each other, L2 serves the repeats
      }
    }
  };

  double acc_se = 0.0, acc_s = 0.0;
  float shx = 0.f, shy = 0.f;
  load(0);
  for (int t = 0; t < nstrip; ++t) {
    const int c = t / nsc, r0 = (t - c * nsc) * FM_SH, nr = min(FM_SH, H - r0);
#pragma unroll
    for (int u = 0; u < FM_VEC; ++u) {
      const int i = tid + u * FM_THREADS;
      if (i < nr * W4) {
        const float4 a = rx[u], b = ry[u];
        const float d0 = a.x - b.x, d1 = a.y - b.y, d2 = a.z - b.z, d3 = a.w - b.w;
        acc_se += (double)(d0 * d0);
        acc_se += (double)(d1 * d1);
        acc_se += (double)(d2 * d2);
        acc_se += (double)(d3 * d3);
        reinterpret_cast<float4*>(xs)[i] = a;
        reinterpret_cast<float4*>(ys)[i] = b;
      }
    }
    if (t + 1 < nstrip) load(t + 1);
    __syncthreads();
    if (r0 == 0) {   // first strip of a channel
      shx = xs[0];
      shy = ys[0];
    }
    // horizontal sums of 4 consecutive window columns j0 .. j0 + 3 per item, from 10 pixels (three float4 reads; the reads
    // past a row's end only feed columns >= Wv, which land in the ring's padding and are never read)
    for (int k = tid; k < nr * Wg; k += FM_THREADS) {
      const int row = k / Wg, j0 = (k - row * Wg) * 4;
      float a[10], b[10], v[10], o[4];
#pragma unroll
      for (int e = 0; e < 3; ++e) {
        const float4 fx = *reinterpret_cast<const float4*>(xs + row * W + j0 + 4 * e);
        const float4 fy = *reinterpret_cast<const float4*>(ys + row * W + j0 + 4 * e);
        const float px[4] = {fx.x, fx.y, fx.z, fx.w}, py[4] = {fy.x, fy.y, fy.z, fy.w};
#pragma unroll
        for (int z = 0; z < 4; ++z)
          if (4 * e + z < 10) {
            a[4 * e + z] = px[z] - shx;
            b[4 * e + z] = py[z] - shy;
          }
      }
      float* h = hs + ((r0 + row) & (FM_RING - 1)) * Wp + j0;
#pragma unroll
      for (int q = 0; q < 5; ++q) {
#pragma unroll
        for (int d = 0; d < 10; ++d) v[d] = q == 0 ? a[d] : q == 1 ? b[d] : q == 2 ? a[d] * a[d] : q == 3 ? b[d] * b[d] : a[d] * b[d];
        box7x4(v, o);
        *reinterpret_cast<float4*>(h + q * qs) = make_float4(o[0], o[1], o[2], o[3]);
      }
    }
    __syncthreads();
    // windows whose bottom row lies in this strip: top rows o_lo .. o_lo + n_o - 1, four consecutive top rows per item (the
    // rows past the last window read ring rows of no window; their results are dropped)
    const int o_lo = max(r0 - 6, 0), n_o = r0 + nr - 6 - o_lo;
    const int n_g = (n_o + 3) / 4;
    for (int k = tid; k < n_g * Wv; k += FM_THREADS) {
      const int gi = k / Wv, j = k - gi * Wv, o0 = o_lo + 4 * gi;
      float s[5][4], v[10];
#pragma unroll
      for (int q = 0; q < 5; ++q) {
#pragma unroll
        for (int d = 0; d < 10; ++d) v[d] = hs[q * qs + ((o0 + d) & (FM_RING - 1)) * Wp + j];
        box7x4(v, s[q]);
      }
      const float inv49 = 1.f / 49.f, unb = 49.f / 48.f;
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        if (4 * gi + r >= n_o) break;
        const float mx = s[0][r] * inv49, my = s[1][r] * inv49;   // shifted means
        const float vx = unb * (s[2][r] * inv49 - mx * mx), vy = unb * (s[3][r] * inv49 - my * my);
        const float vxy = unb * (s[4][r] * inv49 - mx * my);
        const float ux = mx + shx, uy = my + shy;
        const float num = (2.f * ux * uy + c1) * (2.f * vxy + c2);
        const float den = (ux * ux + uy * uy + c1) * (vx + vy + c2);
        acc_s += (double)(num / den);
      }
    }
  }
  acc_se = warp_sum_d(acc_se);
  acc_s = warp_sum_d(acc_s);
  if ((tid & 31) == 0) {
    red[0][tid >> 5] = acc_se;
    red[1][tid >> 5] = acc_s;
  }
  __syncthreads();
  if (tid == 0) {
    double se = 0.0, ss = 0.0;
#pragma unroll
    for (int w = 0; w < FM_THREADS / 32; ++w) {
      se += red[0][w];
      ss += red[1][w];
    }
    const double mse = se / (double)fsz;
    double* o = out + 3 * (size_t)blockIdx.x;
    o[0] = mse;
    o[1] = mse == 0.0 ? (double)INFINITY : 10.0 * log10(range2 / mse);
    o[2] = ss / ((double)C * (H - 6) * (W - 6));
  }
}

__global__ void __launch_bounds__(PM_THREADS) pose_metrics_kernel(const float* __restrict__ pred, const float* __restrict__ gt,
                                                                  const int32_t* __restrict__ pairs, int n_pairs, int J,
                                                                  double* __restrict__ out) {
  const int p = blockIdx.x * (PM_THREADS / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (p >= n_pairs) return;
  const float* a = pred + (size_t)pairs[2 * p] * J * 3;
  const float* b = gt + (size_t)pairs[2 * p + 1] * J * 3;
  double se = 0.0, dist = 0.0;
  for (int j = lane; j < J; j += 32) {
    const double dx = (double)a[3 * j] - b[3 * j], dy = (double)a[3 * j + 1] - b[3 * j + 1], dz = (double)a[3 * j + 2] - b[3 * j + 2];
    const double d2 = dx * dx + dy * dy + dz * dz;
    se += d2;
    dist += sqrt(d2);
  }
  se = warp_sum_d(se);
  dist = warp_sum_d(dist);
  if (lane == 0) {
    out[2 * (size_t)p] = se / (3.0 * J);
    out[2 * (size_t)p + 1] = dist / J;
  }
}

}  // namespace

extern "C" int p2pvg_frame_metrics(const float* pred, const float* gt, const int32_t* pairs, int n_pairs, int C, int H, int W,
                                   float data_range, double* out, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  P2PVG_REQUIRE(pred && gt && ((pairs && out) || n_pairs == 0), P2PVG_ERR_BAD_ARG, "frame_metrics: null pointer");
  P2PVG_REQUIRE(((uintptr_t)pred & 15) == 0 && ((uintptr_t)gt & 15) == 0 && ((uintptr_t)pairs & 3) == 0 &&
                    ((uintptr_t)out & 7) == 0,
                P2PVG_ERR_BAD_ARG, "frame_metrics: pred / gt must be 16-byte, pairs 4-byte and out 8-byte aligned");
  P2PVG_REQUIRE(C >= 1 && H >= 7 && W >= 8 && W % 4 == 0, P2PVG_ERR_BAD_ARG,
                "frame_metrics: C = %d, H = %d, W = %d (needs C >= 1, H >= 7, W >= 8, W %% 4 == 0)", C, H, W);
  P2PVG_REQUIRE(n_pairs >= 0, P2PVG_ERR_BAD_ARG, "frame_metrics: n_pairs = %d", n_pairs);
  P2PVG_REQUIRE(isfinite(data_range) && data_range > 0.f, P2PVG_ERR_BAD_ARG, "frame_metrics: data_range = %g", (double)data_range);
  P2PVG_REQUIRE(W <= FM_MAX_W, P2PVG_ERR_UNSUPPORTED, "frame_metrics: W = %d (at most %d)", W, FM_MAX_W);
  P2PVG_REQUIRE((long long)C * H * W < (1LL << 31), P2PVG_ERR_UNSUPPORTED, "frame_metrics: C * H * W = %lld", (long long)C * H * W);
  if (n_pairs == 0) return P2PVG_OK;
  const float c1 = (0.01f * data_range) * (0.01f * data_range), c2 = (0.03f * data_range) * (0.03f * data_range);
  frame_metrics_kernel<<<n_pairs, FM_THREADS, frame_metrics_smem(W), st>>>(pred, gt, pairs, C, H, W, c1, c2,
                                                                           (double)data_range * data_range, out);
  return p2pvg_check_launch("frame_metrics");
}

extern "C" int p2pvg_pose_metrics(const float* pred, const float* gt, const int32_t* pairs, int n_pairs, int J, double* out, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  P2PVG_REQUIRE(pred && gt && ((pairs && out) || n_pairs == 0), P2PVG_ERR_BAD_ARG, "pose_metrics: null pointer");
  P2PVG_REQUIRE(((uintptr_t)pred & 3) == 0 && ((uintptr_t)gt & 3) == 0 && ((uintptr_t)pairs & 3) == 0 && ((uintptr_t)out & 7) == 0,
                P2PVG_ERR_BAD_ARG, "pose_metrics: misaligned pointer");
  P2PVG_REQUIRE(J >= 1 && n_pairs >= 0, P2PVG_ERR_BAD_ARG, "pose_metrics: J = %d, n_pairs = %d", J, n_pairs);
  if (n_pairs == 0) return P2PVG_OK;
  const int per = PM_THREADS / 32;
  pose_metrics_kernel<<<(n_pairs + per - 1) / per, PM_THREADS, 0, st>>>(pred, gt, pairs, n_pairs, J, out);
  return p2pvg_check_launch("pose_metrics");
}
