// The two thin ends of the vgg stacks in eval mode (generation, reference models/vgg_64.py:22 and :87-90): the first
// encoder layer (nc -> 64 channels, 3x3, BatchNorm on running statistics, LeakyReLU) and the closing ConvTranspose2d(64, nc,
// 3, 1, 1) + Sigmoid.  Both move 64 channels per pixel against <= 4 * 9 MACs per channel: HBM-bound, so they run on the CUDA
// cores in exact fp32 FFMA and read the fp32 parameters in PyTorch's layout (staged once per CTA in shared memory).  They
// replace nchw_to_nhwc + im2col3 + GEMM + bn_act and GEMM + col2im3 + cast + sigmoid + nhwc_to_nchw, and with them the
// [pixels, 9 * nc] column buffers.
#include "common.cuh"

namespace {

constexpr int BLOCK = 256;

inline int grid_for(long long total) {
  const long long g = (total + BLOCK - 1) / BLOCK, cap = 132LL * 16;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

// one thread per (pixel, group of 8 output channels): the 8 threads of a pixel read the same 9 * NC inputs (one warp
// instruction) and store 8 adjacent channels, so a pixel's 64 channels go out as one contiguous 128 / 256-byte row.
// Accumulation order per channel: (ci, kh, kw), the order of the weight in memory; out-of-map taps add 0 * w.
template <typename T, int NC>
__global__ void __launch_bounds__(BLOCK) vgg_first_eval_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                               const float* __restrict__ bias, const float* __restrict__ scale,
                                                               const float* __restrict__ shift, T* __restrict__ y, long long total,
                                                               int H, int W) {
  __shared__ __align__(16) float ws[NC * 9][64];   // [tap of (ci, kh, kw)][output channel]
  __shared__ __align__(16) float cs[3][64];        // bias, scale, shift
  for (int i = threadIdx.x; i < NC * 9 * 64; i += BLOCK) {
    const int k = i / 64, c = i - k * 64;
    ws[k][c] = w[c * NC * 9 + k];
  }
  for (int i = threadIdx.x; i < 64; i += BLOCK) {
    cs[0][i] = bias[i];
    cs[1][i] = scale[i];
    cs[2][i] = shift[i];
  }
  __syncthreads();
  const long long HW = (long long)H * W;
  for (long long idx = (long long)blockIdx.x * BLOCK + threadIdx.x; idx < total; idx += (long long)gridDim.x * BLOCK) {
    const int c0 = (int)(idx & 7) * 8;
    const long long pix = idx >> 3;
    const long long n = pix / HW;
    const int rem = (int)(pix - n * HW);
    const int yy = rem / W, xx = rem - yy * W;
    const float* xn = x + n * NC * HW;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; j++) acc[j] = 0.f;
#pragma unroll
    for (int ci = 0; ci < NC; ci++) {
#pragma unroll
      for (int kh = 0; kh < 3; kh++) {
        const int sy = yy + kh - 1;
#pragma unroll
        for (int kw = 0; kw < 3; kw++) {
          const int sx = xx + kw - 1;
          const float v = (sy >= 0 && sy < H && sx >= 0 && sx < W) ? __ldg(xn + ci * HW + (long long)sy * W + sx) : 0.f;
          const float4 wa = *reinterpret_cast<const float4*>(&ws[(ci * 3 + kh) * 3 + kw][c0]);
          const float4 wb = *reinterpret_cast<const float4*>(&ws[(ci * 3 + kh) * 3 + kw][c0 + 4]);
          acc[0] = fmaf(v, wa.x, acc[0]); acc[1] = fmaf(v, wa.y, acc[1]); acc[2] = fmaf(v, wa.z, acc[2]); acc[3] = fmaf(v, wa.w, acc[3]);
          acc[4] = fmaf(v, wb.x, acc[4]); acc[5] = fmaf(v, wb.y, acc[5]); acc[6] = fmaf(v, wb.z, acc[6]); acc[7] = fmaf(v, wb.w, acc[7]);
        }
      }
    }
    // the arithmetic of p2pvg_conv_gemm's eval epilogue: act(scale * (acc + bias) + shift)
#pragma unroll
    for (int j = 0; j < 8; j++) {
      const float z = fmaf(acc[j] + cs[0][c0 + j], cs[1][c0 + j], cs[2][c0 + j]);
      acc[j] = z > 0.f ? z : 0.2f * z;
    }
    T* dst = y + pix * 64 + c0;
    if constexpr (sizeof(T) == 2) {
      st_raw16(dst, pack16<T>(acc));
    } else {
      st_raw16(dst, pack16<T>(acc));
      st_raw16(dst + 4, pack16<T>(acc + 4));
    }
  }
}

// one thread per output pixel, all NC channels: the 9 neighbouring input rows of 64 channels are read as 16-byte vectors
// (32 consecutive pixels of a warp read 32 consecutive rows per tap), every weight is a shared-memory broadcast.
// Accumulation order per channel: (kh, kw, ci), then + bias, then the sigmoid; out-of-map taps are skipped.
template <typename T, int NC>
__global__ void __launch_bounds__(BLOCK) vgg_last_eval_kernel(const T* __restrict__ d, const float* __restrict__ w,
                                                              const float* __restrict__ bias, float* __restrict__ out, long long npix,
                                                              int H, int W) {
  constexpr int V = VecN<T>::N;
  __shared__ float ws[9 * 64 * NC];   // [kh][kw][ci][c]
  for (int i = threadIdx.x; i < 9 * 64 * NC; i += BLOCK) {
    const int c = i % NC, ci = (i / NC) % 64, tap = i / (NC * 64);
    ws[i] = w[(ci * NC + c) * 9 + tap];
  }
  __syncthreads();
  const long long HW = (long long)H * W;
  for (long long pix = (long long)blockIdx.x * BLOCK + threadIdx.x; pix < npix; pix += (long long)gridDim.x * BLOCK) {
    const long long n = pix / HW;
    const int rem = (int)(pix - n * HW);
    const int yy = rem / W, xx = rem - yy * W;
    float acc[NC];
#pragma unroll
    for (int c = 0; c < NC; c++) acc[c] = 0.f;
#pragma unroll 1
    for (int tap = 0; tap < 9; tap++) {
      const int kh = tap / 3, kw = tap - kh * 3;
      const int sy = yy + 1 - kh, sx = xx + 1 - kw;
      if (sy < 0 || sy >= H || sx < 0 || sx >= W) continue;
      const T* src = d + ((n * H + sy) * W + sx) * 64;
      const float* wt = ws + tap * 64 * NC;
#pragma unroll
      for (int v0 = 0; v0 < 64; v0 += V) {
        float f[V];
        unpack16<T>(ld_raw16(src + v0), f);
#pragma unroll
        for (int i = 0; i < V; i++)
#pragma unroll
          for (int c = 0; c < NC; c++) acc[c] = fmaf(f[i], wt[(v0 + i) * NC + c], acc[c]);
      }
    }
#pragma unroll
    for (int c = 0; c < NC; c++) out[(n * NC + c) * HW + rem] = sigmoidf_(acc[c] + __ldg(bias + c));
  }
}

template <typename T>
int first_nc(int nc, const float* x, const float* w, const float* bias, const float* scale, const float* shift, void* y, long long total,
             int H, int W, cudaStream_t st) {
  const int grid = grid_for(total);
  switch (nc) {
    case 1: vgg_first_eval_kernel<T, 1><<<grid, BLOCK, 0, st>>>(x, w, bias, scale, shift, (T*)y, total, H, W); break;
    case 2: vgg_first_eval_kernel<T, 2><<<grid, BLOCK, 0, st>>>(x, w, bias, scale, shift, (T*)y, total, H, W); break;
    case 3: vgg_first_eval_kernel<T, 3><<<grid, BLOCK, 0, st>>>(x, w, bias, scale, shift, (T*)y, total, H, W); break;
    default: vgg_first_eval_kernel<T, 4><<<grid, BLOCK, 0, st>>>(x, w, bias, scale, shift, (T*)y, total, H, W); break;
  }
  return p2pvg_check_launch("vgg_first_eval");
}

template <typename T>
int last_nc(int nc, const void* d, const float* w, const float* bias, float* out, long long npix, int H, int W, cudaStream_t st) {
  const int grid = grid_for(npix);
  switch (nc) {
    case 1: vgg_last_eval_kernel<T, 1><<<grid, BLOCK, 0, st>>>((const T*)d, w, bias, out, npix, H, W); break;
    case 2: vgg_last_eval_kernel<T, 2><<<grid, BLOCK, 0, st>>>((const T*)d, w, bias, out, npix, H, W); break;
    case 3: vgg_last_eval_kernel<T, 3><<<grid, BLOCK, 0, st>>>((const T*)d, w, bias, out, npix, H, W); break;
    default: vgg_last_eval_kernel<T, 4><<<grid, BLOCK, 0, st>>>((const T*)d, w, bias, out, npix, H, W); break;
  }
  return p2pvg_check_launch("vgg_last_eval");
}

}  // namespace

extern "C" int p2pvg_vgg_first_eval(const float* x, int nc, const float* w, const float* bias, const float* scale, const float* shift,
                                    void* y, int y_dtype, int N, int H, int W, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  P2PVG_REQUIRE(x && w && bias && scale && shift && y, P2PVG_ERR_BAD_ARG, "vgg_first_eval: null argument");
  P2PVG_REQUIRE(N >= 0 && H >= 1 && W >= 1, P2PVG_ERR_BAD_ARG, "vgg_first_eval: bad size N=%d H=%d W=%d", N, H, W);
  P2PVG_REQUIRE((reinterpret_cast<uintptr_t>(y) & 15) == 0, P2PVG_ERR_BAD_ARG, "vgg_first_eval: y must be 16-byte aligned");
  P2PVG_REQUIRE(nc >= 1 && nc <= 4, P2PVG_ERR_UNSUPPORTED, "vgg_first_eval: nc = %d (1..4 supported)", nc);
  if (N == 0) return P2PVG_OK;
  const long long total = (long long)N * H * W * 8;
  DISPATCH_DTYPE(y_dtype, T, return first_nc<T>(nc, x, w, bias, scale, shift, y, total, H, W, st));
  return P2PVG_OK;
}

extern "C" int p2pvg_vgg_last_eval(const void* d, int d_dtype, const float* w, const float* bias, float* out, int nc, int N, int H, int W,
                                   void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  P2PVG_REQUIRE(d && w && bias && out, P2PVG_ERR_BAD_ARG, "vgg_last_eval: null argument");
  P2PVG_REQUIRE(N >= 0 && H >= 1 && W >= 1, P2PVG_ERR_BAD_ARG, "vgg_last_eval: bad size N=%d H=%d W=%d", N, H, W);
  P2PVG_REQUIRE((reinterpret_cast<uintptr_t>(d) & 15) == 0, P2PVG_ERR_BAD_ARG, "vgg_last_eval: d must be 16-byte aligned");
  P2PVG_REQUIRE(nc >= 1 && nc <= 4, P2PVG_ERR_UNSUPPORTED, "vgg_last_eval: nc = %d (1..4 supported)", nc);
  if (N == 0) return P2PVG_OK;
  DISPATCH_DTYPE(d_dtype, T, return last_nc<T>(nc, d, w, bias, out, (long long)N * H * W, H, W, st));
  return P2PVG_OK;
}
