// The two ends of the dcgan stacks have 1 or 3 image channels on one side: too thin for tensor-core tiles and purely
// HBM-bound (they read or write the widest activation of the network).  Direct CUDA-core kernels, fp32 master weights.
//
//   conv_thin_in : y[N,H/2,W/2,Co] = conv4x4/s2/p1(x[N,H,W,Ci]),  Ci in {1,3}, weights [Co][Ci][4][4]
//                  - encoder c1 forward                         (models/dcgan_64.py:34, nn.Conv2d(nc, 64, 4, 2, 1))
//                  - data-gradient of the last decoder layer    (models/dcgan_64.py:76, nn.ConvTranspose2d(128, nc, 4, 2, 1)):
//                    the ConvT weight [Cin][nc][4][4] has exactly this layout with Co = Cin
//   convT_thin_out: y[N,2H,2W,Co] = convT4x4/s2/p1(x[N,H,W,Ci]) + bias + addend[src],  Co in {1,3}, weights [Ci][Co][4][4]
//                  - last decoder layer forward; the skip half of the concatenated input is evaluated once per distinct
//                    source call into an fp32 `addend` and indexed through grp_src (as in conv_gemm kind 2)
#include "common.cuh"

namespace {

// thread = (8/4-channel output vector cv, pixel lane): the filter taps of its output channels live in REGISTERS (CI == 1) or are
// read as float4 from shared memory (CI == 3); per pixel only the 16*CI input samples and one 16-byte store remain.
template <typename T, int CI>
__global__ void __launch_bounds__(256) conv_thin_in_kernel(const T* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                                           T* __restrict__ y, int N, int H, int W, int Co) {
  constexpr int V = VecN<T>::N;
  constexpr int TAPS = 16 * CI;
  extern __shared__ __align__(16) float wsm[];  // [TAPS][Co]
  for (int i = threadIdx.x; i < TAPS * Co; i += blockDim.x) {
    const int co = i % Co, t = i / Co;       // t = (kh*4+kw)*CI + ci
    const int ci = t % CI, k = t / CI;
    wsm[i] = w[((long long)co * CI + ci) * 16 + k];
  }
  __syncthreads();
  const int Ho = H >> 1, Wo = W >> 1, CV = Co / V;
  const int cv = threadIdx.x % CV, plane = threadIdx.x / CV, planes = blockDim.x / CV;
  float wreg[CI == 1 ? TAPS : 1][V];
  float bv[V];
#pragma unroll
  for (int j = 0; j < V; j++) bv[j] = bias ? bias[cv * V + j] : 0.f;
  if (CI == 1) {
#pragma unroll
    for (int t = 0; t < TAPS; t++)
#pragma unroll
      for (int j = 0; j < V; j++) wreg[CI == 1 ? t : 0][j] = wsm[t * Co + cv * V + j];
  }
  const long long npix = (long long)N * Ho * Wo;
  for (long long p = (long long)blockIdx.x * planes + plane; p < npix; p += (long long)gridDim.x * planes) {
    const int ox = (int)(p % Wo);
    const long long t2 = p / Wo;
    const int oy = (int)(t2 % Ho);
    const int n = (int)(t2 / Ho);
    float acc[V];
#pragma unroll
    for (int j = 0; j < V; j++) acc[j] = bv[j];
#pragma unroll
    for (int kh = 0; kh < 4; kh++) {
      const int iy = 2 * oy - 1 + kh;
#pragma unroll
      for (int kw = 0; kw < 4; kw++) {
        const int ix = 2 * ox - 1 + kw;
        const bool ok = (iy >= 0) && (iy < H) && (ix >= 0) && (ix < W);
        const T* xp = x + (((long long)n * H + (ok ? iy : 0)) * W + (ok ? ix : 0)) * CI;
#pragma unroll
        for (int ci = 0; ci < CI; ci++) {
          const float xv = ok ? ld_f<T>(xp + ci) : 0.f;
          const int t = (kh * 4 + kw) * CI + ci;
          if (CI == 1) {
#pragma unroll
            for (int j = 0; j < V; j++) acc[j] = fmaf(xv, wreg[CI == 1 ? t : 0][j], acc[j]);
          } else {
            const float* wr = wsm + t * Co + cv * V;
#pragma unroll
            for (int j = 0; j < V; j += 4) {
              const float4 w4 = *reinterpret_cast<const float4*>(wr + j);
              acc[j] = fmaf(xv, w4.x, acc[j]); acc[j + 1] = fmaf(xv, w4.y, acc[j + 1]);
              acc[j + 2] = fmaf(xv, w4.z, acc[j + 2]); acc[j + 3] = fmaf(xv, w4.w, acc[j + 3]);
            }
          }
        }
      }
    }
    st_raw16(y + p * Co + cv * V, pack16<T>(acc));
  }
}

// one thread per output pixel; CO (1 or 3) output channels held in registers; Ci % 8 == 0; weights read as float4 from smem
template <typename T, typename TO, int CO>
__global__ void __launch_bounds__(256) convT_thin_out_kernel(const T* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                                             const float* __restrict__ addend, const int* __restrict__ grp_src,
                                                             int imgs_per_group, TO* __restrict__ y, int N, int H, int W, int Ci) {
  constexpr int V = VecN<T>::N;
  extern __shared__ __align__(16) float wsm[];  // [16][CO][Ci]
  for (int i = threadIdx.x; i < 16 * CO * Ci; i += blockDim.x) {
    const int ci = i % Ci, r = i / Ci;
    const int co = r % CO, k = r / CO;
    wsm[i] = w[((long long)ci * CO + co) * 16 + k];
  }
  __syncthreads();
  const int Ho = 2 * H, Wo = 2 * W;
  const long long total = (long long)N * Ho * Wo;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (long long)gridDim.x * blockDim.x) {
    const int ox = (int)(p % Wo);
    const long long t2 = p / Wo;
    const int oy = (int)(t2 % Ho);
    const int n = (int)(t2 / Ho);
    float acc[CO];
#pragma unroll
    for (int co = 0; co < CO; co++) acc[co] = bias ? bias[co] : 0.f;
    if (addend) {
      const int n2 = grp_src[n / imgs_per_group] * imgs_per_group + (n % imgs_per_group);
      const float* ar = addend + (((long long)n2 * Ho + oy) * Wo + ox) * CO;
#pragma unroll
      for (int co = 0; co < CO; co++) acc[co] += ar[co];
    }
    const int kh0 = (oy + 1) & 1, kw0 = (ox + 1) & 1;
#pragma unroll
    for (int a = 0; a < 2; a++) {
      const int kh = kh0 + 2 * a, ty = oy + 1 - kh, iy = ty >> 1;
      if (ty < 0 || iy >= H) continue;
#pragma unroll
      for (int b = 0; b < 2; b++) {
        const int kw = kw0 + 2 * b, tx = ox + 1 - kw, ix = tx >> 1;
        if (tx < 0 || ix >= W) continue;
        const T* xp = x + (((long long)n * H + iy) * W + ix) * Ci;
        const float* wr = wsm + (kh * 4 + kw) * CO * Ci;
        for (int c0 = 0; c0 < Ci; c0 += V) {
          float xv[V];
          unpack16<T>(ld_raw16(xp + c0), xv);
#pragma unroll
          for (int co = 0; co < CO; co++) {
            const float* wc = wr + co * Ci + c0;
            float s0 = 0.f, s1 = 0.f;
#pragma unroll
            for (int j = 0; j < V; j += 4) {
              const float4 w4 = *reinterpret_cast<const float4*>(wc + j);
              s0 = fmaf(xv[j], w4.x, s0); s1 = fmaf(xv[j + 1], w4.y, s1);
              s0 = fmaf(xv[j + 2], w4.z, s0); s1 = fmaf(xv[j + 3], w4.w, s1);
            }
            acc[co] += s0 + s1;
          }
        }
      }
    }
#pragma unroll
    for (int co = 0; co < CO; co++) st_f<TO>(y + p * CO + co, acc[co]);
  }
}

inline int grid_for(long long total, int block) {
  long long g = (total + block - 1) / block;
  const long long cap = 132LL * 16;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace

int p2pvg_conv_thin_in_impl(const void* x, int dtype, const float* w, const float* bias, void* y, int N, int H, int W, int Ci, int Co,
                            cudaStream_t st) {
  const int vec = dtype == P2PVG_BF16 ? 8 : 4;
  P2PVG_REQUIRE((Ci == 1 || Ci == 3) && Co % vec == 0 && 256 % (Co / vec) == 0 && (H % 2 == 0) && (W % 2 == 0), P2PVG_ERR_UNSUPPORTED,
                "conv_thin_in: unsupported shape Ci=%d Co=%d %dx%d", Ci, Co, H, W);
  P2PVG_REQUIRE((reinterpret_cast<uintptr_t>(y) & 15) == 0, P2PVG_ERR_BAD_ARG, "conv_thin_in: output not 16-byte aligned");
  if (N == 0) return P2PVG_OK;
  const size_t smem = (size_t)16 * Ci * Co * sizeof(float);
  const long long npix = (long long)N * (H / 2) * (W / 2);
  const int planes = 256 / (Co / vec);
  long long blocks = (npix + planes - 1) / planes;
  if (blocks > 132 * 16) blocks = 132 * 16;
  if (Ci == 1) {
    DISPATCH_DTYPE(dtype, T, (conv_thin_in_kernel<T, 1><<<(int)blocks, 256, smem, st>>>((const T*)x, w, bias, (T*)y, N, H, W, Co)));
  } else {
    DISPATCH_DTYPE(dtype, T, (conv_thin_in_kernel<T, 3><<<(int)blocks, 256, smem, st>>>((const T*)x, w, bias, (T*)y, N, H, W, Co)));
  }
  return p2pvg_check_launch("conv_thin_in");
}

int p2pvg_convT_thin_out_impl(const void* x, int dtype, const float* w, const float* bias, const float* addend, const int* grp_src,
                              int imgs_per_group, void* y, int y_dtype, int N, int H, int W, int Ci, int Co, cudaStream_t st) {
  const int vec = dtype == P2PVG_BF16 ? 8 : 4;
  P2PVG_REQUIRE((Co == 1 || Co == 3) && Ci % vec == 0, P2PVG_ERR_UNSUPPORTED, "convT_thin_out: unsupported shape Ci=%d Co=%d", Ci, Co);
  P2PVG_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0, P2PVG_ERR_BAD_ARG, "convT_thin_out: input not 16-byte aligned");
  P2PVG_REQUIRE(addend == nullptr || (grp_src != nullptr && imgs_per_group > 0), P2PVG_ERR_BAD_ARG, "convT_thin_out: addend needs grp_src");
  P2PVG_REQUIRE(y_dtype == dtype || y_dtype == P2PVG_F32, P2PVG_ERR_BAD_ARG, "convT_thin_out: output dtype must be the input dtype or fp32");
  if (N == 0) return P2PVG_OK;
  const size_t smem = (size_t)16 * Co * Ci * sizeof(float);
  P2PVG_REQUIRE(smem <= 48 * 1024, P2PVG_ERR_UNSUPPORTED, "convT_thin_out: Ci too large");
  const long long total = (long long)N * 4 * H * W;
  const int grid = grid_for(total, 256);
#define LAUNCH(TI, TO, CO_) \
  convT_thin_out_kernel<TI, TO, CO_><<<grid, 256, smem, st>>>((const TI*)x, w, bias, addend, grp_src, imgs_per_group, (TO*)y, N, H, W, Ci)
  if (Co == 1) {
    if (dtype == P2PVG_BF16 && y_dtype == P2PVG_BF16) LAUNCH(bf16, bf16, 1);
    else if (dtype == P2PVG_BF16) LAUNCH(bf16, float, 1);
    else LAUNCH(float, float, 1);
  } else {
    if (dtype == P2PVG_BF16 && y_dtype == P2PVG_BF16) LAUNCH(bf16, bf16, 3);
    else if (dtype == P2PVG_BF16) LAUNCH(bf16, float, 3);
    else LAUNCH(float, float, 3);
  }
#undef LAUNCH
  return p2pvg_check_launch("convT_thin_out");
}
