// Fused sigmoid + MSE (forward value and gradient w.r.t. the pre-sigmoid decoder output in one
// pass), the loss finaliser that produces the four host-visible scalars of P2PModel.forward
// (models/p2p_model.py:271), and the flat-arena Adam update with PyTorch-1.0 arithmetic.
#include "common.cuh"

#define MSE_CHUNKS 32

namespace {

template <typename T>
__global__ void __launch_bounds__(256) sigmoid_mse_kernel(const T* __restrict__ raw, const float* __restrict__ x,
                                                          const int* __restrict__ tgt, const float* __restrict__ coef,
                                                          long long E, T* __restrict__ pred, T* __restrict__ d_raw,
                                                          float* __restrict__ partial) {
  const int g = blockIdx.y;
  const float* xt = x + (long long)tgt[g] * E;
  const T* rg = raw + (long long)g * E;
  const float cf = coef[g];
  double acc = 0.0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < E; i += (long long)gridDim.x * blockDim.x) {
    float s = sigmoidf_(ld_f<T>(rg + i));
    float d = s - xt[i];
    acc += (double)d * (double)d;
    if (pred) st_f<T>(pred + (long long)g * E + i, s);
    if (d_raw) st_f<T>(d_raw + (long long)g * E + i, cf * 2.f * d * s * (1.f - s));
  }
  __shared__ double sh[8];
  acc = warp_sum_d(acc);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double v = 0.0;
    for (int w = 0; w < 8; w++) v += sh[w];
    partial[(long long)g * gridDim.x + blockIdx.x] = (float)v;
  }
}

// K5 of SURVEY.md §2.2: the last decoder layer -- ConvTranspose2d(2*64 -> 1, 4, 2, 1) + Sigmoid (models/dcgan_64.py:75-79) --
// fused with the reconstruction / CPC loss (nn.MSELoss, models/p2p_model.py:254,256).  The 16-tap products of every input
// pixel come from the tensor-core GEMMs (col [N*Hi*Wi, 16] for the decoder path, col2 for the shared skip path); this kernel
// gathers the four taps of an output pixel from both, adds the bias, applies the sigmoid, accumulates the squared error
// against the target frame and writes d(loss)/d(raw) -- one pass, no raw-output tensor, 32-bit index arithmetic.
template <typename T, int C>
__global__ void __launch_bounds__(256) convt_c1_loss_kernel(const T* __restrict__ col, const T* __restrict__ col2, const int* __restrict__ grp_src,
                                                            const float* __restrict__ bias, const float* __restrict__ x,
                                                            const int* __restrict__ tgt, const float* __restrict__ coef, int B, int Hi,
                                                            int Wi, T* __restrict__ d_raw, float* __restrict__ partial) {
  const int g = blockIdx.y;
  const unsigned Ho = 2u * Hi, Wo = 2u * Wi;
  const unsigned P = (unsigned)B * Ho * Wo;   // output pixels of the group; E = P * C elements
  const float* xt = x + (long long)tgt[g] * P * C;
  const T* cg = col + (long long)g * B * Hi * Wi * 16 * C;
  const T* sg = col2 + (long long)grp_src[g] * B * Hi * Wi * 16 * C;
  T* dg = d_raw + (long long)g * P * C;
  const float cf = coef[g];
  float b0[C];
#pragma unroll
  for (int c = 0; c < C; c++) b0[c] = bias ? bias[c] : 0.f;
  double acc = 0.0;
  for (unsigned e = blockIdx.x * blockDim.x + threadIdx.x; e < P; e += gridDim.x * blockDim.x) {
    const unsigned ox = e % Wo, r = e / Wo, oy = r % Ho, b = r / Ho;
    const int kh0 = (oy + 1) & 1, kw0 = (ox + 1) & 1;
    float v[C];
#pragma unroll
    for (int c = 0; c < C; c++) v[c] = b0[c];
#pragma unroll
    for (int a = 0; a < 2; a++) {
#pragma unroll
      for (int q = 0; q < 2; q++) {
        const int kh = kh0 + 2 * a, kw = kw0 + 2 * q;
        const int ty = (int)oy + 1 - kh, tx = (int)ox + 1 - kw;
        const int iy = ty >> 1, ix = tx >> 1;
        if (ty < 0 || iy >= Hi || tx < 0 || ix >= Wi) continue;
        const unsigned off = ((((b * Hi + iy) * Wi + ix) << 4) + kh * 4 + kw) * C;
#pragma unroll
        for (int c = 0; c < C; c++) v[c] += ld_f<T>(cg + off + c) + ld_f<T>(sg + off + c);
      }
    }
#pragma unroll
    for (int c = 0; c < C; c++) {
      const float s = sigmoidf_(v[c]);
      const float d = s - xt[e * C + c];
      acc += (double)d * (double)d;
      st_f<T>(dg + e * C + c, cf * 2.f * d * s * (1.f - s));
    }
  }
  __shared__ double sh[8];
  acc = warp_sum_d(acc);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double v = 0.0;
    for (int w = 0; w < 8; w++) v += sh[w];
    partial[(long long)g * gridDim.x + blockIdx.x] = (float)v;
  }
}

__global__ void finalize_losses_kernel(const float* __restrict__ mse_partial, int n_recon, int has_cpc, int nchunk, double E,
                                       const float* __restrict__ kl_sum, float batch_size, const float* __restrict__ align_partial,
                                       int n_align, float seq_len, float* __restrict__ out) {
  // one warp: lane k sums chunk column k of every group (independent loads in flight instead of one thread's dependent chain of
  // n_recon * nchunk), fp64, combined by a fixed shuffle tree (deterministic)
  const int lane = threadIdx.x;
  if (blockIdx.x != 0 || lane >= 32) return;
  double mse = 0.0, cpc = 0.0, al = 0.0;
  for (int k = lane; k < nchunk; k += 32) {
    for (int g = 0; g < n_recon; g++) mse += (double)mse_partial[g * nchunk + k];
    if (has_cpc) cpc += (double)mse_partial[n_recon * nchunk + k];
  }
  for (int s = lane; s < n_align; s += 32) al += (double)align_partial[s];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mse += __shfl_xor_sync(0xffffffffu, mse, o);
    cpc += __shfl_xor_sync(0xffffffffu, cpc, o);
    al += __shfl_xor_sync(0xffffffffu, al, o);
  }
  if (lane == 0) {
    out[0] = (float)(mse / E / seq_len);
    out[1] = (float)((double)kl_sum[0] / batch_size / seq_len);
    out[2] = (float)(cpc / E / seq_len);
    out[3] = (float)(al / seq_len);
  }
}

// n scalars + a sequence number to page-locked host memory (zero-copy store): the host polls the sequence number, so the
// values reach it while the rest of the stream (backward passes, optimiser) is still running
__global__ void publish_scalars_kernel(const float* __restrict__ src, int n, float* host, const int* __restrict__ seq) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  for (int i = 0; i < n; i++) reinterpret_cast<volatile float*>(host)[i] = src[i];
  __threadfence_system();
  reinterpret_cast<volatile int*>(host)[n] = seq[0];
}

// torch-1.0 Adam: denom = sqrt(v) + eps; p -= lr*sqrt(bc2)/bc1 * m/denom
__global__ void adam_legacy_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                                   long long n, double beta1_d, double beta2_d, double eps_d, double lr,
                                   const int* __restrict__ step_ptr) {
  __shared__ float s_step_size;
  if (threadIdx.x == 0) {
    // step counter lives in device memory so that a captured CUDA graph sees the live value
    const double t = (double)step_ptr[0];
    const double bc1 = 1.0 - pow(beta1_d, t), bc2 = 1.0 - pow(beta2_d, t);
    s_step_size = (float)(lr * sqrt(bc2) / bc1);
  }
  __syncthreads();
  const float step_size = s_step_size;
  // scalars are rounded to fp32 exactly as torch rounds python doubles applied to fp32 tensors
  const float beta1 = (float)beta1_d, beta2 = (float)beta2_d, eps = (float)eps_d;
  const float omb1 = (float)(1.0 - beta1_d), omb2 = (float)(1.0 - beta2_d);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float gi = g[i];
    float mi = m[i] * beta1 + omb1 * gi;
    float vi = v[i] * beta2 + omb2 * gi * gi;
    m[i] = mi;
    v[i] = vi;
    p[i] = p[i] - step_size * (mi / (sqrtf(vi) + eps));
  }
}

__global__ void scale_kernel(float* __restrict__ x, long long n, float a) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) x[i] *= a;
}

}  // namespace

extern "C" int p2pvg_mse_chunks(void) { return MSE_CHUNKS; }

extern "C" int p2pvg_sigmoid_mse(const void* raw, int dtype, const float* x, const int* tgt, const float* coef, int G, int64_t E,
                                 void* pred, void* d_raw, float* partial, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (G == 0 || E == 0) return P2PVG_OK;
  dim3 grid(MSE_CHUNKS, G);
  DISPATCH_DTYPE(dtype, T, (sigmoid_mse_kernel<T><<<grid, 256, 0, st>>>((const T*)raw, x, tgt, coef, E, (T*)pred, (T*)d_raw, partial)));
  return p2pvg_check_launch("sigmoid_mse");
}

extern "C" int p2pvg_convt_c1_loss(const void* col, const void* col2, int dtype, const int* grp_src, const float* bias, const float* x,
                                   const int* tgt, const float* coef, int G, int B, int Hi, int Wi, int C, void* d_raw, float* partial,
                                   void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  P2PVG_REQUIRE(col && col2 && grp_src && x && tgt && coef && d_raw && partial, P2PVG_ERR_BAD_ARG, "convt_c1_loss: null argument");
  if (G == 0 || B == 0) return P2PVG_OK;
  P2PVG_REQUIRE(C == 1 || C == 3, P2PVG_ERR_UNSUPPORTED, "convt_c1_loss: 1 or 3 output channels (got %d)", C);
  P2PVG_REQUIRE((long long)B * Hi * Wi * 16 * C < (1LL << 31), P2PVG_ERR_UNSUPPORTED, "convt_c1_loss: group too large for 32-bit indexing");
  dim3 grid(MSE_CHUNKS, G);
  if (C == 1) {
    DISPATCH_DTYPE(dtype, T, (convt_c1_loss_kernel<T, 1><<<grid, 256, 0, st>>>((const T*)col, (const T*)col2, grp_src, bias, x, tgt, coef, B, Hi, Wi,
                                                                               (T*)d_raw, partial)));
  } else {
    DISPATCH_DTYPE(dtype, T, (convt_c1_loss_kernel<T, 3><<<grid, 256, 0, st>>>((const T*)col, (const T*)col2, grp_src, bias, x, tgt, coef, B, Hi, Wi,
                                                                               (T*)d_raw, partial)));
  }
  return p2pvg_check_launch("convt_c1_loss");
}

extern "C" int p2pvg_finalize_losses(const float* mse_partial, int n_recon, int has_cpc, double E, const float* kl_sum, float batch_size,
                                     const float* align_partial, int n_align, float seq_len, float* out, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  finalize_losses_kernel<<<1, 32, 0, st>>>(mse_partial, n_recon, has_cpc, MSE_CHUNKS, E, kl_sum, batch_size, align_partial, n_align,
                                           seq_len, out);
  return p2pvg_check_launch("finalize_losses");
}

extern "C" int p2pvg_publish_scalars(const float* src, int n, float* host_mapped, const int* seq, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n <= 0 || n > 64 || !src || !host_mapped || !seq) {
    p2pvg_set_error("publish_scalars: bad arguments");
    return P2PVG_ERR_BAD_ARG;
  }
  publish_scalars_kernel<<<1, 32, 0, st>>>(src, n, host_mapped, seq);
  return p2pvg_check_launch("publish_scalars");
}

extern "C" int p2pvg_adam_legacy(float* p, const float* g, float* m, float* v, int64_t n, double lr, double beta1, double beta2, double eps,
                                 const int* step_ptr, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) return P2PVG_OK;
  P2PVG_REQUIRE(step_ptr != nullptr, P2PVG_ERR_BAD_ARG, "adam: step counter pointer is null");
  long long blocks = (n + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  adam_legacy_kernel<<<(int)blocks, 256, 0, st>>>(p, g, m, v, n, beta1, beta2, eps, lr, step_ptr);
  return p2pvg_check_launch("adam_legacy");
}

extern "C" int p2pvg_scale(float* x, int64_t n, float a, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) return P2PVG_OK;
  long long blocks = (n + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  scale_kernel<<<(int)blocks, 256, 0, st>>>(x, n, a);
  return p2pvg_check_launch("scale");
}
