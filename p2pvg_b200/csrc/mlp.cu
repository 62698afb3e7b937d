// Row-wise kernels of the h36m pose backbone (reference models/h36m_mlp.py): LayerNorm forward / backward over the
// feature axis and the plain (no sigmoid) mean-squared-error with its gradient.  fp32, one warp per row.
#include "common.cuh"

namespace {

// y = (x - mean) * rstd * gamma + beta per row; C <= 1024
__global__ void layernorm_fwd_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                                     float* __restrict__ y, float* __restrict__ mean, float* __restrict__ rstd, long long rows, int C,
                                     float eps) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* xr = x + row * C;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += xr[c];
  s = warp_sum(s);
  const float m = s / (float)C;
  float v = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float d = xr[c] - m;
    v = fmaf(d, d, v);
  }
  v = warp_sum(v);
  const float r = rsqrtf(v / (float)C + eps);
  if (lane == 0) {
    mean[row] = m;
    rstd[row] = r;
  }
  float* yr = y + row * C;
  for (int c = lane; c < C; c += 32) yr[c] = (xr[c] - m) * r * gamma[c] + beta[c];
}

// dx = rstd * (g - mean_c(g) - xhat * mean_c(g * xhat)),  g = dy * gamma
__global__ void layernorm_bwd_dx_kernel(const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ mean,
                                        const float* __restrict__ rstd, const float* __restrict__ gamma, float* __restrict__ dx,
                                        long long rows, int C) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float m = mean[row], r = rstd[row];
  const float* xr = x + row * C;
  const float* dr = dy + row * C;
  float s0 = 0.f, s1 = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float g = dr[c] * gamma[c], xh = (xr[c] - m) * r;
    s0 += g;
    s1 = fmaf(g, xh, s1);
  }
  s0 = warp_sum(s0) / (float)C;
  s1 = warp_sum(s1) / (float)C;
  float* o = dx + row * C;
  for (int c = lane; c < C; c += 32) {
    const float g = dr[c] * gamma[c], xh = (xr[c] - m) * r;
    o[c] = r * (g - s0 - xh * s1);
  }
}

// partial[chunk][0][c] = sum_rows dy*xhat, partial[chunk][1][c] = sum_rows dy   (two-stage, deterministic)
__global__ void layernorm_bwd_param_kernel(const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ mean,
                                           const float* __restrict__ rstd, long long rows, int C, long long rows_per_chunk,
                                           float* __restrict__ partial) {
  const int c = blockIdx.x * 32 + (threadIdx.x & 31);
  const int lane = threadIdx.x >> 5;
  const long long r0 = (long long)blockIdx.y * rows_per_chunk;
  long long r1 = r0 + rows_per_chunk;
  if (r1 > rows) r1 = rows;
  float a = 0.f, b = 0.f;
  if (c < C)
    for (long long r = r0 + lane; r < r1; r += 8) {
      const float d = dy[r * C + c];
      a = fmaf(d, (x[r * C + c] - mean[r]) * rstd[r], a);
      b += d;
    }
  __shared__ float sa[8][33], sb[8][33];
  sa[lane][threadIdx.x & 31] = a;
  sb[lane][threadIdx.x & 31] = b;
  __syncthreads();
  if (lane == 0 && c < C) {
    float va = 0.f, vb = 0.f;
#pragma unroll
    for (int l = 0; l < 8; l++) {
      va += sa[l][threadIdx.x & 31];
      vb += sb[l][threadIdx.x & 31];
    }
    partial[((long long)blockIdx.y * 2 + 0) * C + c] = va;
    partial[((long long)blockIdx.y * 2 + 1) * C + c] = vb;
  }
}
__global__ void layernorm_bwd_finish_kernel(const float* __restrict__ partial, int nchunk, int C, float* __restrict__ dgamma,
                                            float* __restrict__ dbeta) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float a = 0.f, b = 0.f;
  for (int k = 0; k < nchunk; k++) {
    a += partial[((long long)k * 2 + 0) * C + c];
    b += partial[((long long)k * 2 + 1) * C + c];
  }
  dgamma[c] = a;
  dbeta[c] = b;
}

// per-group sum of squared error partials and d(loss)/d(pred) = coef[g]*2*(pred-x)
__global__ void __launch_bounds__(256) mse_plain_kernel(const float* __restrict__ pred, const float* __restrict__ x, const int* __restrict__ tgt,
                                                        const float* __restrict__ coef, long long E, float* __restrict__ d_pred,
                                                        float* __restrict__ partial) {
  const int g = blockIdx.y;
  const float* xt = x + (long long)tgt[g] * E;
  const float* pg = pred + (long long)g * E;
  const float cf = coef[g];
  double acc = 0.0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < E; i += (long long)gridDim.x * blockDim.x) {
    const float d = pg[i] - xt[i];
    acc += (double)d * (double)d;
    if (d_pred) d_pred[(long long)g * E + i] = cf * 2.f * d;
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

}  // namespace

extern "C" int p2pvg_layernorm_fwd(const float* x, const float* gamma, const float* beta, float* y, float* mean, float* rstd, int64_t rows,
                                   int C, float eps, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (rows == 0) return P2PVG_OK;
  layernorm_fwd_kernel<<<cdiv(rows, 8), 256, 0, st>>>(x, gamma, beta, y, mean, rstd, rows, C, eps);
  return p2pvg_check_launch("layernorm_fwd");
}

extern "C" int p2pvg_layernorm_bwd(const float* dy, const float* x, const float* mean, const float* rstd, const float* gamma, float* dx,
                                   float* dgamma, float* dbeta, int64_t rows, int C, void* ws, size_t ws_bytes, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (rows == 0) return P2PVG_OK;
  if (dgamma) {  // parameter gradients first: dx may alias dy
    long long nchunk = (rows + 255) / 256;
    if (nchunk > 256) nchunk = 256;
    if (nchunk < 1) nchunk = 1;
    const long long rpc = (rows + nchunk - 1) / nchunk;
    nchunk = (rows + rpc - 1) / rpc;
    P2PVG_REQUIRE(ws != nullptr && ws_bytes >= (size_t)nchunk * 2 * C * sizeof(float), P2PVG_ERR_WORKSPACE, "layernorm_bwd: workspace too small");
    dim3 grid(cdiv(C, 32), (unsigned)nchunk);
    layernorm_bwd_param_kernel<<<grid, 256, 0, st>>>(dy, x, mean, rstd, rows, C, rpc, (float*)ws);
    layernorm_bwd_finish_kernel<<<cdiv(C, 128), 128, 0, st>>>((const float*)ws, (int)nchunk, C, dgamma, dbeta);
  }
  layernorm_bwd_dx_kernel<<<cdiv(rows, 8), 256, 0, st>>>(dy, x, mean, rstd, gamma, dx, rows, C);
  return p2pvg_check_launch("layernorm_bwd");
}

extern "C" int p2pvg_mse_plain(const float* pred, const float* x, const int* tgt, const float* coef, int G, int64_t E, float* d_pred,
                               float* partial, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (G == 0 || E == 0) return P2PVG_OK;
  dim3 grid(p2pvg_mse_chunks(), G);
  mse_plain_kernel<<<grid, 256, 0, st>>>(pred, x, tgt, coef, E, d_pred, partial);
  return p2pvg_check_launch("mse_plain");
}
