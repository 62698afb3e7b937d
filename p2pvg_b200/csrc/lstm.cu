// fp32 kernels of the recurrent phase: LSTM cell pointwise math (forward / backward), the
// reparameterisation + KL block, input assembly (latent | global descriptor | time counters), latent
// gradient gathering, the alignment loss with the reference's row-0 broadcast quirk
// (models/p2p_model.py:224-225), column sums for bias gradients and the tanh head.
#include "common.cuh"

namespace {

__global__ void lstm_pointwise_fwd_kernel(float* __restrict__ gates, const float* __restrict__ c_prev, float* __restrict__ c_out,
                                          float* __restrict__ h_out, int B, int R) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * R) return;
  int b = idx / R, j = idx - b * R;
  float* g = gates + (long long)b * 4 * R;
  float i = sigmoidf_(g[j]), f = sigmoidf_(g[R + j]), gg = tanhf(g[2 * R + j]), o = sigmoidf_(g[3 * R + j]);
  float c = f * c_prev[idx] + i * gg;
  g[j] = i; g[R + j] = f; g[2 * R + j] = gg; g[3 * R + j] = o;
  c_out[idx] = c;
  h_out[idx] = o * tanhf(c);
}

__global__ void lstm_pointwise_bwd_kernel(const float* __restrict__ dh, const float* __restrict__ dc_next,
                                          const float* __restrict__ gates, const float* __restrict__ c_prev,
                                          const float* __restrict__ c, float* __restrict__ dgates, float* __restrict__ dc_prev,
                                          int B, int R) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * R) return;
  int b = idx / R, j = idx - b * R;
  const float* g = gates + (long long)b * 4 * R;
  float* dg = dgates + (long long)b * 4 * R;
  float i = g[j], f = g[R + j], gg = g[2 * R + j], o = g[3 * R + j];
  float tc = tanhf(c[idx]);
  float dhv = dh[idx];
  float dc = dhv * o * (1.f - tc * tc) + (dc_next ? dc_next[idx] : 0.f);
  dg[j] = dc * gg * i * (1.f - i);
  dg[R + j] = dc * c_prev[idx] * f * (1.f - f);
  dg[2 * R + j] = dc * i * (1.f - gg * gg);
  dg[3 * R + j] = dhv * tc * o * (1.f - o);
  dc_prev[idx] = dc * f;
}

// z = eps*exp(lv/2)+mu for posterior and prior; KL(N(mu,lv)||N(mu_p,lv_p)) summed (misc/criterion.py:12-15).
// One thread-block cluster of 8 CTAs: the kernel sits on the critical path between the Gaussian heads and the frame predictor, and a
// single CTA needs n/1024 dependent trips; the 8 per-CTA partial sums are combined by CTA 0 through distributed shared memory in
// rank order (deterministic, no workspace, no atomics).
constexpr int RKL_CTAS = 8;
__global__ void __cluster_dims__(RKL_CTAS, 1, 1) __launch_bounds__(1024)
reparam_kl_fwd_kernel(const float* __restrict__ mu, const float* __restrict__ lv, const float* __restrict__ mu_p,
                      const float* __restrict__ lv_p, const float* __restrict__ eps, const float* __restrict__ eps_p,
                      float* __restrict__ z, float* __restrict__ z_p, int n, float* __restrict__ kl_sum) {
  double acc = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float m1 = mu[i], l1 = lv[i], m2 = mu_p[i], l2 = lv_p[i];
    float s1 = expf(0.5f * l1), s2 = expf(0.5f * l2);
    z[i] = eps[i] * s1 + m1;
    z_p[i] = eps_p[i] * s2 + m2;
    float d = m1 - m2;
    float k = logf(s2 / s1) + (expf(l1) + d * d) / (2.f * expf(l2)) - 0.5f;
    acc += (double)k;
  }
  __shared__ double sh[32];
  __shared__ double cta_sum;
  acc = warp_sum_d(acc);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    double v = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0.0;
    v = warp_sum_d(v);
    if (threadIdx.x == 0) cta_sum = v;
  }
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
  uint32_t rank;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
  if (rank == 0 && threadIdx.x == 0) {
    double v = 0.0;
    const uint32_t local = (uint32_t)__cvta_generic_to_shared(&cta_sum);
    for (uint32_t r = 0; r < RKL_CTAS; r++) {
      uint32_t remote;
      asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local), "r"(r));
      double t;
      asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(t) : "r"(remote) : "memory");
      v += t;
    }
    kl_sum[0] = (float)v;
  }
  // nobody may exit while CTA 0 still reads its shared memory
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

__global__ void reparam_kl_bwd_kernel(const float* __restrict__ mu, const float* __restrict__ lv, const float* __restrict__ mu_p,
                                      const float* __restrict__ lv_p, const float* __restrict__ eps, const float* __restrict__ eps_p,
                                      const float* __restrict__ dz, const float* __restrict__ dz_p, float kl_coef,
                                      float* __restrict__ dmu, float* __restrict__ dlv, float* __restrict__ dmu_p,
                                      float* __restrict__ dlv_p, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float m1 = mu[i], l1 = lv[i], m2 = mu_p[i], l2 = lv_p[i];
  float e1 = expf(l1), e2 = expf(l2), d = m1 - m2;
  float gm1 = kl_coef * d / e2;
  float gl1 = kl_coef * (-0.5f + e1 / (2.f * e2));
  float gm2 = -gm1;
  float gl2 = kl_coef * (0.5f - (e1 + d * d) / (2.f * e2));
  if (dz) {
    float v = dz[i];
    gm1 += v;
    gl1 += v * eps[i] * 0.5f * expf(0.5f * l1);
  }
  if (dz_p) {
    float v = dz_p[i];
    gm2 += v;
    gl2 += v * eps_p[i] * 0.5f * expf(0.5f * l2);
  }
  dmu[i] = gm1; dlv[i] = gl1; dmu_p[i] = gm2; dlv_p[i] = gl2;
}

// dst[s,b,:] = [ A[ia[s],b,0:ga] | Bm[ib[s],b,0:gb] | tuc[s] | dt[s] ]
__global__ void build_concat_kernel(float* __restrict__ dst, const float* __restrict__ A, const int* __restrict__ ia, int ga,
                                    const float* __restrict__ Bm, const int* __restrict__ ib, int gb, const float* __restrict__ tuc,
                                    const float* __restrict__ dt, int S, int B, int W) {
  // W >= ga+gb+2 is the row pitch; the padding columns are written as zeros
  long long total = (long long)S * B * W;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    int col = (int)(idx % W);
    long long sb = idx / W;
    int b = (int)(sb % B), s = (int)(sb / B);
    float v;
    if (col < ga) v = A[((long long)ia[s] * B + b) * ga + col];
    else if (col < ga + gb) v = Bm[((long long)ib[s] * B + b) * gb + (col - ga)];
    else if (col == ga + gb) v = tuc[s];
    else if (col == ga + gb + 1) v = dt[s];
    else v = 0.f;
    dst[idx] = v;
  }
}

// dst[t,b,j] (+)= sum_{s<S: idx[s]==t} src[s,b,col0+j]     (dst [T,B,g], src [S,B,W])
__global__ void gather_add_cols_kernel(float* __restrict__ dst, const float* __restrict__ src, const int* __restrict__ idx, int S,
                                       int T, int B, int g, int W, int col0, int init) {
  long long total = (long long)T * B * g;
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (long long)gridDim.x * blockDim.x) {
    int j = (int)(k % g);
    long long tb = k / g;
    int b = (int)(tb % B), t = (int)(tb / B);
    float acc = init ? 0.f : dst[k];
    for (int s = 0; s < S; s++)
      if (idx[s] == t) acc += src[((long long)s * B + b) * W + col0 + j];
    dst[k] = acc;
  }
}

// pairs s=0..P-1: loss_s = mean_{b,j} (H[in[s],0,j] - h_pred[s,b,j])^2
//   d_hpred[s,b,j] += coef*2*(h_pred - h0)/(B*g);   dH[in[s],0,j] += coef*2*sum_b (h0 - h_pred)/(B*g)
__global__ void __launch_bounds__(1024) align_kernel(const float* __restrict__ H, const int* __restrict__ in_idx, const float* __restrict__ h_pred, int P,
                             int B, int g, float coef, float* __restrict__ loss_partial, float* __restrict__ d_hpred,
                             float* __restrict__ dH) {
  // block = one pair s; thread = (column jl of a 128-column pass, row lane of 8): a lane walks rows lane, lane+8, ... so the
  // dependent read-modify-write chain per thread is B/8 long instead of B; the 8 lanes of a column are combined in a fixed
  // order (deterministic)
  constexpr int CW = 128, RL = 8;
  const int s = blockIdx.x;
  const int jl = threadIdx.x % CW, lane = threadIdx.x / CW;
  const float invn = 1.f / ((float)B * (float)g);
  __shared__ float dsh[RL][CW];
  __shared__ double sh[32];
  double lacc = 0.0;
  const long long hrow = ((long long)in_idx[s] * B + 0) * g;
  for (int j0 = 0; j0 < g; j0 += CW) {
    const int j = j0 + jl;
    float dsum = 0.f;
    if (j < g) {
      const float h0 = H[hrow + j];
      for (int b = lane; b < B; b += RL) {
        const long long o = ((long long)s * B + b) * g + j;
        const float diff = h0 - h_pred[o];
        lacc += (double)diff * (double)diff;
        dsum += diff;
        if (d_hpred) d_hpred[o] += -coef * 2.f * diff * invn;
      }
    }
    dsh[lane][jl] = dsum;
    __syncthreads();
    if (lane == 0 && j < g && dH) {
      float t = 0.f;
#pragma unroll
      for (int l = 0; l < RL; l++) t += dsh[l][jl];
      dH[hrow + j] += coef * 2.f * t * invn;
    }
    __syncthreads();
  }
  lacc = warp_sum_d(lacc);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = lacc;
  __syncthreads();
  if (threadIdx.x < 32) {
    double v = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0.0;
    v = warp_sum_d(v);
    if (threadIdx.x == 0) loss_partial[s] = (float)(v * (double)invn);
  }
}

// out[c] (+)= sum_r x[r, c]   — two deterministic stages: per-chunk partials, then a column-wise finish
template <typename T>
__global__ void colsum_partial_kernel(const T* __restrict__ x, long long rows, int cols, long long ld, long long rows_per_chunk,
                                      float* __restrict__ part) {
  const int c = blockIdx.x * 32 + (threadIdx.x & 31);
  const int lane = threadIdx.x >> 5;  // 8 row lanes
  const long long r0 = (long long)blockIdx.y * rows_per_chunk;
  long long r1 = r0 + rows_per_chunk;
  if (r1 > rows) r1 = rows;
  float acc = 0.f;
  if (c < cols)
    for (long long r = r0 + lane; r < r1; r += 8) acc += ld_f<T>(&x[r * ld + c]);
  __shared__ float sh[8][33];
  sh[lane][threadIdx.x & 31] = acc;
  __syncthreads();
  if (lane == 0 && c < cols) {
    float v = 0.f;
#pragma unroll
    for (int l = 0; l < 8; l++) v += sh[l][threadIdx.x & 31];
    part[(long long)blockIdx.y * cols + c] = v;
  }
}
__global__ void colsum_finish_kernel(const float* __restrict__ part, int nchunk, int cols, float* __restrict__ out, int accumulate) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  float v = 0.f;
  for (int k = 0; k < nchunk; k++) v += part[(long long)k * cols + c];
  out[c] = accumulate ? out[c] + v : v;
}

__global__ void act_fwd_kernel(float* __restrict__ x, long long n, int act) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float v = x[i];
    if (act == P2PVG_ACT_TANH) v = tanhf(v);
    else if (act == P2PVG_ACT_LRELU) v = v > 0.f ? v : 0.2f * v;
    else if (act == P2PVG_ACT_SIGMOID) v = sigmoidf_(v);
    else if (act == P2PVG_ACT_RELU) v = fmaxf(v, 0.f);
    x[i] = v;
  }
}
__global__ void act_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, float* __restrict__ dx, long long n, int act) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float yv = y[i], g = 1.f;
    if (act == P2PVG_ACT_TANH) g = 1.f - yv * yv;
    else if (act == P2PVG_ACT_LRELU) g = yv > 0.f ? 1.f : 0.2f;
    else if (act == P2PVG_ACT_SIGMOID) g = yv * (1.f - yv);
    else if (act == P2PVG_ACT_RELU) g = yv > 0.f ? 1.f : 0.f;
    dx[i] = dy[i] * g;
  }
}

inline int grid_for(long long total, int block) {
  long long g = (total + block - 1) / block;
  const long long cap = 132LL * 16;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace

extern "C" int p2pvg_lstm_pointwise_fwd(float* gates, const float* c_prev, float* c_out, float* h_out, int B, int R, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (B * R == 0) return P2PVG_OK;
  lstm_pointwise_fwd_kernel<<<cdiv((long long)B * R, 256), 256, 0, st>>>(gates, c_prev, c_out, h_out, B, R);
  return p2pvg_check_launch("lstm_pointwise_fwd");
}
extern "C" int p2pvg_lstm_pointwise_bwd(const float* dh, const float* dc_next, const float* gates, const float* c_prev, const float* c,
                                        float* dgates, float* dc_prev, int B, int R, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (B * R == 0) return P2PVG_OK;
  lstm_pointwise_bwd_kernel<<<cdiv((long long)B * R, 256), 256, 0, st>>>(dh, dc_next, gates, c_prev, c, dgates, dc_prev, B, R);
  return p2pvg_check_launch("lstm_pointwise_bwd");
}
extern "C" int p2pvg_reparam_kl_fwd(const float* mu, const float* lv, const float* mu_p, const float* lv_p, const float* eps,
                                    const float* eps_p, float* z, float* z_p, int n, float* kl_sum, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  reparam_kl_fwd_kernel<<<RKL_CTAS, 1024, 0, st>>>(mu, lv, mu_p, lv_p, eps, eps_p, z, z_p, n, kl_sum);
  return p2pvg_check_launch("reparam_kl_fwd");
}
extern "C" int p2pvg_reparam_kl_bwd(const float* mu, const float* lv, const float* mu_p, const float* lv_p, const float* eps,
                                    const float* eps_p, const float* dz, const float* dz_p, float kl_coef, float* dmu, float* dlv,
                                    float* dmu_p, float* dlv_p, int n, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) return P2PVG_OK;
  reparam_kl_bwd_kernel<<<cdiv(n, 256), 256, 0, st>>>(mu, lv, mu_p, lv_p, eps, eps_p, dz, dz_p, kl_coef, dmu, dlv, dmu_p, dlv_p, n);
  return p2pvg_check_launch("reparam_kl_bwd");
}
extern "C" int p2pvg_build_concat(float* dst, const float* A, const int* ia, int ga, const float* Bm, const int* ib, int gb,
                                  const float* tuc, const float* dt, int S, int B, int ld, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  P2PVG_REQUIRE(ld >= ga + gb + 2, P2PVG_ERR_BAD_ARG, "build_concat: row pitch %d < %d", ld, ga + gb + 2);
  long long total = (long long)S * B * ld;
  if (total == 0) return P2PVG_OK;
  build_concat_kernel<<<grid_for(total, 256), 256, 0, st>>>(dst, A, ia, ga, Bm, ib, gb, tuc, dt, S, B, ld);
  return p2pvg_check_launch("build_concat");
}
extern "C" int p2pvg_gather_add_cols(float* dst, const float* src, const int* idx, int S, int T, int B, int g, int W, int col0, int init,
                                     void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  long long total = (long long)T * B * g;
  if (total == 0) return P2PVG_OK;
  gather_add_cols_kernel<<<grid_for(total, 256), 256, 0, st>>>(dst, src, idx, S, T, B, g, W, col0, init);
  return p2pvg_check_launch("gather_add_cols");
}
extern "C" int p2pvg_align(const float* H, const int* in_idx, const float* h_pred, int P, int B, int g, float coef, float* loss_partial,
                           float* d_hpred, float* dH, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (P <= 0) return P2PVG_OK;
  align_kernel<<<P, 1024, 0, st>>>(H, in_idx, h_pred, P, B, g, coef, loss_partial, d_hpred, dH);
  return p2pvg_check_launch("align");
}
extern "C" int p2pvg_colsum(const void* x, int dtype, int64_t rows, int cols, int64_t ld, float* out, int accumulate, void* ws,
                            size_t ws_bytes, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (cols == 0) return P2PVG_OK;
  // very thin contiguous matrices (bias gradient of a 1/3-channel layer): fold 256 rows into one so that a warp reads 32
  // consecutive elements, then sum the 256*cols folded columns per original column
  constexpr int FOLD = 256;
  if (cols <= 4 && ld == cols && rows >= 64 * FOLD && rows % FOLD == 0 && ws != nullptr &&
      ws_bytes >= (size_t)(1025 * FOLD * cols) * sizeof(float)) {
    float* tmp = reinterpret_cast<float*>(ws) + (size_t)1024 * FOLD * cols;
    int rc = p2pvg_colsum(x, dtype, rows / FOLD, FOLD * cols, (long long)FOLD * cols, tmp, 0, ws, (size_t)1024 * FOLD * cols * sizeof(float), st);
    if (rc) return rc;
    return p2pvg_colsum(tmp, P2PVG_F32, FOLD, cols, cols, out, accumulate, ws, (size_t)1024 * FOLD * cols * sizeof(float), st);
  }
  // enough chunks to fill the machine (132 SMs x a few blocks), at least 64 rows per chunk
  long long want = (132LL * 8) / cdiv(cols, 32) + 1;
  long long maxc = (rows + 63) / 64;
  long long nchunk = want < maxc ? want : maxc;
  if (nchunk < 1) nchunk = 1;
  if (nchunk > 1024) nchunk = 1024;
  P2PVG_REQUIRE(ws != nullptr && ws_bytes >= (size_t)nchunk * cols * sizeof(float), P2PVG_ERR_WORKSPACE, "colsum: workspace too small");
  long long rpc = (rows + nchunk - 1) / nchunk;
  if (rpc < 1) rpc = 1;
  nchunk = rows > 0 ? (rows + rpc - 1) / rpc : 1;
  dim3 grid(cdiv(cols, 32), (unsigned)nchunk);
  DISPATCH_DTYPE(dtype, T, (colsum_partial_kernel<T><<<grid, 256, 0, st>>>((const T*)x, rows, cols, ld, rpc, (float*)ws)));
  colsum_finish_kernel<<<cdiv(cols, 128), 128, 0, st>>>((const float*)ws, (int)nchunk, cols, out, accumulate);
  return p2pvg_check_launch("colsum");
}
extern "C" int p2pvg_act_fwd(float* x, int64_t n, int act, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) return P2PVG_OK;
  act_fwd_kernel<<<grid_for(n, 256), 256, 0, st>>>(x, n, act);
  return p2pvg_check_launch("act_fwd");
}
extern "C" int p2pvg_act_bwd(const float* dy, const float* y, float* dx, int64_t n, int act, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) return P2PVG_OK;
  act_bwd_kernel<<<grid_for(n, 256), 256, 0, st>>>(dy, y, dx, n, act);
  return p2pvg_check_launch("act_bwd");
}
