// Training-mode BatchNorm over NHWC activations with statistics grouped per original module call
// (group g = one encoder/decoder call of the reference; SURVEY.md §3.3).  x is [G, R, C] with R rows
// (= B*H*W) per group.  Reductions are deterministic two-stage (per-chunk partials in fp64, then a
// finalize kernel); all kernels are streaming / HBM-bound.
#include "common.cuh"

#define BN_MAXCHUNK 64

namespace {

__device__ __forceinline__ float act_grad(float y, int act) {
  if (act == P2PVG_ACT_LRELU) return y > 0.f ? 1.f : 0.2f;
  if (act == P2PVG_ACT_TANH) return 1.f - y * y;
  return 1.f;
}

// MODE 0: (sum x, sum x^2).  MODE 1: (sum dz, sum dz*xhat), dz = dy*act'(y), xhat=(x-mean)*invstd
// 16-byte vectors along the channel axis (V = 8 bf16 / 4 fp32 channels per thread), 256/CV row lanes per block.
template <typename T, int MODE>
__global__ void __launch_bounds__(256, 3) bn_reduce_kernel(const T* __restrict__ x, const T* __restrict__ dy, const T* __restrict__ y,
                                                        const float* __restrict__ mean, const float* __restrict__ invstd, int act,
                                                        long long R, int C, int rows_per_chunk, double2* __restrict__ partial,
                                                        const float* __restrict__ scale, const float* __restrict__ shift) {
  // y == nullptr (LeakyReLU only): the activation derivative is recomputed from sign(x*scale+shift) instead of reading y
  constexpr int V = VecN<T>::N;
  const int CV = C / V;
  const int lanes = 256 / CV;
  const int cv = threadIdx.x % CV, lane = threadIdx.x / CV;
  const int g = blockIdx.y, chunk = blockIdx.x, nchunk = gridDim.x;
  const long long r0 = (long long)chunk * rows_per_chunk;
  long long r1 = r0 + rows_per_chunk;
  if (r1 > R) r1 = R;
  float s0[V], s1[V], mu[V], is[V], sc[V], sh[V];
  const bool no_y = (MODE == 1) && (y == nullptr);
#pragma unroll
  for (int j = 0; j < V; j++) {
    s0[j] = 0.f; s1[j] = 0.f; mu[j] = 0.f; is[j] = 0.f; sc[j] = 0.f; sh[j] = 0.f;
    if (MODE == 1) {
      mu[j] = mean[(long long)g * C + cv * V + j];
      is[j] = invstd[(long long)g * C + cv * V + j];
      if (no_y) {
        sc[j] = scale[(long long)g * C + cv * V + j];
        sh[j] = shift[(long long)g * C + cv * V + j];
      }
    }
  }
  for (long long r = r0 + lane; r < r1; r += 2 * lanes) {
    // two rows per iteration: all loads issued before use
    const long long off0 = ((long long)g * R + r) * C + cv * V;
    const bool two = (r + lanes) < r1;
    const long long off1 = off0 + (long long)lanes * C;
    uint4 xa = ld_raw16(x + off0), xb = two ? ld_raw16(x + off1) : make_uint4(0u, 0u, 0u, 0u);
    uint4 da, db, ya, yb;
    if (MODE == 1) {
      da = ld_raw16(dy + off0);
      db = two ? ld_raw16(dy + off1) : make_uint4(0u, 0u, 0u, 0u);
      ya = yb = make_uint4(0u, 0u, 0u, 0u);
      if (!no_y) {
        ya = ld_raw16(y + off0);
        if (two) yb = ld_raw16(y + off1);
      }
    }
#pragma unroll
    for (int h = 0; h < 2; h++) {
      if (h == 1 && !two) break;
      float xv[V], dv[V], yv[V];
      unpack16<T>(h ? xb : xa, xv);
      if (MODE == 1) {
        unpack16<T>(h ? db : da, dv);
        unpack16<T>(h ? yb : ya, yv);
      }
#pragma unroll
      for (int j = 0; j < V; j++) {
        if (MODE == 0) {
          s0[j] += xv[j];
          s1[j] = fmaf(xv[j], xv[j], s1[j]);
        } else {
          const float ya_ = no_y ? fmaf(xv[j], sc[j], sh[j]) : yv[j];  // only its sign matters for LeakyReLU
          float dz = dv[j] * act_grad(ya_, act);
          s0[j] += dz;
          s1[j] = fmaf(dz, (xv[j] - mu[j]) * is[j], s1[j]);
        }
      }
    }
  }
  __shared__ float sh0[256 * V];
  __shared__ float sh1[256 * V];
#pragma unroll
  for (int j = 0; j < V; j++) {
    sh0[threadIdx.x * V + j] = s0[j];
    sh1[threadIdx.x * V + j] = s1[j];
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += 256) {
    const int cvv = c / V, j = c % V;
    double a = 0.0, b = 0.0;
    for (int l = 0; l < lanes; l++) {
      a += (double)sh0[(l * CV + cvv) * V + j];
      b += (double)sh1[(l * CV + cvv) * V + j];
    }
    partial[((long long)g * nchunk + chunk) * C + c] = make_double2(a, b);
  }
}

__global__ void bn_fwd_finalize_kernel(const double2* __restrict__ partial, int nchunk, int G, int C, long long R,
                                       const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                       float* __restrict__ mean, float* __restrict__ invstd, float* __restrict__ var_unbiased,
                                       float* __restrict__ scale, float* __restrict__ shift) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= G * C) return;
  int g = idx / C, c = idx % C;
  double a = 0.0, b = 0.0;
  for (int k = 0; k < nchunk; k++) {
    double2 p = partial[((long long)g * nchunk + k) * C + c];
    a += p.x;
    b += p.y;
  }
  double m = a / (double)R;
  double var = b / (double)R - m * m;
  if (var < 0.0) var = 0.0;
  double is = 1.0 / sqrt(var + (double)eps);
  mean[idx] = (float)m;
  invstd[idx] = (float)is;
  var_unbiased[idx] = (float)(R > 1 ? var * (double)R / (double)(R - 1) : var);
  float sc = gamma[c] * (float)is;
  scale[idx] = sc;
  shift[idx] = beta[c] - (float)m * sc;
}

// Statistics whose per-tile column sums came out of a GEMM epilogue (conv_gemm / gemm_tc `stat_partial`): partial is
// [G * parts_per_group][ldp] float2 (sum, sum of squares); channel c of group g = sum over the group's partial rows and
// over the `fold` column groups f*C + c (a GEMM row may hold several pixels / taps of the same channel), giving
// mean / invstd / unbiased var / scale / shift.
// Block = 32 channels x 8 part-lanes, fp64 combine, fixed order (deterministic).
__global__ void __launch_bounds__(256) bn_finalize_tiles_kernel(const float2* __restrict__ partial, int parts_per_group, int ldp, int fold,
                                                                int G, int C, double count, const float* __restrict__ gamma,
                                                                const float* __restrict__ beta, float eps, float* __restrict__ mean,
                                                                float* __restrict__ invstd, float* __restrict__ var_unbiased,
                                                                float* __restrict__ scale, float* __restrict__ shift) {
  const int g = blockIdx.y, cl = threadIdx.x & 31, pl = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cl;
  double a = 0.0, b = 0.0;
  if (c < C) {
    const float2* base = partial + (long long)g * parts_per_group * ldp;
    for (int p = pl; p < parts_per_group; p += 8) {
      const float2* row = base + (long long)p * ldp + c;
      for (int f = 0; f < fold; f++) {
        const float2 v = row[(long long)f * C];
        a += (double)v.x;
        b += (double)v.y;
      }
    }
  }
  __shared__ double sa[8][33], sb[8][33];
  sa[pl][cl] = a;
  sb[pl][cl] = b;
  __syncthreads();
  if (pl == 0 && c < C) {
    for (int k = 1; k < 8; k++) { a += sa[k][cl]; b += sb[k][cl]; }
    const long long idx = (long long)g * C + c;
    const double m = a / count;
    double var = b / count - m * m;
    if (var < 0.0) var = 0.0;
    const double is = 1.0 / sqrt(var + (double)eps);
    mean[idx] = (float)m;
    invstd[idx] = (float)is;
    var_unbiased[idx] = (float)(count > 1.0 ? var * count / (count - 1.0) : var);
    const float sc = gamma[c] * (float)is;
    scale[idx] = sc;
    shift[idx] = beta[c] - (float)m * sc;
  }
}

__global__ void bn_bwd_finalize_kernel(const double2* __restrict__ partial, int nchunk, int G, int C,
                                       float* __restrict__ sum_dz, float* __restrict__ sum_dzx) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= G * C) return;
  int g = idx / C, c = idx % C;
  double a = 0.0, b = 0.0;
  for (int k = 0; k < nchunk; k++) {
    double2 p = partial[((long long)g * nchunk + k) * C + c];
    a += p.x;
    b += p.y;
  }
  sum_dz[idx] = (float)a;
  sum_dzx[idx] = (float)b;
}

// grid (chunk, group); thread = (channel vector cv, row lane); scale / shift of the thread's channels stay in registers
template <typename T>
__global__ void __launch_bounds__(256) bn_act_kernel(const T* __restrict__ x, T* __restrict__ y, const float* __restrict__ scale,
                                                     const float* __restrict__ shift, long long R, int C, int rows_per_chunk, int act) {
  constexpr int V = VecN<T>::N;
  const int CV = C / V;
  const int lanes = 256 / CV;
  const int cv = threadIdx.x % CV, lane = threadIdx.x / CV;
  const int g = blockIdx.y;
  const long long r0 = (long long)blockIdx.x * rows_per_chunk;
  long long r1 = r0 + rows_per_chunk;
  if (r1 > R) r1 = R;
  float sc[V], sh[V];
#pragma unroll
  for (int j = 0; j < V; j++) {
    sc[j] = scale[(long long)g * C + cv * V + j];
    sh[j] = shift[(long long)g * C + cv * V + j];
  }
  for (long long r = r0 + lane; r < r1; r += 4 * lanes) {
    uint4 raw[4];
    long long off[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
      off[u] = ((long long)g * R + r + (long long)u * lanes) * C + cv * V;
      if (r + (long long)u * lanes < r1) raw[u] = ld_raw16(x + off[u]);
    }
#pragma unroll
    for (int u = 0; u < 4; u++) {
      if (r + (long long)u * lanes >= r1) break;
      float v[V];
      unpack16<T>(raw[u], v);
#pragma unroll
      for (int j = 0; j < V; j++) {
        float z = fmaf(v[j], sc[j], sh[j]);
        if (act == P2PVG_ACT_LRELU) z = z > 0.f ? z : 0.2f * z;
        else if (act == P2PVG_ACT_TANH) z = tanhf(z);
        v[j] = z;
      }
      st_raw16(y + off[u], pack16<T>(v));
    }
  }
}

// grid (chunk, group); thread = (channel vector cv, row lane): the per-(group,channel) parameters stay in registers
// and only the activations stream through.
template <typename T>
__global__ void __launch_bounds__(256, 3) bn_bwd_apply_kernel(const T* __restrict__ dy, const T* __restrict__ x, const T* __restrict__ y,
                                                           const float* __restrict__ mean, const float* __restrict__ invstd,
                                                           const float* __restrict__ gamma, const float* __restrict__ sum_dz,
                                                           const float* __restrict__ sum_dzx, long long R, int C, int rows_per_chunk,
                                                           int act, T* __restrict__ dx, const float* __restrict__ scale,
                                                           const float* __restrict__ shift) {
  constexpr int V = VecN<T>::N;
  const int CV = C / V;
  const int lanes = 256 / CV;
  const int cv = threadIdx.x % CV, lane = threadIdx.x / CV;
  const int g = blockIdx.y;
  const long long r0 = (long long)blockIdx.x * rows_per_chunk;
  long long r1 = r0 + rows_per_chunk;
  if (r1 > R) r1 = R;
  const bool no_y = (y == nullptr);
  const float invR = 1.f / (float)R;
  float mu[V], is[V], k0[V], k1[V], k2[V], sc[V], sh[V];
#pragma unroll
  for (int j = 0; j < V; j++) {
    const long long gc = (long long)g * C + cv * V + j;
    mu[j] = mean[gc];
    is[j] = invstd[gc];
    k0[j] = gamma[cv * V + j] * is[j];          // dx = k0 * (dz - k1 - xhat * k2)
    k1[j] = sum_dz[gc] * invR;
    k2[j] = sum_dzx[gc] * invR;
    sc[j] = no_y ? scale[gc] : 0.f;
    sh[j] = no_y ? shift[gc] : 0.f;
  }
  for (long long r = r0 + lane; r < r1; r += 2 * lanes) {
    const long long off0 = ((long long)g * R + r) * C + cv * V;
    const bool two = (r + lanes) < r1;
    const long long off1 = off0 + (long long)lanes * C;
    const uint4 z4 = make_uint4(0u, 0u, 0u, 0u);
    const uint4 da = ld_raw16(dy + off0), xa = ld_raw16(x + off0);
    const uint4 db = two ? ld_raw16(dy + off1) : z4, xb = two ? ld_raw16(x + off1) : z4;
    uint4 ya = z4, yb = z4;
    if (!no_y) {
      ya = ld_raw16(y + off0);
      if (two) yb = ld_raw16(y + off1);
    }
#pragma unroll
    for (int h = 0; h < 2; h++) {
      if (h == 1 && !two) break;
      float dv[V], xv[V], yv[V], o[V];
      unpack16<T>(h ? db : da, dv);
      unpack16<T>(h ? xb : xa, xv);
      unpack16<T>(h ? yb : ya, yv);
#pragma unroll
      for (int j = 0; j < V; j++) {
        const float xhat = (xv[j] - mu[j]) * is[j];
        const float ya_ = no_y ? fmaf(xv[j], sc[j], sh[j]) : yv[j];
        const float dz = dv[j] * act_grad(ya_, act);
        o[j] = k0[j] * (dz - k1[j] - xhat * k2[j]);
      }
      st_raw16(dx + (h ? off1 : off0), pack16<T>(o));
    }
  }
}

__global__ void bn_param_grad_kernel(const float* __restrict__ sum_dz, const float* __restrict__ sum_dzx, int G, int C,
                                     float* __restrict__ dgamma, float* __restrict__ dbeta) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float a = 0.f, b = 0.f;
  for (int g = 0; g < G; g++) {
    a += sum_dzx[(long long)g * C + c];
    b += sum_dz[(long long)g * C + c];
  }
  dgamma[c] = a;
  dbeta[c] = b;
}

__global__ void bn_eval_coeffs_kernel(const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ rmean,
                                      const float* __restrict__ rvar, float eps, int C, float* __restrict__ scale, float* __restrict__ shift) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float sc = gamma[c] / sqrtf(rvar[c] + eps);
  scale[c] = sc;
  shift[c] = beta[c] - rmean[c] * sc;
}

__global__ void bn_ema_kernel(float* __restrict__ rmean, float* __restrict__ rvar, const float* __restrict__ mean,
                              const float* __restrict__ var_unbiased, const int* __restrict__ order, int ncalls, int C,
                              float momentum) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float m = rmean[c], v = rvar[c];
  for (int k = 0; k < ncalls; k++) {
    int g = order[k];
    m = (1.f - momentum) * m + momentum * mean[(long long)g * C + c];
    v = (1.f - momentum) * v + momentum * var_unbiased[(long long)g * C + c];
  }
  rmean[c] = m;
  rvar[c] = v;
}

__attribute__((unused)) inline int grid_for(long long total, int block) {
  long long g = (total + block - 1) / block;
  const long long cap = 132LL * 64;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

struct Chunking {
  int nchunk, rows_per_chunk;
};
inline Chunking choose_chunks(long long R, int C, int vec) {
  int lanes = 256 / (C / vec);
  if (lanes < 1) lanes = 1;
  long long want = (R + (long long)lanes * 16 - 1) / ((long long)lanes * 16);  // >=16 rows per thread
  int nchunk = (int)(want < 1 ? 1 : (want > BN_MAXCHUNK ? BN_MAXCHUNK : want));
  int rpc = (int)((R + nchunk - 1) / nchunk);
  nchunk = (int)((R + rpc - 1) / rpc);
  return Chunking{nchunk, rpc};
}

inline int check_bn_shape(int C, int vec, const char* what) {
  int CV = C / vec;
  if (C % vec != 0 || CV < 1 || CV > 256 || (256 % CV) != 0) {
    p2pvg_set_error("%s: unsupported channel count %d (need C a multiple of the 16-byte vector, C/vec a divisor of 256)", what, C);
    return P2PVG_ERR_UNSUPPORTED;
  }
  return P2PVG_OK;
}

}  // namespace

size_t p2pvg_bn_workspace_bytes_impl(int G, int C) { return (size_t)G * BN_MAXCHUNK * C * sizeof(double2); }

int p2pvg_bn_fwd_stats_impl(const void* x, int dtype, int G, long long R, int C, const float* gamma, const float* beta, float eps,
                            void* ws, size_t ws_bytes, float* mean, float* invstd, float* var_unbiased, float* scale,
                            float* shift, cudaStream_t st) {
  const int vec = dtype == P2PVG_BF16 ? 8 : 4;
  if (int e = check_bn_shape(C, vec, "bn_fwd_stats")) return e;
  P2PVG_REQUIRE(ws_bytes >= p2pvg_bn_workspace_bytes_impl(G, C), P2PVG_ERR_WORKSPACE, "bn_fwd_stats: workspace too small");
  if (G == 0) return P2PVG_OK;
  Chunking ch = choose_chunks(R, C, vec);
  dim3 grid(ch.nchunk, G);
  DISPATCH_DTYPE(dtype, T, (bn_reduce_kernel<T, 0><<<grid, 256, 0, st>>>((const T*)x, nullptr, nullptr, nullptr, nullptr, 0, R, C,
                                                                         ch.rows_per_chunk, (double2*)ws, nullptr, nullptr)));
  bn_fwd_finalize_kernel<<<cdiv((long long)G * C, 256), 256, 0, st>>>((const double2*)ws, ch.nchunk, G, C, R, gamma, beta, eps, mean,
                                                                      invstd, var_unbiased, scale, shift);
  return p2pvg_check_launch("bn_fwd_stats");
}

int p2pvg_bn_act_impl(const void* x, void* y, int dtype, const float* scale, const float* shift, int G, long long R, int C, int act,
                      cudaStream_t st) {
  const int vec = dtype == P2PVG_BF16 ? 8 : 4;
  if (int e = check_bn_shape(C, vec, "bn_act")) return e;
  if (G == 0 || R == 0) return P2PVG_OK;
  Chunking ch = choose_chunks(R, C, vec);
  dim3 grid(ch.nchunk, G);
  DISPATCH_DTYPE(dtype, T, (bn_act_kernel<T><<<grid, 256, 0, st>>>((const T*)x, (T*)y, scale, shift, R, C, ch.rows_per_chunk, act)));
  return p2pvg_check_launch("bn_act");
}

int p2pvg_bn_bwd_impl(const void* dy, const void* x, const void* y, int dtype, const float* mean, const float* invstd,
                      const float* gamma, int G, long long R, int C, int act, void* ws, size_t ws_bytes, void* dx, float* sum_dz,
                      float* sum_dzx, const float* scale, const float* shift, cudaStream_t st) {
  P2PVG_REQUIRE(y != nullptr || (act == P2PVG_ACT_LRELU && scale && shift), P2PVG_ERR_BAD_ARG,
                "bn_bwd: y may only be omitted for LeakyReLU with scale/shift supplied");
  const int vec = dtype == P2PVG_BF16 ? 8 : 4;
  if (int e = check_bn_shape(C, vec, "bn_bwd")) return e;
  P2PVG_REQUIRE(ws_bytes >= p2pvg_bn_workspace_bytes_impl(G, C), P2PVG_ERR_WORKSPACE, "bn_bwd: workspace too small");
  if (G == 0) return P2PVG_OK;
  Chunking ch = choose_chunks(R, C, vec);
  dim3 grid(ch.nchunk, G);
  DISPATCH_DTYPE(dtype, T, (bn_reduce_kernel<T, 1><<<grid, 256, 0, st>>>((const T*)x, (const T*)dy, (const T*)y, mean, invstd, act, R, C,
                                                                         ch.rows_per_chunk, (double2*)ws, scale, shift)));
  bn_bwd_finalize_kernel<<<cdiv((long long)G * C, 256), 256, 0, st>>>((const double2*)ws, ch.nchunk, G, C, sum_dz, sum_dzx);
  DISPATCH_DTYPE(dtype, T, (bn_bwd_apply_kernel<T><<<grid, 256, 0, st>>>((const T*)dy, (const T*)x, (const T*)y, mean, invstd, gamma, sum_dz,
                                                                         sum_dzx, R, C, ch.rows_per_chunk, act, (T*)dx, scale, shift)));
  return p2pvg_check_launch("bn_bwd");
}

int p2pvg_bn_param_grad_impl(const float* sum_dz, const float* sum_dzx, int G, int C, float* dgamma, float* dbeta, cudaStream_t st) {
  bn_param_grad_kernel<<<cdiv(C, 128), 128, 0, st>>>(sum_dz, sum_dzx, G, C, dgamma, dbeta);
  return p2pvg_check_launch("bn_param_grad");
}

int p2pvg_bn_ema_impl(float* rmean, float* rvar, const float* mean, const float* var_unbiased, const int* order, int ncalls, int C,
                      float momentum, cudaStream_t st) {
  bn_ema_kernel<<<cdiv(C, 128), 128, 0, st>>>(rmean, rvar, mean, var_unbiased, order, ncalls, C, momentum);
  return p2pvg_check_launch("bn_ema");
}

int p2pvg_bn_eval_coeffs_impl(const float* gamma, const float* beta, const float* rmean, const float* rvar, float eps, int C, float* scale,
                              float* shift, cudaStream_t st) {
  bn_eval_coeffs_kernel<<<cdiv(C, 128), 128, 0, st>>>(gamma, beta, rmean, rvar, eps, C, scale, shift);
  return p2pvg_check_launch("bn_eval_coeffs");
}

// Forward statistics from GEMM-epilogue partials (see bn_finalize_tiles_kernel).  R = elements per (group, channel).
int p2pvg_bn_fwd_finalize_tiles_impl(const void* partial, int parts_per_group, int ldp, int fold, int G, long long R, int C,
                                     const float* gamma, const float* beta, float eps, float* mean, float* invstd, float* var_unbiased,
                                     float* scale, float* shift, cudaStream_t st) {
  P2PVG_REQUIRE(partial && parts_per_group > 0 && fold > 0 && ldp >= fold * C, P2PVG_ERR_BAD_ARG, "bn_fwd_finalize_tiles: bad partial layout");
  if (G == 0) return P2PVG_OK;
  dim3 grid(cdiv(C, 32), G);
  bn_finalize_tiles_kernel<<<grid, 256, 0, st>>>((const float2*)partial, parts_per_group, ldp, fold, G, C, (double)R, gamma, beta, eps, mean,
                                                 invstd, var_unbiased, scale, shift);
  return p2pvg_check_launch("bn_fwd_finalize_tiles");
}
