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

// dx of one element: k0 = gamma * invstd, k1 = sum(dz) / R, k2 = sum(dz * xhat) / R; ya = the activation output (or any
// value of its sign for LeakyReLU).  Every apply pass computes dx through this one expression, so they agree bit for bit.
__device__ __forceinline__ float bn_dx(float dv, float xv, float ya, int act, float mu, float is, float k0, float k1, float k2) {
  const float xhat = (xv - mu) * is;
  const float dz = dv * act_grad(ya, act);
  return k0 * (dz - k1 - xhat * k2);
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
        const float ya_ = no_y ? fmaf(xv[j], sc[j], sh[j]) : yv[j];
        o[j] = bn_dx(dv[j], xv[j], ya_, act, mu[j], is[j], k0[j], k1[j], k2[j]);
      }
      st_raw16(dx + (h ? off1 : off0), pack16<T>(o));
    }
  }
}

// The per-(group, channel) coefficients of bn_bwd_apply_kernel for the 8 bf16 channels starting at gc, for the
// weight-gradient apply pass below (LeakyReLU, slope recomputed from sign(x*scale+shift)).
struct BnBwdCoef {
  float mu[8], is[8], k0[8], k1[8], k2[8], sc[8], sh[8];
};
__device__ __forceinline__ void load_bwd_coef(BnBwdCoef& k, long long gc, int c, const float* __restrict__ mean,
                                              const float* __restrict__ invstd, const float* __restrict__ gamma,
                                              const float* __restrict__ sum_dz, const float* __restrict__ sum_dzx,
                                              const float* __restrict__ scale, const float* __restrict__ shift, float invR) {
#pragma unroll
  for (int j = 0; j < 8; j++) {
    k.mu[j] = mean[gc + j];
    k.is[j] = invstd[gc + j];
    k.k0[j] = gamma[c + j] * k.is[j];
    k.k1[j] = sum_dz[gc + j] * invR;
    k.k2[j] = sum_dzx[gc + j] * invR;
    k.sc[j] = scale[gc + j];
    k.sh[j] = shift[gc + j];
  }
}
// dx of one row's 8 channels, rounded to bf16 (returned packed, and as floats in o)
__device__ __forceinline__ uint4 bwd_dx8(const BnBwdCoef& k, uint4 d, uint4 x, float* o) {
  float dv[8], xv[8];
  unpack16<bf16>(d, dv);
  unpack16<bf16>(x, xv);
#pragma unroll
  for (int j = 0; j < 8; j++) o[j] = bn_dx(dv[j], xv[j], fmaf(xv[j], k.sc[j], k.sh[j]), P2PVG_ACT_LRELU, k.mu[j], k.is[j], k.k0[j], k.k1[j], k.k2[j]);
  const uint4 r = pack16<bf16>(o);
  unpack16<bf16>(r, o);
  return r;
}

// bn_bwd_apply_kernel (bf16, LeakyReLU) that also writes the skip-frame sums of dx: grid (chunk, source f), and the block of
// source f handles the rows of every group g with grp_src[g] == f, in increasing g.  dx_sum[f] = bf16(sum of the
// bf16-rounded dx in fp32, starting from 0) -- group_sum_kernel's order, so it is bit-identical to a group_sum of the
// stored dx; a source no group maps to comes out as zeros.  A thread owns 4 channels (8-byte vectors) of SKIP_ROWS rows of
// the chunk: the group's coefficients are loaded once per group for all of them, the rows' loads are all in flight at
// once, and the running sums live in shared memory (private to the thread, so no barrier).
#define SKIP_ROWS 6
__global__ void __launch_bounds__(256, 2) bn_bwd_apply_skip_kernel(const bf16* dy, const bf16* __restrict__ x,
                                                                    const float* __restrict__ mean, const float* __restrict__ invstd,
                                                                    const float* __restrict__ gamma, const float* __restrict__ sum_dz,
                                                                    const float* __restrict__ sum_dzx, const float* __restrict__ scale,
                                                                    const float* __restrict__ shift, const int* __restrict__ grp_src,
                                                                    int G, long long R, int C, bf16* dx, bf16* __restrict__ dx_sum) {
  __shared__ float4 acc[SKIP_ROWS][256];
  const int CV = C / 4;
  const int lanes = 256 / CV;
  const int cv = threadIdx.x % CV, lane = threadIdx.x / CV;
  const int f = blockIdx.y;
  const long long r = (long long)blockIdx.x * (SKIP_ROWS * lanes) + lane;   // rows r + u * lanes
  const float invR = 1.f / (float)R;
#pragma unroll
  for (int u = 0; u < SKIP_ROWS; u++) acc[u][threadIdx.x] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int g = 0; g < G; g++) {
    if (grp_src[g] != f) continue;
    const long long gc = (long long)g * C + cv * 4;
    const float4 mu = *reinterpret_cast<const float4*>(mean + gc), is = *reinterpret_cast<const float4*>(invstd + gc);
    const float4 ga = *reinterpret_cast<const float4*>(gamma + cv * 4);
    const float4 s0 = *reinterpret_cast<const float4*>(sum_dz + gc), s1 = *reinterpret_cast<const float4*>(sum_dzx + gc);
    const float4 sc = *reinterpret_cast<const float4*>(scale + gc), sh = *reinterpret_cast<const float4*>(shift + gc);
    const float mu_[4] = {mu.x, mu.y, mu.z, mu.w}, is_[4] = {is.x, is.y, is.z, is.w}, ga_[4] = {ga.x, ga.y, ga.z, ga.w};
    const float s0_[4] = {s0.x, s0.y, s0.z, s0.w}, s1_[4] = {s1.x, s1.y, s1.z, s1.w};
    const float sc_[4] = {sc.x, sc.y, sc.z, sc.w}, sh_[4] = {sh.x, sh.y, sh.z, sh.w};
    uint2 d[SKIP_ROWS], xa[SKIP_ROWS];
#pragma unroll
    for (int u = 0; u < SKIP_ROWS; u++) {
      if (r + (long long)u * lanes < R) {
        const long long off = ((long long)g * R + r + (long long)u * lanes) * C + cv * 4;
        d[u] = *reinterpret_cast<const uint2*>(dy + off);
        xa[u] = *reinterpret_cast<const uint2*>(x + off);
      }
    }
#pragma unroll
    for (int u = 0; u < SKIP_ROWS; u++) {
      if (r + (long long)u * lanes >= R) break;
      const uint32_t dw[2] = {d[u].x, d[u].y}, xw[2] = {xa[u].x, xa[u].y};
      float o[4];
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const float dv = __uint_as_float((j & 1) ? (dw[j >> 1] & 0xffff0000u) : (dw[j >> 1] << 16));
        const float xv = __uint_as_float((j & 1) ? (xw[j >> 1] & 0xffff0000u) : (xw[j >> 1] << 16));
        o[j] = bn_dx(dv, xv, fmaf(xv, sc_[j], sh_[j]), P2PVG_ACT_LRELU, mu_[j], is_[j], ga_[j] * is_[j], s0_[j] * invR, s1_[j] * invR);
      }
      const __nv_bfloat162 p0 = __floats2bfloat162_rn(o[0], o[1]), p1 = __floats2bfloat162_rn(o[2], o[3]);
      uint2 pk;
      pk.x = *reinterpret_cast<const uint32_t*>(&p0);
      pk.y = *reinterpret_cast<const uint32_t*>(&p1);
      *reinterpret_cast<uint2*>(dx + ((long long)g * R + r + (long long)u * lanes) * C + cv * 4) = pk;
      float4 a = acc[u][threadIdx.x];
      a.x += __low2float(p0); a.y += __high2float(p0); a.z += __low2float(p1); a.w += __high2float(p1);
      acc[u][threadIdx.x] = a;
    }
  }
#pragma unroll
  for (int u = 0; u < SKIP_ROWS; u++) {
    if (r + (long long)u * lanes >= R) break;
    const float4 a = acc[u][threadIdx.x];
    st_f4<bf16>(dx_sum + ((long long)f * R + r + (long long)u * lanes) * C + cv * 4, f4{{a.x, a.y, a.z, a.w}});
  }
}

// bn_bwd_apply_kernel (bf16, LeakyReLU, C = 64) of a layer whose convolution (4x4, stride 2, pad 1) reads a 1-channel map
// `cin` of twice the output resolution: dx is not stored; its weight gradient gW[c][tap] = sum over rows of bf16(dx[c]) *
// cin[tap] is accumulated instead, on the tensor cores: per 64-row tile the block puts the rounded dx (as A = [64 ch][64
// rows]) and the rows' 16 taps (as B^T = [16 taps][64 rows]) into shared memory as bf16 row pairs, and warp w runs
// mma.m16n8k16 (fp32 accumulate) on channels 16 (w / 2) .. + 15 and taps 8 (w % 2) .. + 7 over the tile's four 16-row
// steps.  The products are exact (bf16 x bf16); the block writes its [64][16] fp32 sums as one partial.
// Shared-memory word (row, k2) of a [rows][32 row pairs] bf16x2 array sits at k2 ^ 4 * swz(row): the fragment loads (8
// rows x 4 pairs per warp) and the stores (8 channels x 4 row pairs of the apply mapping; one tap x 32 pairs) are then
// free of bank conflicts.
#define WG_TILE 64
__device__ __forceinline__ int wg_word(int row, int k2, int swz) { return row * (WG_TILE / 2) + (k2 ^ (4 * swz)); }
// B^T[n][p] = (tap n of tile row 2 p, of row 2 p + 1): thread = (row pair p, taps n0, n0 + 1).  The taps of row r (of the
// group's rows) are the 4x4 / stride-2 / pad-1 patch of the 1-channel map cin_g [images][2 Ho][2 Ho] at (r / Ho^2, r % Ho^2)
__device__ __forceinline__ void stage_taps(uint32_t* sB, const bf16* __restrict__ cin_g, int t0, int r1, int lgHo) {
  const int Ho = 1 << lgHo, Wi = 2 * Ho;
  const int p = threadIdx.x & 31, n0 = (threadIdx.x >> 5) * 2;
  uint32_t v[2][2] = {{0u, 0u}, {0u, 0u}};
#pragma unroll
  for (int h = 0; h < 2; h++) {
    const int r = t0 + 2 * p + h;
    if (r >= r1) continue;
    const int oy = (r >> lgHo) & (Ho - 1), ox = r & (Ho - 1);
    const bf16* src = cin_g + (long long)(r >> (2 * lgHo)) * Wi * Wi;
#pragma unroll
    for (int e = 0; e < 2; e++) {
      const int n = n0 + e, iy = 2 * oy - 1 + (n >> 2), ix = 2 * ox - 1 + (n & 3);
      if (iy >= 0 && iy < Wi && ix >= 0 && ix < Wi) v[e][h] = __bfloat16_as_ushort(src[iy * Wi + ix]);
    }
  }
#pragma unroll
  for (int e = 0; e < 2; e++) sB[wg_word(n0 + e, p, (n0 + e) & 7)] = v[e][0] | (v[e][1] << 16);
}
// acc += A[16 (w / 2) .. + 15][tile] * B[tile][8 (w % 2) .. + 7] for warp w: four m16n8k16 steps over the tile's 64 rows
__device__ __forceinline__ void mma_tile(const uint32_t* sA, const uint32_t* sB, float* acc) {
  const int warp = threadIdx.x >> 5, ln = threadIdx.x & 31, gid = ln >> 2, tig = ln & 3;
  const int mrow = (warp >> 1) * 16 + gid, ncol = (warp & 1) * 8 + gid;
  const int sa0 = (mrow & 7) ^ (mrow >> 3), sa1 = ((mrow + 8) & 7) ^ ((mrow + 8) >> 3);
#pragma unroll
  for (int ks = 0; ks < WG_TILE / 16; ks++) {
    const int k2 = ks * 8 + tig;
    const uint32_t a0 = sA[wg_word(mrow, k2, sa0)], a1 = sA[wg_word(mrow + 8, k2, sa1)];
    const uint32_t a2 = sA[wg_word(mrow, k2 + 4, sa0)], a3 = sA[wg_word(mrow + 8, k2 + 4, sa1)];
    const uint32_t b0 = sB[wg_word(ncol, k2, ncol & 7)], b1 = sB[wg_word(ncol, k2 + 4, ncol & 7)];
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(acc[0]), "+f"(acc[1]), "+f"(acc[2]), "+f"(acc[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
  }
}
// the warp's 16 x 8 accumulator tile -> out[64][16]: (gid, 2 tig + {0, 1}) and (gid + 8, ...)
__device__ __forceinline__ void store_wgrad_partial(float* out, const float* acc) {
  const int warp = threadIdx.x >> 5, ln = threadIdx.x & 31, gid = ln >> 2, tig = ln & 3;
  const int mrow = (warp >> 1) * 16 + gid, nc = (warp & 1) * 8 + 2 * tig;
  *reinterpret_cast<float2*>(&out[mrow * 16 + nc]) = make_float2(acc[0], acc[1]);
  *reinterpret_cast<float2*>(&out[(mrow + 8) * 16 + nc]) = make_float2(acc[2], acc[3]);
}
__global__ void __launch_bounds__(256, 2) bn_bwd_apply_wgrad_c1_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x,
                                                                        const float* __restrict__ mean, const float* __restrict__ invstd,
                                                                        const float* __restrict__ gamma, const float* __restrict__ sum_dz,
                                                                        const float* __restrict__ sum_dzx, const float* __restrict__ scale,
                                                                        const float* __restrict__ shift, const bf16* __restrict__ cin,
                                                                        int lgHo, int R, int rows_per_chunk, float* __restrict__ wpart) {
  constexpr int C = 64;
  __shared__ uint32_t sA[2][C * WG_TILE / 2];   // double-buffered: one barrier per tile
  __shared__ uint32_t sB[2][16 * WG_TILE / 2];
  const int cv = threadIdx.x & 7, pr = threadIdx.x >> 3;   // apply mapping: 8 channels x the tile's row pair pr
  const int g = blockIdx.y;
  const int r0 = blockIdx.x * rows_per_chunk;
  const int r1 = min(r0 + rows_per_chunk, R);
  const float invR = 1.f / (float)R;
  BnBwdCoef k;
  load_bwd_coef(k, (long long)g * C + cv * 8, cv * 8, mean, invstd, gamma, sum_dz, sum_dzx, scale, shift, invR);
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  const bf16* cin_g = cin + (long long)g * (R >> (2 * lgHo)) * (4 << (2 * lgHo));
  const bf16* dy_g = dy + (long long)g * R * C + cv * 8;
  const bf16* x_g = x + (long long)g * R * C + cv * 8;
  const uint4 z4 = make_uint4(0u, 0u, 0u, 0u);
  // this thread's two rows of the first tile; each tile's loads are issued before the previous tile's MMAs
  uint4 da = z4, xa = z4, db = z4, xb = z4;
  {
    const int ra = r0 + 2 * pr;
    if (ra < r1) { da = ld_raw16(dy_g + (long long)ra * C); xa = ld_raw16(x_g + (long long)ra * C); }
    if (ra + 1 < r1) { db = ld_raw16(dy_g + (long long)(ra + 1) * C); xb = ld_raw16(x_g + (long long)(ra + 1) * C); }
  }
  int buf = 0;
  for (int t0 = r0; t0 < r1; t0 += WG_TILE, buf ^= 1) {
    {  // dx of rows 2 pr, 2 pr + 1 -> A[c][pr] = (dx[2 pr][c], dx[2 pr + 1][c])
      const int ra = t0 + 2 * pr;
      float o[8];
      const uint4 pa = ra < r1 ? bwd_dx8(k, da, xa, o) : z4;
      const uint4 pb = ra + 1 < r1 ? bwd_dx8(k, db, xb, o) : z4;
      const uint32_t wa[4] = {pa.x, pa.y, pa.z, pa.w}, wb[4] = {pb.x, pb.y, pb.z, pb.w};
#pragma unroll
      for (int j = 0; j < 8; j++) sA[buf][wg_word(cv * 8 + j, pr, j ^ cv)] = __byte_perm(wa[j >> 1], wb[j >> 1], (j & 1) ? 0x7632 : 0x5410);
      const int rn = ra + WG_TILE;
      da = xa = db = xb = z4;
      if (rn < r1) { da = ld_raw16(dy_g + (long long)rn * C); xa = ld_raw16(x_g + (long long)rn * C); }
      if (rn + 1 < r1) { db = ld_raw16(dy_g + (long long)(rn + 1) * C); xb = ld_raw16(x_g + (long long)(rn + 1) * C); }
    }
    stage_taps(sB[buf], cin_g, t0, r1, lgHo);
    __syncthreads();
    mma_tile(sA[buf], sB[buf], acc);
  }
  store_wgrad_partial(wpart + ((long long)g * gridDim.x + blockIdx.x) * (C * 16), acc);
}

// bn_reduce_kernel<bf16, 1> (LeakyReLU from sign(x*scale+shift), C = 64, same rows, same order, same partials) of a layer
// whose output y = bf16(lrelu(x*scale+shift)) -- bit-identical to what bn_act_kernel stored -- feeds a 4x4 / stride-2 /
// pad-1 transposed convolution to one channel at twice the resolution: it also accumulates that convolution's weight
// gradient gW[c][tap] = sum over rows of y[c] * dout[tap], dout the gradient of the 1-channel output map, on the tensor
// cores as bn_bwd_apply_wgrad_c1_kernel does (the threads of rows 2p and 2p + 1 swap one row's y to form A's row pairs).
__global__ void __launch_bounds__(256, 2) bn_reduce_wgrad_c1_kernel(const bf16* __restrict__ x, const bf16* __restrict__ dy,
                                                                     const float* __restrict__ mean, const float* __restrict__ invstd,
                                                                     int R, int rows_per_chunk, double2* __restrict__ partial,
                                                                     const float* __restrict__ scale, const float* __restrict__ shift,
                                                                     const bf16* __restrict__ dout, int lgHo, float* __restrict__ wpart) {
  constexpr int C = 64, V = 8, CV = 8, lanes = 32;
  __shared__ uint32_t sA[2][C * WG_TILE / 2];
  __shared__ uint32_t sB[2][16 * WG_TILE / 2];
  const int cv = threadIdx.x % CV, lane = threadIdx.x / CV;
  const int g = blockIdx.y, chunk = blockIdx.x, nchunk = gridDim.x;
  const int r0 = chunk * rows_per_chunk;
  const int r1 = min(r0 + rows_per_chunk, R);
  float s0[V], s1[V], mu[V], is[V], sc[V], sh[V];
#pragma unroll
  for (int j = 0; j < V; j++) {
    s0[j] = 0.f; s1[j] = 0.f;
    mu[j] = mean[(long long)g * C + cv * V + j];
    is[j] = invstd[(long long)g * C + cv * V + j];
    sc[j] = scale[(long long)g * C + cv * V + j];
    sh[j] = shift[(long long)g * C + cv * V + j];
  }
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  const bf16* dout_g = dout + (long long)g * (R >> (2 * lgHo)) * (4 << (2 * lgHo));
  const uint4 z4 = make_uint4(0u, 0u, 0u, 0u);
  // rows t0 + lane and t0 + lane + 32 of each 64-row tile, exactly as bn_reduce_kernel's iteration over r = t0 + lane; each
  // tile's loads are issued before the previous tile's MMAs
  const bf16* x_t = x + ((long long)g * R + lane) * C + cv * V;
  const bf16* dy_t = dy + ((long long)g * R + lane) * C + cv * V;
  uint4 xa = z4, xb = z4, da = z4, db = z4;
  if (r0 + lane < r1) { xa = ld_raw16(x_t + (long long)r0 * C); da = ld_raw16(dy_t + (long long)r0 * C); }
  if (r0 + lane + lanes < r1) { xb = ld_raw16(x_t + (long long)(r0 + lanes) * C); db = ld_raw16(dy_t + (long long)(r0 + lanes) * C); }
  int buf = 0;
  for (int t0 = r0; t0 < r1; t0 += 2 * lanes, buf ^= 1) {
    const int r = t0 + lane;
    const bool one = r < r1, two = (r + lanes) < r1;
    float yv[2][V];
#pragma unroll
    for (int h = 0; h < 2; h++) {
      float xv[V], dv[V];
      unpack16<bf16>(h ? xb : xa, xv);
      unpack16<bf16>(h ? db : da, dv);
#pragma unroll
      for (int j = 0; j < V; j++) {
        const float ya_ = fmaf(xv[j], sc[j], sh[j]);
        yv[h][j] = ya_ > 0.f ? ya_ : 0.2f * ya_;
        if (h == 0 ? !one : !two) continue;
        float dz = dv[j] * act_grad(ya_, P2PVG_ACT_LRELU);
        s0[j] += dz;
        s1[j] = fmaf(dz, (xv[j] - mu[j]) * is[j], s1[j]);
      }
    }
    uint4 ya = one ? pack16<bf16>(yv[0]) : z4, yb = two ? pack16<bf16>(yv[1]) : z4;
    xa = xb = da = db = z4;
    if (r + 2 * lanes < r1) { xa = ld_raw16(x_t + (long long)(t0 + 2 * lanes) * C); da = ld_raw16(dy_t + (long long)(t0 + 2 * lanes) * C); }
    if (r + 3 * lanes < r1) { xb = ld_raw16(x_t + (long long)(t0 + 3 * lanes) * C); db = ld_raw16(dy_t + (long long)(t0 + 3 * lanes) * C); }
    {  // even lane: rows (lane, lane + 1) = pair lane / 2; odd lane: rows (lane + 31, lane + 32) = pair 16 + lane / 2
      const bool odd = lane & 1;
      uint4 snd = odd ? ya : yb, rcv;
      rcv.x = __shfl_xor_sync(0xffffffffu, snd.x, CV);
      rcv.y = __shfl_xor_sync(0xffffffffu, snd.y, CV);
      rcv.z = __shfl_xor_sync(0xffffffffu, snd.z, CV);
      rcv.w = __shfl_xor_sync(0xffffffffu, snd.w, CV);
      const uint4 lo = odd ? rcv : ya, hi = odd ? yb : rcv;
      const int pr = odd ? 16 + (lane >> 1) : (lane >> 1);
      const uint32_t wl[4] = {lo.x, lo.y, lo.z, lo.w}, wh[4] = {hi.x, hi.y, hi.z, hi.w};
#pragma unroll
      for (int j = 0; j < 8; j++) sA[buf][wg_word(cv * 8 + j, pr, j ^ cv)] = __byte_perm(wl[j >> 1], wh[j >> 1], (j & 1) ? 0x7632 : 0x5410);
    }
    stage_taps(sB[buf], dout_g, t0, r1, lgHo);
    __syncthreads();
    mma_tile(sA[buf], sB[buf], acc);
  }
  store_wgrad_partial(wpart + ((long long)g * nchunk + chunk) * (C * 16), acc);
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

// dw[e] = sum over the nparts partials of entry e (fp64, fixed order): block = 32 entries x 32 part lanes
__global__ void __launch_bounds__(1024) wgrad_partials_finalize_kernel(const float* __restrict__ wpart, int nparts, int E, float* __restrict__ dw) {
  const int el = threadIdx.x & 31, pl = threadIdx.x >> 5;
  const int e = blockIdx.x * 32 + el;
  double a = 0.0;
  if (e < E) {
    int p = pl;
    for (; p + 96 < nparts; p += 128) {
      const float v0 = wpart[(long long)p * E + e], v1 = wpart[(long long)(p + 32) * E + e];
      const float v2 = wpart[(long long)(p + 64) * E + e], v3 = wpart[(long long)(p + 96) * E + e];
      a += (double)v0;
      a += (double)v1;
      a += (double)v2;
      a += (double)v3;
    }
    for (; p < nparts; p += 32) a += (double)wpart[(long long)p * E + e];
  }
  __shared__ double s[32][33];
  s[pl][el] = a;
  __syncthreads();
  if (pl == 0 && e < E) {
    for (int q = 1; q < 32; q++) a += s[q][el];
    dw[e] = (float)a;
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

extern "C" size_t p2pvg_bn_workspace_bytes(int G, int C) { return (size_t)G * BN_MAXCHUNK * C * sizeof(double2); }

extern "C" int p2pvg_bn_fwd_stats(const void* x, int dtype, int G, int64_t R, int C, const float* gamma, const float* beta, float eps,
                                  void* ws, size_t ws_bytes, float* mean, float* invstd, float* var_unbiased, float* scale, float* shift,
                                  void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const int vec = dtype == P2PVG_BF16 ? 8 : 4;
  if (int e = check_bn_shape(C, vec, "bn_fwd_stats")) return e;
  P2PVG_REQUIRE(ws_bytes >= p2pvg_bn_workspace_bytes(G, C), P2PVG_ERR_WORKSPACE, "bn_fwd_stats: workspace too small");
  if (G == 0) return P2PVG_OK;
  Chunking ch = choose_chunks(R, C, vec);
  dim3 grid(ch.nchunk, G);
  DISPATCH_DTYPE(dtype, T, (bn_reduce_kernel<T, 0><<<grid, 256, 0, st>>>((const T*)x, nullptr, nullptr, nullptr, nullptr, 0, R, C,
                                                                         ch.rows_per_chunk, (double2*)ws, nullptr, nullptr)));
  bn_fwd_finalize_kernel<<<cdiv((long long)G * C, 256), 256, 0, st>>>((const double2*)ws, ch.nchunk, G, C, R, gamma, beta, eps, mean,
                                                                      invstd, var_unbiased, scale, shift);
  return p2pvg_check_launch("bn_fwd_stats");
}

extern "C" int p2pvg_bn_act(const void* x, void* y, int dtype, const float* scale, const float* shift, int G, int64_t R, int C, int act,
                            void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const int vec = dtype == P2PVG_BF16 ? 8 : 4;
  if (int e = check_bn_shape(C, vec, "bn_act")) return e;
  if (G == 0 || R == 0) return P2PVG_OK;
  Chunking ch = choose_chunks(R, C, vec);
  dim3 grid(ch.nchunk, G);
  DISPATCH_DTYPE(dtype, T, (bn_act_kernel<T><<<grid, 256, 0, st>>>((const T*)x, (T*)y, scale, shift, R, C, ch.rows_per_chunk, act)));
  return p2pvg_check_launch("bn_act");
}

extern "C" int p2pvg_bn_bwd(const void* dy, const void* x, const void* y, int dtype, const float* mean, const float* invstd,
                            const float* gamma, int G, int64_t R, int C, int act, void* ws, size_t ws_bytes, void* dx, float* sum_dz,
                            float* sum_dzx, const float* scale, const float* shift, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  P2PVG_REQUIRE(y != nullptr || (act == P2PVG_ACT_LRELU && scale && shift), P2PVG_ERR_BAD_ARG,
                "bn_bwd: y may only be omitted for LeakyReLU with scale/shift supplied");
  const int vec = dtype == P2PVG_BF16 ? 8 : 4;
  if (int e = check_bn_shape(C, vec, "bn_bwd")) return e;
  P2PVG_REQUIRE(ws_bytes >= p2pvg_bn_workspace_bytes(G, C), P2PVG_ERR_WORKSPACE, "bn_bwd: workspace too small");
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

extern "C" size_t p2pvg_bn_wgrad_c1_partial_bytes(int G) { return (size_t)G * BN_MAXCHUNK * 64 * 16 * sizeof(float); }

// log2(Ho) for the weight-gradient passes: Ho a power of two, R a whole number of Ho x Ho maps below 2^31 rows
static int wgrad_c1_geometry(const char* what, long long R, int Ho, int G, size_t wpart_bytes, int* lg) {
  *lg = 0;
  while (*lg < 15 && (1 << *lg) < Ho) (*lg)++;
  P2PVG_REQUIRE(Ho >= 1 && (1 << *lg) == Ho && R % ((long long)Ho * Ho) == 0 && R < (1LL << 31), P2PVG_ERR_BAD_ARG,
                "%s: R = %lld is not a whole number of %dx%d maps (Ho a power of two, R < 2^31)", what, R, Ho, Ho);
  P2PVG_REQUIRE(wpart_bytes >= p2pvg_bn_wgrad_c1_partial_bytes(G), P2PVG_ERR_WORKSPACE, "%s: partial buffer too small", what);
  return P2PVG_OK;
}

// The reduce pass and finalize of p2pvg_bn_bwd (bf16, LeakyReLU recomputed from scale / shift).  dout != NULL: the reduce pass
// also writes the weight gradient dw of the 1-channel transposed convolution that reads y (bn_reduce_wgrad_c1_kernel).
static int bn_bwd_sums_lrelu(const char* what, const void* dy, const void* x, const float* mean, const float* invstd, int G, long long R,
                             int C, void* ws, size_t ws_bytes, float* sum_dz, float* sum_dzx, const float* scale, const float* shift,
                             const void* dout, int Ho, float* wpart, size_t wpart_bytes, float* dw, cudaStream_t st) {
  P2PVG_REQUIRE(dy && x && mean && invstd && sum_dz && sum_dzx && scale && shift, P2PVG_ERR_BAD_ARG, "%s: null pointer", what);
  if (int e = check_bn_shape(C, 8, what)) return e;
  P2PVG_REQUIRE(ws_bytes >= p2pvg_bn_workspace_bytes(G, C), P2PVG_ERR_WORKSPACE, "%s: workspace too small", what);
  Chunking ch = choose_chunks(R, C, 8);
  if (dout) {
    P2PVG_REQUIRE(C == 64 && wpart && dw, P2PVG_ERR_BAD_ARG, "%s: the weight-gradient reduce needs C = 64, wpart and dw", what);
    int lg;
    if (int e = wgrad_c1_geometry(what, R, Ho, G, wpart_bytes, &lg)) return e;
    bn_reduce_wgrad_c1_kernel<<<dim3(ch.nchunk, G), 256, 0, st>>>((const bf16*)x, (const bf16*)dy, mean, invstd, (int)R, ch.rows_per_chunk,
                                                                  (double2*)ws, scale, shift, (const bf16*)dout, lg, wpart);
    wgrad_partials_finalize_kernel<<<C * 16 / 32, 1024, 0, st>>>(wpart, G * ch.nchunk, C * 16, dw);
  } else {
    bn_reduce_kernel<bf16, 1><<<dim3(ch.nchunk, G), 256, 0, st>>>((const bf16*)x, (const bf16*)dy, nullptr, mean, invstd, P2PVG_ACT_LRELU, R,
                                                                   C, ch.rows_per_chunk, (double2*)ws, scale, shift);
  }
  bn_bwd_finalize_kernel<<<cdiv((long long)G * C, 256), 256, 0, st>>>((const double2*)ws, ch.nchunk, G, C, sum_dz, sum_dzx);
  return P2PVG_OK;
}

extern "C" int p2pvg_bn_bwd_group_sum(const void* dy, const void* x, const float* mean, const float* invstd, const float* gamma, int G,
                                      int64_t R, int C, void* ws, size_t ws_bytes, void* dx, float* sum_dz, float* sum_dzx,
                                      const float* scale, const float* shift, const int* grp_src, int F, void* dx_sum, const void* dout,
                                      int Ho, float* wpart, size_t wpart_bytes, float* dw, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  P2PVG_REQUIRE(gamma && dx && grp_src && dx_sum && F >= 1, P2PVG_ERR_BAD_ARG, "bn_bwd_group_sum: bad arguments");
  if (G == 0 || R == 0) return P2PVG_OK;
  if (int e = bn_bwd_sums_lrelu("bn_bwd_group_sum", dy, x, mean, invstd, G, R, C, ws, ws_bytes, sum_dz, sum_dzx, scale, shift, dout, Ho,
                                wpart, wpart_bytes, dw, st)) return e;
  const long long rpb = SKIP_ROWS * (256 / (C / 4));
  const long long nblk = (R + rpb - 1) / rpb;
  P2PVG_REQUIRE(nblk < (1LL << 31) && F <= 65535, P2PVG_ERR_UNSUPPORTED, "bn_bwd_group_sum: grid too large");
  bn_bwd_apply_skip_kernel<<<dim3((unsigned)nblk, F), 256, 0, st>>>((const bf16*)dy, (const bf16*)x, mean, invstd, gamma, sum_dz, sum_dzx,
                                                                   scale, shift, grp_src, G, R, C, (bf16*)dx, (bf16*)dx_sum);
  return p2pvg_check_launch("bn_bwd_group_sum");
}

extern "C" int p2pvg_bn_bwd_wgrad_c1(const void* dy, const void* x, const float* mean, const float* invstd, const float* gamma, int G,
                                     int64_t R, void* ws, size_t ws_bytes, float* sum_dz, float* sum_dzx, const float* scale,
                                     const float* shift, const void* cin, int Ho, float* wpart, size_t wpart_bytes, float* dw,
                                     void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const int C = 64;
  P2PVG_REQUIRE(gamma && cin && wpart && dw, P2PVG_ERR_BAD_ARG, "bn_bwd_wgrad_c1: null pointer");
  int lg;
  if (int e = wgrad_c1_geometry("bn_bwd_wgrad_c1", R, Ho, G, wpart_bytes, &lg)) return e;
  if (G == 0 || R == 0) {
    cudaMemsetAsync(dw, 0, C * 16 * sizeof(float), st);
    return p2pvg_check_launch("bn_bwd_wgrad_c1");
  }
  if (int e = bn_bwd_sums_lrelu("bn_bwd_wgrad_c1", dy, x, mean, invstd, G, R, C, ws, ws_bytes, sum_dz, sum_dzx, scale, shift, nullptr, 0,
                                nullptr, 0, nullptr, st)) return e;
  Chunking ch = choose_chunks(R, C, 8);
  bn_bwd_apply_wgrad_c1_kernel<<<dim3(ch.nchunk, G), 256, 0, st>>>((const bf16*)dy, (const bf16*)x, mean, invstd, gamma, sum_dz, sum_dzx,
                                                                   scale, shift, (const bf16*)cin, lg, (int)R, ch.rows_per_chunk, wpart);
  wgrad_partials_finalize_kernel<<<C * 16 / 32, 1024, 0, st>>>(wpart, G * ch.nchunk, C * 16, dw);
  return p2pvg_check_launch("bn_bwd_wgrad_c1");
}

extern "C" int p2pvg_bn_param_grad(const float* sum_dz, const float* sum_dzx, int G, int C, float* dgamma, float* dbeta, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  bn_param_grad_kernel<<<cdiv(C, 128), 128, 0, st>>>(sum_dz, sum_dzx, G, C, dgamma, dbeta);
  return p2pvg_check_launch("bn_param_grad");
}

extern "C" int p2pvg_bn_ema(float* rmean, float* rvar, const float* mean, const float* var_unbiased, const int* order, int ncalls, int C,
                            float momentum, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  bn_ema_kernel<<<cdiv(C, 128), 128, 0, st>>>(rmean, rvar, mean, var_unbiased, order, ncalls, C, momentum);
  return p2pvg_check_launch("bn_ema");
}

extern "C" int p2pvg_bn_eval_coeffs(const float* gamma, const float* beta, const float* rmean, const float* rvar, float eps, int C,
                                    float* scale, float* shift, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  bn_eval_coeffs_kernel<<<cdiv(C, 128), 128, 0, st>>>(gamma, beta, rmean, rvar, eps, C, scale, shift);
  return p2pvg_check_launch("bn_eval_coeffs");
}

// Forward statistics from GEMM-epilogue partials (see bn_finalize_tiles_kernel).  R = elements per (group, channel).
extern "C" int p2pvg_bn_fwd_finalize_tiles(const void* partial, int parts_per_group, int ldp, int fold, int G, int64_t R, int C,
                                           const float* gamma, const float* beta, float eps, float* mean, float* invstd,
                                           float* var_unbiased, float* scale, float* shift, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  P2PVG_REQUIRE(partial && parts_per_group > 0 && fold > 0 && ldp >= fold * C, P2PVG_ERR_BAD_ARG, "bn_fwd_finalize_tiles: bad partial layout");
  if (G == 0) return P2PVG_OK;
  dim3 grid(cdiv(C, 32), G);
  bn_finalize_tiles_kernel<<<grid, 256, 0, st>>>((const float2*)partial, parts_per_group, ldp, fold, G, C, (double)R, gamma, beta, eps, mean,
                                                 invstd, var_unbiased, scale, shift);
  return p2pvg_check_launch("bn_fwd_finalize_tiles");
}
