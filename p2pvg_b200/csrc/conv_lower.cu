// Lowering kernels that turn the dcgan 4x4/stride-2/pad-1 (transposed) convolutions into GEMMs on
// NHWC activations, plus the small layout utilities (permute / cast / indexed add / segment sum).
// All of them are HBM-bound streaming kernels: one thread per 4 channels, fully coalesced on the
// channel axis.
#include "common.cuh"

namespace {

// ---- im2col: x [N,H,W,C] -> col [N*(H/2)*(W/2), 16*C], K order (kh, kw, c) ----------------------
// 16-byte vectors (8 bf16 / 4 fp32), four independent copies in flight per thread.
template <typename T>
__global__ void __launch_bounds__(256) im2col_vec_kernel(const T* __restrict__ x, T* __restrict__ col, int N, int H, int W, int C) {
  constexpr int V = VecN<T>::N;
  const int Ho = H >> 1, Wo = W >> 1, CV = C / V;
  const long long total = (long long)N * Ho * Wo * 16 * CV;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long base = (long long)blockIdx.x * blockDim.x + threadIdx.x; base < total; base += 4 * stride) {
    uint4 v[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const long long idx = base + u * stride;
      v[u] = make_uint4(0u, 0u, 0u, 0u);
      if (idx < total) {
        const int cv = (int)(idx % CV);
        const long long r = idx / CV;
        const int tap = (int)(r & 15);
        const long long row = r >> 4;
        const int ox = (int)(row % Wo);
        const long long t = row / Wo;
        const int oy = (int)(t % Ho);
        const int n = (int)(t / Ho);
        const int iy = 2 * oy - 1 + (tap >> 2), ix = 2 * ox - 1 + (tap & 3);
        if (iy >= 0 && iy < H && ix >= 0 && ix < W) v[u] = ld_raw16(x + (((long long)n * H + iy) * W + ix) * C + cv * V);
      }
    }
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const long long idx = base + u * stride;
      if (idx < total) st_raw16(col + idx * V, v[u]);
    }
  }
}

template <typename T>
__global__ void im2col_scalar_kernel(const T* __restrict__ x, T* __restrict__ col, int N, int H, int W, int C) {
  const int Ho = H >> 1, Wo = W >> 1;
  const long long total = (long long)N * Ho * Wo * 16 * C;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    int c = (int)(idx % C);
    long long r = idx / C;
    int tap = (int)(r & 15);
    long long row = r >> 4;
    int ox = (int)(row % Wo);
    long long t = row / Wo;
    int oy = (int)(t % Ho);
    int n = (int)(t / Ho);
    int iy = 2 * oy - 1 + (tap >> 2), ix = 2 * ox - 1 + (tap & 3);
    bool ok = (iy >= 0 && iy < H && ix >= 0 && ix < W);
    st_f<T>(col + idx, ok ? ld_f<T>(x + (((long long)n * H + iy) * W + ix) * C + c) : 0.f);
  }
}

// 1..4 channel images (the first encoder layer, the data gradient of the last decoder layer): one thread per
// (output pixel, kh) copies the 4*C contiguous input elements of that filter row with vector stores
template <typename T, int C>
__global__ void __launch_bounds__(256) im2col_smallc_kernel(const T* __restrict__ x, T* __restrict__ col, int N, int H, int W) {
  const int Ho = H >> 1, Wo = W >> 1;
  const long long total = (long long)N * Ho * Wo * 4;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int kh = (int)(idx & 3);
    const long long row = idx >> 2;
    const int ox = (int)(row % Wo);
    const long long t = row / Wo;
    const int oy = (int)(t % Ho);
    const long long n = t / Ho;
    const int iy = 2 * oy - 1 + kh, ix0 = 2 * ox - 1;
    float v[4 * C];
    const bool yok = (iy >= 0 && iy < H);
    const T* src = x + ((n * H + (yok ? iy : 0)) * W) * C;
#pragma unroll
    for (int kw = 0; kw < 4; kw++) {
      const int ix = ix0 + kw;
      const bool ok = yok && ix >= 0 && ix < W;
#pragma unroll
      for (int c = 0; c < C; c++) v[kw * C + c] = ok ? ld_f<T>(src + (long long)ix * C + c) : 0.f;
    }
    T* dst = col + idx * (4 * C);
    if (sizeof(T) == 2) {
#pragma unroll
      for (int j = 0; j < C; j++) {  // 4 bf16 = 8 bytes per store
        __nv_bfloat162 p0 = __floats2bfloat162_rn(v[4 * j], v[4 * j + 1]), p1 = __floats2bfloat162_rn(v[4 * j + 2], v[4 * j + 3]);
        uint2 pk;
        pk.x = *reinterpret_cast<uint32_t*>(&p0);
        pk.y = *reinterpret_cast<uint32_t*>(&p1);
        *reinterpret_cast<uint2*>(reinterpret_cast<bf16*>(dst) + 4 * j) = pk;
      }
    } else {
#pragma unroll
      for (int j = 0; j < C; j++)
        *reinterpret_cast<float4*>(reinterpret_cast<float*>(dst) + 4 * j) = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
    }
  }
}

// ---- col2im (gather form): y [N,2Hi,2Wi,C] <- col [N*Hi*Wi, 16*C] (+ col2 of a shared source) ----
template <typename T, int V>
__global__ void __launch_bounds__(256) col2im_k4s2p1_kernel(const T* __restrict__ col, const T* __restrict__ col2,
                                                            const int* __restrict__ grp_src, int imgs_per_group, T* __restrict__ y,
                                                            int N, int Hi, int Wi, int C, const float* __restrict__ bias, int accumulate) {
  const int Ho = Hi * 2, Wo = Wi * 2, CV = C / V;
  const long long total = (long long)N * Ho * Wo * CV;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(idx % CV);
    const long long p = idx / CV;
    const int ox = (int)(p % Wo);
    const long long t = p / Wo;
    const int oy = (int)(t % Ho);
    const int n = (int)(t / Ho);
    int n2 = 0;
    if (col2) n2 = grp_src[n / imgs_per_group] * imgs_per_group + (n % imgs_per_group);
    float acc[V];
#pragma unroll
    for (int j = 0; j < V; j++) acc[j] = bias ? bias[cv * V + j] : 0.f;
    const int kh0 = (oy + 1) & 1, kw0 = (ox + 1) & 1;
    // gather the (up to) 2x2 contributing taps; issue all loads first
    uint4 raw[8];
    bool on[4];
#pragma unroll
    for (int a = 0; a < 2; a++) {
#pragma unroll
      for (int b = 0; b < 2; b++) {
        const int kh = kh0 + 2 * a, kw = kw0 + 2 * b;
        const int ty = oy + 1 - kh, tx = ox + 1 - kw;
        const int iy = ty >> 1, ix = tx >> 1;
        const bool ok = (ty >= 0) && (iy < Hi) && (tx >= 0) && (ix < Wi);
        on[a * 2 + b] = ok;
        if (V > 1) {
          raw[a * 2 + b] = make_uint4(0u, 0u, 0u, 0u);
          raw[4 + a * 2 + b] = make_uint4(0u, 0u, 0u, 0u);
        }
        if (!ok) continue;
        const long long off = ((((long long)n * Hi + iy) * Wi + ix) * 16 + kh * 4 + kw) * C + cv * V;
        if (V > 1) {
          raw[a * 2 + b] = ld_raw16(col + off);
          if (col2) raw[4 + a * 2 + b] = ld_raw16(col2 + ((((long long)n2 * Hi + iy) * Wi + ix) * 16 + kh * 4 + kw) * C + cv * V);
        } else {
          acc[0] += ld_f<T>(col + off);
          if (col2) acc[0] += ld_f<T>(col2 + ((((long long)n2 * Hi + iy) * Wi + ix) * 16 + kh * 4 + kw) * C + cv * V);
        }
      }
    }
    T* dst = y + p * C + cv * V;
    if (V > 1) {
#pragma unroll
      for (int q = 0; q < 4; q++) {
        if (!on[q]) continue;
        float f[V > 1 ? V : 8];
        unpack16<T>(raw[q], f);
#pragma unroll
        for (int j = 0; j < V; j++) acc[j] += f[j];
        if (col2) {
          unpack16<T>(raw[4 + q], f);
#pragma unroll
          for (int j = 0; j < V; j++) acc[j] += f[j];
        }
      }
      if (accumulate) {
        float f[V > 1 ? V : 8];
        unpack16<T>(ld_raw16(dst), f);
#pragma unroll
        for (int j = 0; j < V; j++) acc[j] += f[j];
      }
      st_raw16(dst, pack16<T>(acc));
    } else {
      st_f<T>(dst, accumulate ? ld_f<T>(dst) + acc[0] : acc[0]);
    }
  }
}

// ---- generic 4-D permute / cast: dst (contiguous, dims d[0..3]) <- src with per-dst-dim strides ---
struct Perm4 {
  int d[4];
  long long s[4];
};
template <typename TS, typename TD>
__global__ void permute4_kernel(const TS* __restrict__ src, TD* __restrict__ dst, Perm4 p, int accumulate) {
  const long long total = (long long)p.d[0] * p.d[1] * p.d[2] * p.d[3];
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    long long r = idx;
    int i3 = (int)(r % p.d[3]); r /= p.d[3];
    int i2 = (int)(r % p.d[2]); r /= p.d[2];
    int i1 = (int)(r % p.d[1]); r /= p.d[1];
    int i0 = (int)r;
    float v = ld_f<TS>(src + i0 * p.s[0] + i1 * p.s[1] + i2 * p.s[2] + i3 * p.s[3]);
    if (accumulate) v += ld_f<TD>(dst + idx);
    st_f<TD>(dst + idx, v);
  }
}

// flat copy / cast (permute4 with one contiguous dimension): 4 elements per thread, 16-byte accesses on the wider side
template <typename TS, typename TD>
__global__ void __launch_bounds__(256) cast_flat4_kernel(const TS* __restrict__ src, TD* __restrict__ dst, long long n4) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const f4 v = ld_f4<TS>(src + i * 4);
    st_f4<TD>(dst + i * 4, v);
  }
}

// ---- frames NCHW fp32 -> NHWC, both precisions from one read: the fp32 copy is the MSE target, the activation-dtype copy
// feeds the first convolution.  One thread = 4 consecutive pixels of one frame: C float4 plane loads (coalesced per
// plane), 4*C contiguous outputs.
template <int C, typename TA>
__global__ void __launch_bounds__(256) nchw_to_nhwc_dual_kernel(const float* __restrict__ src, float* __restrict__ dst32,
                                                                TA* __restrict__ dsta, long long N, int hw4) {
  const long long total = N * hw4;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const long long n = idx / hw4;
    const int p4 = (int)(idx - n * hw4);
    const float* s = src + (n * C * hw4 + p4) * 4;
    float v[C][4];
#pragma unroll
    for (int c = 0; c < C; c++) {
      const float4 t = *reinterpret_cast<const float4*>(s + (long long)c * hw4 * 4);
      v[c][0] = t.x; v[c][1] = t.y; v[c][2] = t.z; v[c][3] = t.w;
    }
    float o[4 * C];
#pragma unroll
    for (int q = 0; q < 4; q++)
#pragma unroll
      for (int c = 0; c < C; c++) o[q * C + c] = v[c][q];
    const long long ob = idx * 4 * C;
    if (dst32) {
#pragma unroll
      for (int j = 0; j < C; j++) *reinterpret_cast<float4*>(dst32 + ob + 4 * j) = make_float4(o[4 * j], o[4 * j + 1], o[4 * j + 2], o[4 * j + 3]);
    }
    if (dsta) {
      if constexpr (sizeof(TA) == 2) {   // 4*C bf16 = C 8-byte stores
#pragma unroll
        for (int j = 0; j < C; j++) {
          const __nv_bfloat162 lo = __floats2bfloat162_rn(o[4 * j], o[4 * j + 1]), hi = __floats2bfloat162_rn(o[4 * j + 2], o[4 * j + 3]);
          uint2 u;
          u.x = *reinterpret_cast<const unsigned*>(&lo);
          u.y = *reinterpret_cast<const unsigned*>(&hi);
          *reinterpret_cast<uint2*>(dsta + ob + 4 * j) = u;
        }
      } else {
#pragma unroll
        for (int j = 0; j < C; j++)
          *reinterpret_cast<float4*>(dsta + ob + 4 * j) = make_float4(o[4 * j], o[4 * j + 1], o[4 * j + 2], o[4 * j + 3]);
      }
    }
  }
}

// ---- dst[dst_idx[f]] += src[f] over F groups of n elements -------------------------------------
template <typename T>
__global__ void add_indexed_kernel(T* __restrict__ dst, const T* __restrict__ src, const int* __restrict__ dst_idx, int F, long long n) {
  const long long total = (long long)F * n;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    int f = (int)(idx / n);
    long long j = idx - (long long)f * n;
    T* d = dst + (long long)dst_idx[f] * n + j;
    st_f<T>(d, ld_f<T>(d) + ld_f<T>(src + idx));
  }
}

// ---- out[f] = sum over groups g with src[g]==f of in[g]  (n elements per group, n % 4 == 0) -----
template <typename T>
__global__ void group_sum_kernel(const T* __restrict__ in, T* __restrict__ out, const int* __restrict__ grp_src, int G, int F, long long n4) {
  const long long total = (long long)F * n4;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    int f = (int)(idx / n4);
    long long j = idx - (long long)f * n4;
    f4 acc = {{0.f, 0.f, 0.f, 0.f}};
    for (int g = 0; g < G; g++) {
      if (grp_src[g] != f) continue;
      f4 v = ld_f4<T>(in + ((long long)g * n4 + j) * 4);
#pragma unroll
      for (int q = 0; q < 4; q++) acc.v[q] += v.v[q];
    }
    st_f4<T>(out + idx * 4, acc);
  }
}

// dst[(gi,r), (gj,c)] = (gi == gj) ? src[r, c] : 0   -- g copies of a small weight matrix on the diagonal, so that g
// consecutive rows of a thin [M, C] operand can be multiplied as one [M/g, g*C] row without out-of-bounds TMA boxes
template <typename TS, typename TD>
__global__ void blockdiag_kernel(const TS* __restrict__ src, TD* __restrict__ dst, int R, int C, int g) {
  const long long total = (long long)g * R * g * C;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % C);
    long long t = idx / C;
    const int gj = (int)(t % g);
    t /= g;
    const int r = (int)(t % R);
    const int gi = (int)(t / R);
    st_f<TD>(dst + idx, gi == gj ? ld_f<TS>(src + (long long)r * C + c) : 0.f);
  }
}

// batched 2-D transpose  dst[a][q][p] = src[a][p][q]  through a 32x33 shared-memory tile: both the reads and the writes
// are coalesced.  Packs conv weights W[Cout][Cin][taps] -> [Cout][taps][Cin] (and back for the weight gradients), where
// the generic strided gather of permute4 touches one 4-byte element per 64-byte segment.
template <typename TS, typename TD>
__global__ void __launch_bounds__(256) transpose_batched_kernel(const TS* __restrict__ src, TD* __restrict__ dst, int P, int Q) {
  __shared__ float tile[32][33];
  const long long a = blockIdx.z;
  const int p0 = blockIdx.y * 32, q0 = blockIdx.x * 32;
  const TS* s = src + a * P * Q;
  TD* d = dst + a * P * Q;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8
#pragma unroll
  for (int i = 0; i < 32; i += 8) {
    const int p = p0 + ty + i, q = q0 + tx;
    if (p < P && q < Q) tile[ty + i][tx] = ld_f<TS>(s + (long long)p * Q + q);
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 32; i += 8) {
    const int q = q0 + ty + i, pp = p0 + tx;
    if (q < Q && pp < P) st_f<TD>(d + (long long)q * P + pp, tile[tx][ty + i]);
  }
}

inline int grid_for(long long total, int block) {
  long long g = (total + block - 1) / block;
  const long long cap = 132LL * 64;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace

extern "C" int p2pvg_im2col_k4s2p1(const void* x, void* col, int dtype, int N, int H, int W, int C, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  P2PVG_REQUIRE((H % 2 == 0) && (W % 2 == 0), P2PVG_ERR_BAD_ARG, "im2col: odd spatial size %dx%d", H, W);
  if (N == 0) return P2PVG_OK;
  const int vec = (dtype == P2PVG_BF16) ? 8 : 4;
  const bool aligned = ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(col)) & 15) == 0;
  if (C % vec == 0 && aligned) {
    long long total = (long long)N * (H / 2) * (W / 2) * 16 * (C / vec);
    DISPATCH_DTYPE(dtype, T, (im2col_vec_kernel<T><<<grid_for((total + 3) / 4, 256), 256, 0, st>>>((const T*)x, (T*)col, N, H, W, C)));
  } else if (C <= 4 && (reinterpret_cast<uintptr_t>(col) & 15) == 0) {
    long long total = (long long)N * (H / 2) * (W / 2) * 4;
#define P2PVG_SMALLC(CC) DISPATCH_DTYPE(dtype, T, (im2col_smallc_kernel<T, CC><<<grid_for(total, 256), 256, 0, st>>>((const T*)x, (T*)col, N, H, W)))
    if (C == 1) P2PVG_SMALLC(1);
    else if (C == 2) P2PVG_SMALLC(2);
    else if (C == 3) P2PVG_SMALLC(3);
    else P2PVG_SMALLC(4);
#undef P2PVG_SMALLC
  } else {
    long long total = (long long)N * (H / 2) * (W / 2) * 16 * C;
    DISPATCH_DTYPE(dtype, T, (im2col_scalar_kernel<T><<<grid_for(total, 256), 256, 0, st>>>((const T*)x, (T*)col, N, H, W, C)));
  }
  return p2pvg_check_launch("im2col_k4s2p1");
}

extern "C" int p2pvg_col2im_k4s2p1(const void* col, const void* col2, const int* grp_src, int imgs_per_group, void* y, int dtype, int N,
                                   int Hi, int Wi, int C, const float* bias, int accumulate, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (N == 0) return P2PVG_OK;
  P2PVG_REQUIRE(col2 == nullptr || (grp_src != nullptr && imgs_per_group > 0), P2PVG_ERR_BAD_ARG, "col2im: col2 needs grp_src");
  const int vec = (dtype == P2PVG_BF16) ? 8 : 4;
  const bool aligned = ((reinterpret_cast<uintptr_t>(col) | reinterpret_cast<uintptr_t>(col2) | reinterpret_cast<uintptr_t>(y)) & 15) == 0;
  if (C % vec == 0 && aligned) {
    long long total = (long long)N * Hi * 2 * Wi * 2 * (C / vec);
    if (dtype == P2PVG_BF16)
      col2im_k4s2p1_kernel<bf16, 8><<<grid_for(total, 256), 256, 0, st>>>((const bf16*)col, (const bf16*)col2, grp_src, imgs_per_group,
                                                                          (bf16*)y, N, Hi, Wi, C, bias, accumulate);
    else
      col2im_k4s2p1_kernel<float, 4><<<grid_for(total, 256), 256, 0, st>>>((const float*)col, (const float*)col2, grp_src,
                                                                           imgs_per_group, (float*)y, N, Hi, Wi, C, bias, accumulate);
  } else {
    long long total = (long long)N * Hi * 2 * Wi * 2 * C;
    DISPATCH_DTYPE(dtype, T, (col2im_k4s2p1_kernel<T, 1><<<grid_for(total, 256), 256, 0, st>>>(
                                 (const T*)col, (const T*)col2, grp_src, imgs_per_group, (T*)y, N, Hi, Wi, C, bias, accumulate)));
  }
  return p2pvg_check_launch("col2im_k4s2p1");
}

extern "C" int p2pvg_permute4(const void* src, int src_dtype, void* dst, int dst_dtype, const int* dims, const int64_t* src_strides,
                              int accumulate, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  Perm4 p;
  long long total = 1;
  for (int i = 0; i < 4; i++) {
    p.d[i] = dims[i];
    p.s[i] = src_strides[i];
    total *= dims[i];
  }
  if (total == 0) return P2PVG_OK;
  // the frequent special case "cast a contiguous buffer" (e.g. the bf16 operand copies of the LSTM weight-gradient GEMMs)
  // (any gather whose source strides are those of a contiguous tensor of the same dims, size-1 dims ignored)
  bool dense = true;
  long long expect = 1;
  for (int i = 3; i >= 0; i--) {
    if (p.d[i] == 1) continue;
    if (p.s[i] != expect) dense = false;
    expect *= p.d[i];
  }
  const bool flat = dense && !accumulate && total % 4 == 0 &&
                    (reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) % 16 == 0;
  if (flat) {
    const long long n4 = total / 4;
    const int gf = grid_for(n4, 256);
#define LF(TS, TD) cast_flat4_kernel<TS, TD><<<gf, 256, 0, st>>>((const TS*)src, (TD*)dst, n4)
    if (src_dtype == P2PVG_F32 && dst_dtype == P2PVG_F32) LF(float, float);
    else if (src_dtype == P2PVG_F32 && dst_dtype == P2PVG_BF16) LF(float, bf16);
    else if (src_dtype == P2PVG_BF16 && dst_dtype == P2PVG_F32) LF(bf16, float);
    else if (src_dtype == P2PVG_BF16 && dst_dtype == P2PVG_BF16) LF(bf16, bf16);
    else {
      p2pvg_set_error("permute4: bad dtypes");
      return P2PVG_ERR_BAD_ARG;
    }
#undef LF
    return p2pvg_check_launch("permute4 (flat)");
  }
  int g = grid_for(total, 256);
#define L(TS, TD) permute4_kernel<TS, TD><<<g, 256, 0, st>>>((const TS*)src, (TD*)dst, p, accumulate)
  if (src_dtype == P2PVG_F32 && dst_dtype == P2PVG_F32) L(float, float);
  else if (src_dtype == P2PVG_F32 && dst_dtype == P2PVG_BF16) L(float, bf16);
  else if (src_dtype == P2PVG_BF16 && dst_dtype == P2PVG_F32) L(bf16, float);
  else if (src_dtype == P2PVG_BF16 && dst_dtype == P2PVG_BF16) L(bf16, bf16);
  else {
    p2pvg_set_error("permute4: bad dtypes");
    return P2PVG_ERR_BAD_ARG;
  }
#undef L
  return p2pvg_check_launch("permute4");
}

extern "C" int p2pvg_nchw_to_nhwc_dual(const float* src, float* dst32, void* dsta, int act_dtype, int64_t N, int hw, int C, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (N == 0) return P2PVG_OK;
  if (hw % 4 != 0 || (C != 2 && C != 3 && C != 4) || (!dst32 && !dsta)) {
    p2pvg_set_error("nchw_to_nhwc_dual: needs H*W % 4 == 0, C in {2,3,4} and at least one destination");
    return P2PVG_ERR_UNSUPPORTED;
  }
  const int hw4 = hw / 4;
  const int g = grid_for(N * hw4, 256);
#define L(CC, TA) nchw_to_nhwc_dual_kernel<CC, TA><<<g, 256, 0, st>>>(src, dst32, (TA*)dsta, N, hw4)
#define LC(TA) do { if (C == 2) L(2, TA); else if (C == 3) L(3, TA); else L(4, TA); } while (0)
  if (!dsta || act_dtype == P2PVG_F32) LC(float);
  else if (act_dtype == P2PVG_BF16) LC(bf16);
  else {
    p2pvg_set_error("nchw_to_nhwc_dual: bad activation dtype");
    return P2PVG_ERR_BAD_ARG;
  }
#undef LC
#undef L
  return p2pvg_check_launch("nchw_to_nhwc_dual");
}

extern "C" int p2pvg_add_indexed(void* dst, const void* src, int dtype, const int* dst_idx, int F, int64_t n, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (F == 0 || n == 0) return P2PVG_OK;
  DISPATCH_DTYPE(dtype, T, (add_indexed_kernel<T><<<grid_for((long long)F * n, 256), 256, 0, st>>>((T*)dst, (const T*)src, dst_idx, F, n)));
  return p2pvg_check_launch("add_indexed");
}

extern "C" int p2pvg_transpose_batched(const void* src, int src_dtype, void* dst, int dst_dtype, int A, int P, int Q, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  P2PVG_REQUIRE(A > 0 && P > 0 && Q > 0 && A <= 65535, P2PVG_ERR_BAD_ARG, "transpose_batched: bad shape %d x %d x %d", A, P, Q);
  dim3 grid(cdiv(Q, 32), cdiv(P, 32), A);
  if (src_dtype == P2PVG_F32 && dst_dtype == P2PVG_F32) transpose_batched_kernel<float, float><<<grid, 256, 0, st>>>((const float*)src, (float*)dst, P, Q);
  else if (src_dtype == P2PVG_F32 && dst_dtype == P2PVG_BF16) transpose_batched_kernel<float, bf16><<<grid, 256, 0, st>>>((const float*)src, (bf16*)dst, P, Q);
  else if (src_dtype == P2PVG_BF16 && dst_dtype == P2PVG_BF16) transpose_batched_kernel<bf16, bf16><<<grid, 256, 0, st>>>((const bf16*)src, (bf16*)dst, P, Q);
  else {
    p2pvg_set_error("transpose_batched: unsupported dtype pair %d -> %d", src_dtype, dst_dtype);
    return P2PVG_ERR_BAD_ARG;
  }
  return p2pvg_check_launch("transpose_batched");
}

extern "C" int p2pvg_blockdiag(const void* src, int src_dtype, void* dst, int dst_dtype, int R, int C, int g, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  P2PVG_REQUIRE(R > 0 && C > 0 && g > 0, P2PVG_ERR_BAD_ARG, "blockdiag: bad shape");
  const long long total = (long long)g * R * g * C;
  const int grid = grid_for(total, 256);
  if (src_dtype == P2PVG_F32 && dst_dtype == P2PVG_F32) blockdiag_kernel<float, float><<<grid, 256, 0, st>>>((const float*)src, (float*)dst, R, C, g);
  else if (src_dtype == P2PVG_F32 && dst_dtype == P2PVG_BF16) blockdiag_kernel<float, bf16><<<grid, 256, 0, st>>>((const float*)src, (bf16*)dst, R, C, g);
  else if (src_dtype == P2PVG_BF16 && dst_dtype == P2PVG_BF16) blockdiag_kernel<bf16, bf16><<<grid, 256, 0, st>>>((const bf16*)src, (bf16*)dst, R, C, g);
  else {
    p2pvg_set_error("blockdiag: unsupported dtype pair %d -> %d", src_dtype, dst_dtype);
    return P2PVG_ERR_BAD_ARG;
  }
  return p2pvg_check_launch("blockdiag");
}

extern "C" int p2pvg_group_sum(const void* in, void* out, int dtype, const int* grp_src, int G, int F, int64_t n, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  P2PVG_REQUIRE(n % 4 == 0, P2PVG_ERR_BAD_ARG, "group_sum: n must be a multiple of 4");
  if (F == 0 || n == 0) return P2PVG_OK;
  DISPATCH_DTYPE(dtype, T, (group_sum_kernel<T><<<grid_for((long long)F * (n / 4), 256), 256, 0, st>>>((const T*)in, (T*)out, grp_src, G, F, n / 4)));
  return p2pvg_check_launch("group_sum");
}
