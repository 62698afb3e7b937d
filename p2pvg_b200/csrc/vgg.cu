// Data-movement kernels of the vgg_64 backbone (reference models/vgg_64.py): MaxPool2d(2,2), nearest x2 upsampling,
// and the explicit 3x3 / stride-1 / pad-1 lowering used by the fp32 path and by the 3-channel ends of the network
// (the >= 64-channel layers run as implicit GEMMs in conv_gemm.cu, kinds 3-5).  All tensors NHWC; HBM-bound.
#include "common.cuh"

namespace {

inline int grid_for(long long total, int block) {
  long long g = (total + block - 1) / block;
  const long long cap = 132LL * 64;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

// col[(n,y,x), tap*C + c] = x[n, y + sgn*(kh-1), x + sgn*(kw-1), c]  (zero outside the map); columns [9C, ld) = 0
template <typename T>
__global__ void im2col3_kernel(const T* __restrict__ x, T* __restrict__ col, int N, int H, int W, int C, int ld, int sgn) {
  const long long total = (long long)N * H * W * ld;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(idx % ld);
    const long long pix = idx / ld;
    float v = 0.f;
    if (j < 9 * C) {
      const int tap = j / C, c = j - tap * C;
      const int kh = tap / 3, kw = tap - kh * 3;
      const int xx = (int)(pix % W);
      const int yy = (int)((pix / W) % H);
      const long long n = pix / ((long long)W * H);
      const int sy = yy + sgn * (kh - 1), sx = xx + sgn * (kw - 1);
      if (sy >= 0 && sy < H && sx >= 0 && sx < W) v = ld_f(x + ((n * H + sy) * W + sx) * C + c);
    }
    st_f(col + idx, v);
  }
}

// y[(n,y,x), c] = bias[c] + sum_tap col[(n, y-(kh-1), x-(kw-1)), tap*C + c]     (ConvTranspose2d(k=3, s=1, p=1) scatter as a gather)
template <typename T>
__global__ void col2im3_kernel(const T* __restrict__ col, T* __restrict__ y, int N, int H, int W, int C, int ld, const float* __restrict__ bias) {
  const long long total = (long long)N * H * W * C;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % C);
    const long long pix = idx / C;
    const int xx = (int)(pix % W);
    const int yy = (int)((pix / W) % H);
    const long long n = pix / ((long long)W * H);
    float acc = bias ? bias[c] : 0.f;
#pragma unroll
    for (int kh = 0; kh < 3; kh++) {
      const int sy = yy - (kh - 1);
      if (sy < 0 || sy >= H) continue;
#pragma unroll
      for (int kw = 0; kw < 3; kw++) {
        const int sx = xx - (kw - 1);
        if (sx < 0 || sx >= W) continue;
        acc += ld_f(col + ((n * H + sy) * W + sx) * ld + (kh * 3 + kw) * C + c);
      }
    }
    st_f(y + idx, acc);
  }
}

template <typename T>
__global__ void maxpool2_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, int N, int H, int W, int C) {
  const int Ho = H / 2, Wo = W / 2;
  const long long total = (long long)N * Ho * Wo * C;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % C);
    const long long p = idx / C;
    const int xo = (int)(p % Wo), yo = (int)((p / Wo) % Ho);
    const long long n = p / ((long long)Wo * Ho);
    const T* b = x + ((n * H + 2 * yo) * W + 2 * xo) * C + c;
    const float v = fmaxf(fmaxf(ld_f(b), ld_f(b + C)), fmaxf(ld_f(b + (long long)W * C), ld_f(b + (long long)W * C + C)));
    st_f(y + idx, v);
  }
}

// gradient goes to the first maximum of each window in row-major order (torch's max_pool2d tie rule)
template <typename T>
__global__ void maxpool2_bwd_kernel(const T* __restrict__ x, const T* __restrict__ dy, T* __restrict__ dx, int N, int H, int W, int C) {
  const int Ho = H / 2, Wo = W / 2;
  const long long total = (long long)N * Ho * Wo * C;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % C);
    const long long p = idx / C;
    const int xo = (int)(p % Wo), yo = (int)((p / Wo) % Ho);
    const long long n = p / ((long long)Wo * Ho);
    const long long base = ((n * H + 2 * yo) * W + 2 * xo) * C + c;
    const long long off[4] = {0, (long long)C, (long long)W * C, (long long)W * C + C};
    int best = 0;
    float bv = ld_f(x + base);
#pragma unroll
    for (int k = 1; k < 4; k++) {
      const float v = ld_f(x + base + off[k]);
      if (v > bv) { bv = v; best = k; }
    }
    const float g = ld_f(dy + idx);
#pragma unroll
    for (int k = 0; k < 4; k++) st_f(dx + base + off[k], k == best ? g : 0.f);
  }
}

template <typename T>
__global__ void upsample2_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, int N, int H, int W, int C) {
  const int Ho = 2 * H, Wo = 2 * W;
  const long long total = (long long)N * Ho * Wo * C;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % C);
    const long long p = idx / C;
    const int xo = (int)(p % Wo), yo = (int)((p / Wo) % Ho);
    const long long n = p / ((long long)Wo * Ho);
    y[idx] = x[((n * H + (yo >> 1)) * W + (xo >> 1)) * C + c];
  }
}

template <typename T>
__global__ void upsample2_bwd_kernel(const T* __restrict__ dy, T* __restrict__ dx, int N, int H, int W, int C) {
  const long long total = (long long)N * H * W * C;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % C);
    const long long p = idx / C;
    const int xi = (int)(p % W), yi = (int)((p / W) % H);
    const long long n = p / ((long long)W * H);
    const T* b = dy + ((n * 2 * H + 2 * yi) * (2 * W) + 2 * xi) * C + c;
    const long long row = 2LL * W * C;
    st_f(dx + idx, (ld_f(b) + ld_f(b + C)) + (ld_f(b + row) + ld_f(b + row + C)));
  }
}

// ---- 16-byte-vector versions (C a multiple of the vector width, < 2^31 vectors): one thread per (pixel, channel vector),
// 32-bit index arithmetic.  The scalar kernels above remain for odd channel counts (the 1/3-channel ends).
template <typename T>
__global__ void __launch_bounds__(256) maxpool2_fwd_vec_kernel(const T* __restrict__ x, T* __restrict__ y, unsigned total, int H, int W, int CV) {
  constexpr int V = VecN<T>::N;
  const unsigned Ho = H / 2, Wo = W / 2;
  for (unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const unsigned cv = idx % CV, p = idx / CV;
    const unsigned xo = p % Wo, q = p / Wo, yo = q % Ho, n = q / Ho;
    const long long base = ((((long long)n * H + 2 * yo) * W + 2 * xo) * CV + cv) * V;
    const long long dxo = (long long)CV * V, dyo = (long long)W * CV * V;
    float a[V], b[V], c[V], d[V];
    unpack16<T>(ld_raw16(x + base), a);
    unpack16<T>(ld_raw16(x + base + dxo), b);
    unpack16<T>(ld_raw16(x + base + dyo), c);
    unpack16<T>(ld_raw16(x + base + dyo + dxo), d);
#pragma unroll
    for (int j = 0; j < V; j++) a[j] = fmaxf(fmaxf(a[j], b[j]), fmaxf(c[j], d[j]));
    st_raw16(y + (long long)idx * V, pack16<T>(a));
  }
}

template <typename T>
__global__ void __launch_bounds__(256) maxpool2_bwd_vec_kernel(const T* __restrict__ x, const T* __restrict__ dy, T* __restrict__ dx, unsigned total,
                                                               int H, int W, int CV) {
  constexpr int V = VecN<T>::N;
  const unsigned Ho = H / 2, Wo = W / 2;
  for (unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const unsigned cv = idx % CV, p = idx / CV;
    const unsigned xo = p % Wo, q = p / Wo, yo = q % Ho, n = q / Ho;
    const long long base = ((((long long)n * H + 2 * yo) * W + 2 * xo) * CV + cv) * V;
    const long long off[4] = {0, (long long)CV * V, (long long)W * CV * V, (long long)W * CV * V + (long long)CV * V};
    float v[4][V], g[V], o[4][V];
#pragma unroll
    for (int k = 0; k < 4; k++) unpack16<T>(ld_raw16(x + base + off[k]), v[k]);
    unpack16<T>(ld_raw16(dy + (long long)idx * V), g);
#pragma unroll
    for (int j = 0; j < V; j++) {   // first maximum in row-major order (torch's tie rule)
      int best = 0;
      float bv = v[0][j];
#pragma unroll
      for (int k = 1; k < 4; k++)
        if (v[k][j] > bv) { bv = v[k][j]; best = k; }
#pragma unroll
      for (int k = 0; k < 4; k++) o[k][j] = (k == best) ? g[j] : 0.f;
    }
#pragma unroll
    for (int k = 0; k < 4; k++) st_raw16(dx + base + off[k], pack16<T>(o[k]));
  }
}

// one thread per INPUT pixel vector: read once, write the 2x2 replicas
template <typename T>
__global__ void __launch_bounds__(256) upsample2_fwd_vec_kernel(const T* __restrict__ x, T* __restrict__ y, unsigned total, int H, int W, int CV) {
  constexpr int V = VecN<T>::N;
  for (unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const unsigned cv = idx % CV, p = idx / CV;
    const unsigned xi = p % W, q = p / W, yi = q % H, n = q / H;
    const uint4 v = ld_raw16(x + (long long)idx * V);
    const long long base = ((((long long)n * 2 * H + 2 * yi) * (2 * W) + 2 * xi) * CV + cv) * V;
    const long long dxo = (long long)CV * V, dyo = 2LL * W * CV * V;
    st_raw16(y + base, v);
    st_raw16(y + base + dxo, v);
    st_raw16(y + base + dyo, v);
    st_raw16(y + base + dyo + dxo, v);
  }
}

template <typename T>
__global__ void __launch_bounds__(256) upsample2_bwd_vec_kernel(const T* __restrict__ dy, T* __restrict__ dx, unsigned total, int H, int W, int CV) {
  constexpr int V = VecN<T>::N;
  for (unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const unsigned cv = idx % CV, p = idx / CV;
    const unsigned xi = p % W, q = p / W, yi = q % H, n = q / H;
    const long long base = ((((long long)n * 2 * H + 2 * yi) * (2 * W) + 2 * xi) * CV + cv) * V;
    const long long dxo = (long long)CV * V, dyo = 2LL * W * CV * V;
    float a[V], b[V], c[V], d[V];
    unpack16<T>(ld_raw16(dy + base), a);
    unpack16<T>(ld_raw16(dy + base + dxo), b);
    unpack16<T>(ld_raw16(dy + base + dyo), c);
    unpack16<T>(ld_raw16(dy + base + dyo + dxo), d);
#pragma unroll
    for (int j = 0; j < V; j++) a[j] = (a[j] + b[j]) + (c[j] + d[j]);
    st_raw16(dx + (long long)idx * V, pack16<T>(a));
  }
}

// 3x3 lowering of a few-channel map (9 C <= 32, row pitch 32): one thread per output ROW (pixel) -- 27 scalar gathers, then
// the whole 32-element row (zero padded) goes out as 16-byte vectors (the scalar kernel spent a 64-bit division per element)
template <typename T, int C>
__global__ void __launch_bounds__(256) im2col3_row32_kernel(const T* __restrict__ x, T* __restrict__ col, unsigned npix, int H, int W, int sgn) {
  constexpr int V = VecN<T>::N;
  for (unsigned pix = blockIdx.x * blockDim.x + threadIdx.x; pix < npix; pix += gridDim.x * blockDim.x) {
    const unsigned xx = pix % W, q = pix / W, yy = q % H, n = q / H;
    float row[32];
#pragma unroll
    for (int j = 0; j < 32; j++) row[j] = 0.f;
#pragma unroll
    for (int kh = 0; kh < 3; kh++) {
      const int sy = (int)yy + sgn * (kh - 1);
#pragma unroll
      for (int kw = 0; kw < 3; kw++) {
        const int sx = (int)xx + sgn * (kw - 1);
        if (sy < 0 || sy >= H || sx < 0 || sx >= W) continue;
        const T* src = x + (((long long)n * H + sy) * W + sx) * C;
#pragma unroll
        for (int c = 0; c < C; c++) row[(kh * 3 + kw) * C + c] = ld_f(src + c);
      }
    }
    T* dst = col + (long long)pix * 32;
#pragma unroll
    for (int j = 0; j < 32; j += V) st_raw16(dst + j, pack16<T>(row + j));
  }
}

// dst[g*n + i] += src[grp_src[g]*n + i]   (fp32 addend shared by the groups that reuse a skip frame)
template <typename T>
__global__ void gather_add_kernel(T* __restrict__ dst, const float* __restrict__ src, const int* __restrict__ grp_src, int G, long long n) {
  const long long total = (long long)G * n;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const long long g = idx / n, i = idx - g * n;
    st_f(dst + idx, ld_f(dst + idx) + src[(long long)grp_src[g] * n + i]);
  }
}

// 16-byte vector path: channels a multiple of the vector width, 16-byte aligned tensors, fewer than 2^31 vectors
inline bool vec_ok(int dtype, int C, long long total, const void* a, const void* b, const void* c) {
  const int V = dtype == P2PVG_BF16 ? 8 : 4;
  return C % V == 0 && total / V < (1LL << 31) &&
         ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c)) & 15) == 0;
}

}  // namespace

extern "C" int p2pvg_im2col3(const void* x, void* col, int dtype, int N, int H, int W, int C, int ld, int sgn, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  P2PVG_REQUIRE(ld >= 9 * C, P2PVG_ERR_BAD_ARG, "im2col3: ld %d < 9*C", ld);
  if (N == 0) return P2PVG_OK;
  const long long total = (long long)N * H * W * ld;
  if (ld == 32 && (C == 1 || C == 3) && (long long)N * H * W < (1LL << 31) && (reinterpret_cast<uintptr_t>(col) & 15) == 0) {
    const unsigned npix = (unsigned)((long long)N * H * W);
    const int sg = sgn < 0 ? -1 : 1;
    if (C == 3) { DISPATCH_DTYPE(dtype, T, (im2col3_row32_kernel<T, 3><<<grid_for(npix, 256), 256, 0, st>>>((const T*)x, (T*)col, npix, H, W, sg))); }
    else { DISPATCH_DTYPE(dtype, T, (im2col3_row32_kernel<T, 1><<<grid_for(npix, 256), 256, 0, st>>>((const T*)x, (T*)col, npix, H, W, sg))); }
    return p2pvg_check_launch("im2col3");
  }
  DISPATCH_DTYPE(dtype, T, (im2col3_kernel<T><<<grid_for(total, 256), 256, 0, st>>>((const T*)x, (T*)col, N, H, W, C, ld, sgn < 0 ? -1 : 1)));
  return p2pvg_check_launch("im2col3");
}

extern "C" int p2pvg_col2im3(const void* col, void* y, int dtype, int N, int H, int W, int C, int ld, const float* bias, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  P2PVG_REQUIRE(ld >= 9 * C, P2PVG_ERR_BAD_ARG, "col2im3: ld %d < 9*C", ld);
  if (N == 0) return P2PVG_OK;
  const long long total = (long long)N * H * W * C;
  DISPATCH_DTYPE(dtype, T, (col2im3_kernel<T><<<grid_for(total, 256), 256, 0, st>>>((const T*)col, (T*)y, N, H, W, C, ld, bias)));
  return p2pvg_check_launch("col2im3");
}

extern "C" int p2pvg_maxpool2_fwd(const void* x, void* y, int dtype, int N, int H, int W, int C, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  P2PVG_REQUIRE(H % 2 == 0 && W % 2 == 0, P2PVG_ERR_BAD_ARG, "maxpool2: odd map %dx%d", H, W);
  if (N == 0) return P2PVG_OK;
  const long long total = (long long)N * (H / 2) * (W / 2) * C;
  if (vec_ok(dtype, C, total, x, y, nullptr)) {
    const int V = dtype == P2PVG_BF16 ? 8 : 4;
    const unsigned tv = (unsigned)(total / V);
    DISPATCH_DTYPE(dtype, T, (maxpool2_fwd_vec_kernel<T><<<grid_for(tv, 256), 256, 0, st>>>((const T*)x, (T*)y, tv, H, W, C / V)));
    return p2pvg_check_launch("maxpool2_fwd");
  }
  DISPATCH_DTYPE(dtype, T, (maxpool2_fwd_kernel<T><<<grid_for(total, 256), 256, 0, st>>>((const T*)x, (T*)y, N, H, W, C)));
  return p2pvg_check_launch("maxpool2_fwd");
}

extern "C" int p2pvg_maxpool2_bwd(const void* x, const void* dy, void* dx, int dtype, int N, int H, int W, int C, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  P2PVG_REQUIRE(H % 2 == 0 && W % 2 == 0, P2PVG_ERR_BAD_ARG, "maxpool2: odd map %dx%d", H, W);
  if (N == 0) return P2PVG_OK;
  const long long total = (long long)N * (H / 2) * (W / 2) * C;
  if (vec_ok(dtype, C, total, x, dy, dx)) {
    const int V = dtype == P2PVG_BF16 ? 8 : 4;
    const unsigned tv = (unsigned)(total / V);
    DISPATCH_DTYPE(dtype, T, (maxpool2_bwd_vec_kernel<T><<<grid_for(tv, 256), 256, 0, st>>>((const T*)x, (const T*)dy, (T*)dx, tv, H, W, C / V)));
    return p2pvg_check_launch("maxpool2_bwd");
  }
  DISPATCH_DTYPE(dtype, T, (maxpool2_bwd_kernel<T><<<grid_for(total, 256), 256, 0, st>>>((const T*)x, (const T*)dy, (T*)dx, N, H, W, C)));
  return p2pvg_check_launch("maxpool2_bwd");
}

extern "C" int p2pvg_upsample2_fwd(const void* x, void* y, int dtype, int N, int H, int W, int C, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (N == 0) return P2PVG_OK;
  const long long total = (long long)N * 4 * H * W * C;
  if (vec_ok(dtype, C, total / 4, x, y, nullptr)) {
    const int V = dtype == P2PVG_BF16 ? 8 : 4;
    const unsigned tv = (unsigned)(total / 4 / V);
    DISPATCH_DTYPE(dtype, T, (upsample2_fwd_vec_kernel<T><<<grid_for(tv, 256), 256, 0, st>>>((const T*)x, (T*)y, tv, H, W, C / V)));
    return p2pvg_check_launch("upsample2_fwd");
  }
  DISPATCH_DTYPE(dtype, T, (upsample2_fwd_kernel<T><<<grid_for(total, 256), 256, 0, st>>>((const T*)x, (T*)y, N, H, W, C)));
  return p2pvg_check_launch("upsample2_fwd");
}

extern "C" int p2pvg_upsample2_bwd(const void* dy, void* dx, int dtype, int N, int H, int W, int C, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (N == 0) return P2PVG_OK;
  const long long total = (long long)N * H * W * C;
  if (vec_ok(dtype, C, total, dy, dx, nullptr)) {
    const int V = dtype == P2PVG_BF16 ? 8 : 4;
    const unsigned tv = (unsigned)(total / V);
    DISPATCH_DTYPE(dtype, T, (upsample2_bwd_vec_kernel<T><<<grid_for(tv, 256), 256, 0, st>>>((const T*)dy, (T*)dx, tv, H, W, C / V)));
    return p2pvg_check_launch("upsample2_bwd");
  }
  DISPATCH_DTYPE(dtype, T, (upsample2_bwd_kernel<T><<<grid_for(total, 256), 256, 0, st>>>((const T*)dy, (T*)dx, N, H, W, C)));
  return p2pvg_check_launch("upsample2_bwd");
}

extern "C" int p2pvg_gather_add(void* dst, int dtype, const float* src, const int* grp_src, int G, int64_t n, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (G == 0 || n == 0) return P2PVG_OK;
  DISPATCH_DTYPE(dtype, T, (gather_add_kernel<T><<<grid_for((long long)G * n, 256), 256, 0, st>>>((T*)dst, src, grp_src, G, n)));
  return p2pvg_check_launch("gather_add");
}
