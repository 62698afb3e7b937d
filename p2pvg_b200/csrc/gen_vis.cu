// Composition of the pictures of the reference's generate.py (:117-163) for every output length in one launch: one CTA per
// tile gathers one source frame (or zeros) and writes it, with its control-point border, at (y, x) of one destination
// image -- an fp32 [3][h][w] canvas (the PNGs) or uint8 [h][w][3] frames (the GIFs; a stack of GIF frames is one image of
// their summed height).  The host plans the tiles (p2pvg_b200.generate.plan_video), so the kernel holds no layout rule.
// Every value is a copy, a border constant or vis_to_u8 of one, so the pictures are bit-identical to the reference's
// composition of the same frames.
#include "common.cuh"
#include "vis_common.cuh"

#define GV_THREADS 256

namespace {

__global__ void __launch_bounds__(GV_THREADS) gen_vis_kernel(const float* __restrict__ s0, const float* __restrict__ s1,
                                                              const int64_t* __restrict__ images,
                                                              const int32_t* __restrict__ tiles, int C, int H,
                                                              float* __restrict__ out_f, uint8_t* __restrict__ out_u8) {
  const int32_t* tl = tiles + 6 * (size_t)blockIdx.x;
  const int src = tl[0], idx = tl[1], border = tl[2], img = tl[3], y0 = tl[4], x0 = tl[5];
  const long long off = images[4 * img], kind = images[4 * img + 1], h = images[4 * img + 2], w = images[4 * img + 3];
  const int W = H, HW = H * W;
  const float* f = idx < 0 ? nullptr : (src == 0 ? s0 : s1) + (size_t)idx * C * HW;
  const float bc[3] = {vis_border_value(border, 0), vis_border_value(border, 1), vis_border_value(border, 2)};
  for (int p = threadIdx.x; p < HW; p += GV_THREADS) {
    const int y = p / W, x = p - y * W;
    const bool edge = vis_is_edge(border, y, x, W);
    const long long q = (long long)(y0 + y) * w + x0 + x;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float v = edge ? bc[c] : (f ? f[(C == 1 ? 0 : c) * HW + p] : 0.f);
      if (kind == 0)
        out_f[off + c * h * w + q] = v;
      else
        out_u8[off + q * 3 + c] = vis_to_u8(v);
    }
  }
}

}  // namespace

int p2pvg_vis_tiles_impl(const float* store0, int n0, const float* store1, int n1, int C, int H, const int32_t* tiles_host,
                         int n_tiles, const int64_t* images_host, int n_images, void* tables_dev, float* out_f, long long n_f,
                         uint8_t* out_u8, long long n_u8, cudaStream_t st) {
  P2PVG_REQUIRE(tiles_host && images_host && tables_dev, P2PVG_ERR_BAD_ARG, "vis_tiles: null table");
  P2PVG_REQUIRE(((uintptr_t)tables_dev & 7) == 0, P2PVG_ERR_BAD_ARG, "vis_tiles: tables_dev not 8-byte aligned");
  P2PVG_REQUIRE(C == 1 || C == 3, P2PVG_ERR_BAD_ARG, "vis_tiles: C = %d (needs 1 or 3)", C);
  P2PVG_REQUIRE(H >= 1 && H <= VIS_MAX_W, P2PVG_ERR_BAD_ARG, "vis_tiles: H = W = %d (needs 1..%d)", H, VIS_MAX_W);
  P2PVG_REQUIRE(n_tiles >= 0 && n_images >= 1 && n0 >= 0 && n1 >= 0 && n_f >= 0 && n_u8 >= 0, P2PVG_ERR_BAD_ARG,
                "vis_tiles: n_tiles = %d, n_images = %d, n0 = %d, n1 = %d", n_tiles, n_images, n0, n1);
  P2PVG_REQUIRE((n0 == 0 || store0) && (n1 == 0 || store1) && (n_f == 0 || out_f) && (n_u8 == 0 || out_u8), P2PVG_ERR_BAD_ARG,
                "vis_tiles: null frame store or output");
  P2PVG_REQUIRE((long long)(n0 > n1 ? n0 : n1) * C * H * H < (1LL << 40), P2PVG_ERR_UNSUPPORTED, "vis_tiles: stores too large");
  for (int i = 0; i < n_images; ++i) {
    const long long off = images_host[4 * i], kind = images_host[4 * i + 1], h = images_host[4 * i + 2],
                    w = images_host[4 * i + 3];
    const long long n = kind == 0 ? n_f : n_u8;
    // h, w < 2^20: 3 h w < 2^42 cannot overflow
    P2PVG_REQUIRE((kind == 0 || kind == 1) && off >= 0 && off <= n && h >= 1 && w >= 1 && h < (1LL << 20) && w < (1LL << 20) &&
                      3 * h * w <= n - off,
                  P2PVG_ERR_BAD_ARG, "vis_tiles: image %d = (offset %lld, kind %lld, %lld x %lld) outside its output (%lld values)",
                  i, off, kind, h, w, n);
  }
  for (int k = 0; k < n_tiles; ++k) {
    const int32_t* t = tiles_host + 6 * (size_t)k;
    const int src = t[0], idx = t[1], border = t[2], img = t[3], y = t[4], x = t[5];
    const int n = src == 0 ? n0 : n1;
    P2PVG_REQUIRE((src == 0 || src == 1) && idx >= -1 && idx < n && border >= 0 && border <= 2 && img >= 0 && img < n_images,
                  P2PVG_ERR_BAD_ARG, "vis_tiles: tile %d = (store %d, frame %d, border %d, image %d) out of range (store 0 has %d "
                  "frames, store 1 %d, %d images)", k, src, idx, border, img, n0, n1, n_images);
    P2PVG_REQUIRE(y >= 0 && x >= 0 && y + H <= images_host[4 * img + 2] && x + H <= images_host[4 * img + 3], P2PVG_ERR_BAD_ARG,
                  "vis_tiles: tile %d at (%d, %d) does not fit image %d", k, y, x, img);
  }
  if (n_tiles == 0) return P2PVG_OK;
  int64_t* img_dev = (int64_t*)tables_dev;
  int32_t* tiles_dev = (int32_t*)(img_dev + 4 * (size_t)n_images);
  cudaError_t e = cudaMemcpyAsync(img_dev, images_host, (size_t)n_images * 4 * sizeof(int64_t), cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess)
    e = cudaMemcpyAsync(tiles_dev, tiles_host, (size_t)n_tiles * 6 * sizeof(int32_t), cudaMemcpyHostToDevice, st);
  if (e != cudaSuccess) {
    p2pvg_set_error("vis_tiles: table copy: %s", cudaGetErrorString(e));
    return P2PVG_ERR_CUDA;
  }
  gen_vis_kernel<<<n_tiles, GV_THREADS, 0, st>>>(store0, store1, img_dev, tiles_dev, C, H, out_f, out_u8);
  return p2pvg_check_launch("vis_tiles");
}
