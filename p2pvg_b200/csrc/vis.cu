// Composition of the reference's qualitative pictures (misc/visualize.py:13-87, 176-261) from generated frames: one CTA per
// tile (frame t, row block i, row j) gathers its source frame and writes it, with the control-point border, to the PNG
// canvas, the TensorBoard video tensor and the uint8 GIF frames.  Every output value is a copy, a border constant or a
// truncation of v * 255 in fp32, so the three outputs are bit-identical to the reference's torch / NumPy composition of the
// same frames.
#include "common.cuh"
#include "vis_common.cuh"

#define VIS_THREADS 256
#define VIS_ROWS 6          // rows per block: the ground truth and five samples (misc/visualize.py:105)

namespace {

__global__ void __launch_bounds__(VIS_THREADS) vis_canvas_kernel(const float* __restrict__ s0, const float* __restrict__ s1,
                                                                  const int32_t* __restrict__ tiles, int C, int H, int r_len,
                                                                  int n_block, float* __restrict__ canvas,
                                                                  float* __restrict__ video, uint8_t* __restrict__ gif) {
  const int tile = blockIdx.x;                      // (t * n_block + i) * VIS_ROWS + j
  const int j = tile % VIS_ROWS, i = (tile / VIS_ROWS) % n_block, t = tile / (VIS_ROWS * n_block);
  const int src = tiles[3 * tile], idx = tiles[3 * tile + 1], border = tiles[3 * tile + 2];
  const int W = H, HW = H * W;
  const float* f = idx < 0 ? nullptr : (src == 0 ? s0 : s1) + (size_t)idx * C * HW;
  const float bc[3] = {vis_border_value(border, 0), vis_border_value(border, 1), vis_border_value(border, 2)};
  const size_t cw = (size_t)r_len * W, ch = (size_t)n_block * VIS_ROWS * H;   // PNG canvas [3][ch][cw]
  const size_t vw = (size_t)VIS_ROWS * W, vh = (size_t)n_block * H;           // video / GIF frame [3][vh][vw]
  float* cv = canvas + (size_t)(i * VIS_ROWS + j) * H * cw + (size_t)t * W;
  float* vd = video + (size_t)t * 3 * vh * vw + (size_t)i * H * vw + (size_t)j * W;
  uint8_t* gf = gif + ((size_t)t * vh * vw + (size_t)i * H * vw + (size_t)j * W) * 3;
  for (int p = threadIdx.x; p < HW; p += VIS_THREADS) {
    const int y = p / W, x = p - y * W;
    const bool edge = vis_is_edge(border, y, x, W);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float v = edge ? bc[c] : (f ? f[(C == 1 ? 0 : c) * HW + p] : 0.f);
      cv[c * ch * cw + (size_t)y * cw + x] = v;
      vd[c * vh * vw + (size_t)y * vw + x] = v;
      gf[((size_t)y * vw + x) * 3 + c] = vis_to_u8(v);
    }
  }
}

}  // namespace

int p2pvg_vis_canvas_impl(const float* store0, int n0, const float* store1, int n1, int C, int H, const int32_t* tiles_host,
                          int32_t* tiles_dev, int r_len, int n_block, float* canvas, float* video, uint8_t* gif,
                          cudaStream_t st) {
  P2PVG_REQUIRE(tiles_host && tiles_dev && canvas && video && gif, P2PVG_ERR_BAD_ARG, "vis_canvas: null pointer");
  P2PVG_REQUIRE(C == 1 || C == 3, P2PVG_ERR_BAD_ARG, "vis_canvas: C = %d (needs 1 or 3)", C);
  P2PVG_REQUIRE(H >= 1 && H <= VIS_MAX_W, P2PVG_ERR_BAD_ARG, "vis_canvas: H = W = %d (needs 1..%d)", H, VIS_MAX_W);
  P2PVG_REQUIRE(r_len >= 1 && n_block >= 1 && n0 >= 0 && n1 >= 0, P2PVG_ERR_BAD_ARG,
                "vis_canvas: r_len = %d, n_block = %d, n0 = %d, n1 = %d", r_len, n_block, n0, n1);
  P2PVG_REQUIRE((n0 == 0 || store0) && (n1 == 0 || store1), P2PVG_ERR_BAD_ARG, "vis_canvas: null frame store");
  P2PVG_REQUIRE((long long)r_len * n_block * VIS_ROWS * 3 * H * H < (1LL << 31) &&
                    (long long)(n0 > n1 ? n0 : n1) * C * H * H < (1LL << 40),
                P2PVG_ERR_UNSUPPORTED, "vis_canvas: outputs too large (r_len = %d, n_block = %d, H = %d)", r_len, n_block, H);
  const int n_tiles = r_len * n_block * VIS_ROWS;
  for (int k = 0; k < n_tiles; ++k) {
    const int src = tiles_host[3 * k], idx = tiles_host[3 * k + 1], border = tiles_host[3 * k + 2];
    const int n = src == 0 ? n0 : n1;
    P2PVG_REQUIRE((src == 0 || src == 1) && idx >= -1 && idx < n && border >= 0 && border <= 2, P2PVG_ERR_BAD_ARG,
                  "vis_canvas: tile %d = (store %d, frame %d, border %d) out of range (store 0 has %d frames, store 1 %d)", k,
                  src, idx, border, n0, n1);
  }
  const cudaError_t e = cudaMemcpyAsync(tiles_dev, tiles_host, (size_t)n_tiles * 3 * sizeof(int32_t), cudaMemcpyHostToDevice, st);
  if (e != cudaSuccess) {
    p2pvg_set_error("vis_canvas: tile table copy: %s", cudaGetErrorString(e));
    return P2PVG_ERR_CUDA;
  }
  vis_canvas_kernel<<<n_tiles, VIS_THREADS, 0, st>>>(store0, store1, tiles_dev, C, H, r_len, n_block, canvas, video, gif);
  return p2pvg_check_launch("vis_canvas");
}
