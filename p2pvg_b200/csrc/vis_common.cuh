// Device code shared by the picture compositions (vis.cu, gen_vis.cu): the reference's control-point borders
// (misc/visualize.py:13-87) and its (frame * 255).astype(np.uint8) GIF conversion.
#pragma once
#include <cstdint>

#define VIS_PAD 3           // border width (misc/visualize.py:13, 55)
#define VIS_MAX_W 128
#define VIS_ORANGE 1
#define VIS_RED 2

// channel c of a border pixel: orange (1, 165 / 255, 0) or red (1, 0, 0)
__device__ __forceinline__ float vis_border_value(int border, int c) {
  return c == 0 ? 1.f : (c == 1 && border == VIS_ORANGE) ? (float)(165.0 / 255.0) : 0.f;
}

// pixel (y, x) of a W x W frame lies in the border of a tile whose border is not 0
__device__ __forceinline__ bool vis_is_edge(int border, int y, int x, int W) {
  return border != 0 && !(y >= VIS_PAD && y < W - VIS_PAD && x >= VIS_PAD && x < W - VIS_PAD);
}

// (v * 255).astype(np.uint8): fp32 product, truncated toward zero, low byte
__device__ __forceinline__ uint8_t vis_to_u8(float v) { return (uint8_t)(int)truncf(v * 255.f); }
