// Video clip windows (WeizmannDataset.__getitem__, data/weizmann.py:103-114; BairRobotPush.get_seq, data/bair.py:51-75) cut
// on the device from a resident uint8 clip store.  One CTA writes one output frame (t, b): it resolves the row's entry to a
// clip, a mirror flag and a window start once, then each thread converts 4 pixels at a time (one 4-byte load, one float4
// store), VW_UNROLL loads in flight before the stores, so that every warp store is 512 contiguous bytes.  Pure bandwidth: the
// fp32 frames written are 4x the bytes read.
#include "common.cuh"

#define VW_THREADS 256
#define VW_UNROLL 4

namespace {

// byte i of the result is byte 3 - i of w
__device__ __forceinline__ uint32_t reverse_bytes(uint32_t w) { return __byte_perm(w, 0, 0x0123); }

// ToTensor: u8 -> fp32 u / 255, correctly rounded.  The product with the rounded reciprocal is off by one ulp for some u; one
// FMA residual step corrects it, which is exact for all 256 values (checked exhaustively against IEEE division).
__device__ __forceinline__ float unit_from_u8(uint32_t u) {
  const float x = (float)u, r = 1.f / 255.f;
  const float q = __fmul_rn(x, r);
  return __fmaf_rn(__fmaf_rn(-q, 255.f, x), r, q);
}

__global__ void __launch_bounds__(VW_THREADS) video_windows_kernel(const uint8_t* __restrict__ frames,
                                                                   const int64_t* __restrict__ clip_first,
                                                                   const int32_t* __restrict__ clip_len,
                                                                   const int32_t* __restrict__ entries,
                                                                   const int32_t* __restrict__ draws, int paired_flips, int B,
                                                                   int L, int rows, int w4, float* __restrict__ out) {
  const int t = blockIdx.x / B, b = blockIdx.x - t * B;
  const int e = entries[b];
  const int clip = paired_flips ? e >> 1 : e;
  const bool flip = paired_flips && (e & 1);
  // np.random.randint(0, n_frames - L + 1) -> r % (n_frames - L + 1), r taken as unsigned
  const int start = draws ? (int)((unsigned)draws[b] % (unsigned)(clip_len[clip] - L + 1)) : 0;
  const int n4 = rows * w4;  // 4-pixel words per frame (rows = C * H)
  const uint32_t* src = reinterpret_cast<const uint32_t*>(frames + (size_t)(clip_first[clip] + start + t) * n4 * 4);
  float4* dst = reinterpret_cast<float4*>(out + ((size_t)t * B + b) * n4 * 4);
  for (int i0 = threadIdx.x; i0 < n4; i0 += VW_THREADS * VW_UNROLL) {
    uint32_t w[VW_UNROLL];
#pragma unroll
    for (int u = 0; u < VW_UNROLL; ++u) {
      const int i = i0 + u * VW_THREADS;
      if (i < n4) {
        const int y = i / w4, k = i - y * w4;
        w[u] = flip ? reverse_bytes(__ldg(src + y * w4 + (w4 - 1 - k))) : __ldg(src + i);
      }
    }
#pragma unroll
    for (int u = 0; u < VW_UNROLL; ++u) {
      const int i = i0 + u * VW_THREADS;
      if (i < n4)
        dst[i] = make_float4(unit_from_u8(w[u] & 0xffu), unit_from_u8((w[u] >> 8) & 0xffu), unit_from_u8((w[u] >> 16) & 0xffu),
                             unit_from_u8(w[u] >> 24));
    }
  }
}

}  // namespace

extern "C" int p2pvg_video_windows(const uint8_t* frames, const int64_t* clip_first, const int32_t* clip_len, int n_clips,
                                   const int32_t* entries, const int32_t* draws, int paired_flips, int B, int L, int T, int C, int H, int W,
                                   float* out, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  P2PVG_REQUIRE(frames && clip_first && clip_len && entries && out, P2PVG_ERR_BAD_ARG, "video_windows: null pointer");
  P2PVG_REQUIRE(((uintptr_t)frames & 3) == 0 && ((uintptr_t)out & 15) == 0, P2PVG_ERR_BAD_ARG,
                "video_windows: frames must be 4-byte and out 16-byte aligned");
  P2PVG_REQUIRE(n_clips >= 1, P2PVG_ERR_BAD_ARG, "video_windows: n_clips = %d", n_clips);
  P2PVG_REQUIRE(B >= 0 && T >= 0 && L >= 1 && T <= L, P2PVG_ERR_BAD_ARG, "video_windows: B = %d, T = %d, L = %d (needs 0 <= T <= L)",
                B, T, L);
  P2PVG_REQUIRE(C >= 1 && H >= 1 && W >= 4 && W % 4 == 0, P2PVG_ERR_BAD_ARG,
                "video_windows: C = %d, H = %d, W = %d (needs C, H >= 1, W %% 4 == 0)", C, H, W);
  P2PVG_REQUIRE((long long)C * H * W <= (1LL << 30), P2PVG_ERR_UNSUPPORTED, "video_windows: frame too large");
  if (T == 0 || B == 0) return P2PVG_OK;
  P2PVG_REQUIRE((long long)T * B < (1LL << 31), P2PVG_ERR_UNSUPPORTED, "video_windows: T * B = %lld frames", (long long)T * B);
  video_windows_kernel<<<T * B, VW_THREADS, 0, st>>>(frames, clip_first, clip_len, entries, draws, paired_flips ? 1 : 0, B, L,
                                                     C * H, W / 4, out);
  return p2pvg_check_launch("video_windows");
}
