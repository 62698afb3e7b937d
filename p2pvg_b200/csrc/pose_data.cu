// Human3.6M pose windows (Human36mDataset.__getitem__, constant-speed branch, data/human36m/human36m.py:67-107) gathered on the
// device from resident fp32 pose stores.  A batch is two time-major outputs, [T, B, J, 2] and [T, B, J, 3], and each time step
// of each is one contiguous [B, J, C] slab.  One thread per output float, over both outputs in output order: every warp stores
// 128 contiguous bytes, and since a frame's J * C floats are contiguous in the store, its loads are contiguous runs as well.
#include "common.cuh"

#define PW_THREADS 256

namespace {

__global__ void __launch_bounds__(PW_THREADS) pose_windows_kernel(const float* __restrict__ pose2d, const float* __restrict__ pose3d,
                                                                  int J, const int64_t* __restrict__ seq_first,
                                                                  const int32_t* __restrict__ seq_len,
                                                                  const int32_t* __restrict__ entries,
                                                                  const int32_t* __restrict__ draws, int B, int speed_lo,
                                                                  int n_speeds, int reach, int n2, int n_total,
                                                                  float* __restrict__ out2d, float* __restrict__ out3d) {
  int i = blockIdx.x * PW_THREADS + threadIdx.x;
  if (i >= n_total) return;
  const bool d3 = i >= n2;
  if (d3) i -= n2;
  const int row = (d3 ? 3 : 2) * J;  // floats per (t, b)
  const int tb = i / row, k = i - tb * row;
  const int t = tb / B, b = tb - t * B;
  const int e = entries[b];
  // np.random.randint(0, n - speed_hi * L + 1) and np.random.randint(speed_lo, speed_hi + 1) -> lo + r % (hi - lo), r unsigned
  const int start = (int)((unsigned)draws[b] % (unsigned)(seq_len[e] - reach + 1));
  const int speed = speed_lo + (int)((unsigned)draws[B + b] % (unsigned)n_speeds);
  const long long frame = seq_first[e] + start + (long long)t * speed;
  (d3 ? out3d : out2d)[i] = __ldg((d3 ? pose3d : pose2d) + frame * row + k);
}

}  // namespace

extern "C" int p2pvg_pose_windows(const float* pose2d, const float* pose3d, int J, const int64_t* seq_first, const int32_t* seq_len,
                                  int n_seq, const int32_t* entries, const int32_t* draws, int B, int speed_lo, int speed_hi, int L, int T,
                                  float* out2d, float* out3d, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  P2PVG_REQUIRE(pose2d && pose3d && seq_first && seq_len && entries && draws && out2d && out3d, P2PVG_ERR_BAD_ARG,
                "pose_windows: null pointer");
  P2PVG_REQUIRE((((uintptr_t)pose2d | (uintptr_t)pose3d | (uintptr_t)seq_len | (uintptr_t)entries | (uintptr_t)draws |
                  (uintptr_t)out2d | (uintptr_t)out3d) & 3) == 0 && ((uintptr_t)seq_first & 7) == 0,
                P2PVG_ERR_BAD_ARG, "pose_windows: misaligned pointer");
  P2PVG_REQUIRE(n_seq >= 1 && J >= 1, P2PVG_ERR_BAD_ARG, "pose_windows: n_seq = %d, J = %d", n_seq, J);
  P2PVG_REQUIRE(B >= 0 && T >= 0 && L >= 1 && T <= L, P2PVG_ERR_BAD_ARG, "pose_windows: B = %d, T = %d, L = %d (needs 0 <= T <= L)",
                B, T, L);
  P2PVG_REQUIRE(1 <= speed_lo && speed_lo <= speed_hi, P2PVG_ERR_BAD_ARG, "pose_windows: speed range [%d, %d]", speed_lo, speed_hi);
  P2PVG_REQUIRE((long long)speed_hi * L < (1LL << 31), P2PVG_ERR_UNSUPPORTED, "pose_windows: speed_hi * L = %lld",
                (long long)speed_hi * L);
  const long long n2 = (long long)T * B * J * 2, n_total = (long long)T * B * J * 5;
  P2PVG_REQUIRE(n_total < (1LL << 31), P2PVG_ERR_UNSUPPORTED, "pose_windows: T * B * J * 5 = %lld output floats", n_total);
  if (n_total == 0) return P2PVG_OK;
  pose_windows_kernel<<<(unsigned)((n_total + PW_THREADS - 1) / PW_THREADS), PW_THREADS, 0, st>>>(
      pose2d, pose3d, J, seq_first, seq_len, entries, draws, B, speed_lo, speed_hi - speed_lo + 1, speed_hi * L, (int)n2,
      (int)n_total, out2d, out3d);
  return p2pvg_check_launch("pose_windows");
}
