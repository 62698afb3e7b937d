// Moving MNIST batch synthesis (data/moving_mnist.py:51-105, DynamicLengthMovingMNIST.__getitem__) on the device.
// One CTA renders a chunk of MM_FRAMES frames of one sequence: it replays the num_digits trajectories from the draws
// table (cheap, one thread per digit) up to the end of its chunk, stages the drawn digits in shared memory as fp32, and
// writes the frames with 16-byte stores.  The frames are pure output bandwidth (126 MB per T = 30, B = 256 batch).
#include "common.cuh"

#define MM_THREADS 256
#define MM_FRAMES 8
#define MM_MAX_DIGITS 4
#define MM_DIGIT 32

namespace {

struct DrawCursor {
  const int* row;
  int k;
  // np.random.randint(lo, hi) -> lo + r % (hi - lo) with r the next entry of the row (taken as unsigned, so that a
  // negative entry still lands in range)
  __device__ __forceinline__ int next(int lo, int hi) { return lo + (int)((unsigned)row[k++] % (unsigned)(hi - lo)); }
};

__global__ void __launch_bounds__(MM_THREADS) moving_mnist_kernel(const uint8_t* __restrict__ digits, int n_digits,
                                                                  const int* __restrict__ draws, int draw_stride,
                                                                  float* __restrict__ out, int T, int B, int S, int nd,
                                                                  int deterministic, int row_len) {
  extern __shared__ float smem[];
  float* sdig = smem;                                               // [nd][32*32] fp32 digits
  int* sdraw = reinterpret_cast<int*>(smem + nd * MM_DIGIT * MM_DIGIT);  // [nd][row_len] draws used up to t1
  __shared__ int2 spos[MM_MAX_DIGITS][MM_FRAMES];                   // (sx, sy) of frames t0..t1-1
  __shared__ int sidx[MM_MAX_DIGITS];

  const int b = blockIdx.x;
  const int t0 = blockIdx.y * MM_FRAMES;
  const int t1 = min(T, t0 + MM_FRAMES);
  // the random branch draws at most 4 values per step, so frames < t1 read at most 5 + 4*t1 entries of a row
  const int need = 5 + 4 * t1;
  for (int i = threadIdx.x; i < nd * need; i += MM_THREADS) {
    const int n = i / need, j = i - n * need;
    sdraw[n * row_len + j] = draws[((size_t)b * nd + n) * draw_stride + j];
  }
  __syncthreads();

  if (threadIdx.x < nd) {
    const int n = threadIdx.x;
    const int hi = S - MM_DIGIT;  // positions stay in [0, S-33]
    DrawCursor d{sdraw + n * row_len, 0};
    sidx[n] = d.next(0, n_digits);
    int sx = d.next(0, hi), sy = d.next(0, hi);
    int dx = d.next(-4, 5), dy = d.next(-4, 5);
    for (int t = 0; t < t1; ++t) {
      if (sy < 0) {
        sy = 0;
        if (deterministic) dy = -dy;
        else { dy = d.next(1, 5); dx = d.next(-4, 5); }
      } else if (sy >= hi) {
        sy = hi - 1;
        if (deterministic) dy = -dy;
        else { dy = d.next(-4, 0); dx = d.next(-4, 5); }
      }
      if (sx < 0) {
        sx = 0;
        if (deterministic) dx = -dx;
        else { dx = d.next(1, 5); dy = d.next(-4, 5); }
      } else if (sx >= hi) {
        sx = hi - 1;
        if (deterministic) dx = -dx;
        else { dx = d.next(-4, 0); dy = d.next(-4, 5); }
      }
      if (t >= t0) spos[n][t - t0] = make_int2(sx, sy);
      sy += dy;
      sx += dx;
    }
  }
  __syncthreads();

  // ToTensor: u8 -> fp32 u / 255, correctly rounded
  for (int i = threadIdx.x; i < nd * MM_DIGIT * MM_DIGIT; i += MM_THREADS) {
    const int n = i / (MM_DIGIT * MM_DIGIT), p = i - n * (MM_DIGIT * MM_DIGIT);
    sdig[i] = __fdiv_rn((float)digits[(size_t)sidx[n] * (MM_DIGIT * MM_DIGIT) + p], 255.f);
  }
  __syncthreads();

  const int q = S >> 2;  // float4 per row
  for (int t = t0; t < t1; ++t) {
    float4* frame = reinterpret_cast<float4*>(out + ((size_t)t * B + b) * S * S);
    for (int i = threadIdx.x; i < S * q; i += MM_THREADS) {
      const int y = i / q, x0 = (i - y * q) * 4;
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      // x[t, 0, sy:sy+32, sx:sx+32] += digit, digits in the reference's order, fp32
      for (int n = 0; n < nd; ++n) {
        const int2 p = spos[n][t - t0];
        const int ry = y - p.y;
        if ((unsigned)ry >= MM_DIGIT) continue;
        const float* drow = sdig + n * MM_DIGIT * MM_DIGIT + ry * MM_DIGIT;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int rx = x0 + k - p.x;
          if ((unsigned)rx < MM_DIGIT) v[k] += drow[rx];
        }
      }
      // x[x > 1] = 1
#pragma unroll
      for (int k = 0; k < 4; ++k) v[k] = v[k] > 1.f ? 1.f : v[k];
      frame[i] = make_float4(v[0], v[1], v[2], v[3]);
    }
  }
}

}  // namespace

extern "C" int p2pvg_moving_mnist(const uint8_t* digits, int n_digits, const int32_t* draws, int draw_stride, float* out, int T, int B,
                                  int S, int num_digits, int deterministic, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  P2PVG_REQUIRE(digits && draws && out, P2PVG_ERR_BAD_ARG, "moving_mnist: null pointer");
  P2PVG_REQUIRE(n_digits >= 1, P2PVG_ERR_BAD_ARG, "moving_mnist: n_digits = %d", n_digits);
  P2PVG_REQUIRE(S >= MM_DIGIT + 1 && S % 4 == 0, P2PVG_ERR_BAD_ARG, "moving_mnist: S = %d (needs S >= 33, S %% 4 == 0)", S);
  P2PVG_REQUIRE(num_digits >= 1 && num_digits <= MM_MAX_DIGITS, P2PVG_ERR_BAD_ARG, "moving_mnist: num_digits = %d (1..4)", num_digits);
  P2PVG_REQUIRE(T >= 0 && B >= 0, P2PVG_ERR_BAD_ARG, "moving_mnist: T = %d, B = %d", T, B);
  P2PVG_REQUIRE((long long)draw_stride >= 5 + 4LL * T, P2PVG_ERR_BAD_ARG, "moving_mnist: draw_stride = %d < 5 + 4T (T = %d)", draw_stride, T);
  P2PVG_REQUIRE(((uintptr_t)out & 15) == 0, P2PVG_ERR_BAD_ARG, "moving_mnist: out must be 16-byte aligned");
  if (T == 0 || B == 0) return P2PVG_OK;
  const int row_len = 5 + 4 * T;
  const size_t smem = (size_t)num_digits * (MM_DIGIT * MM_DIGIT + row_len) * sizeof(float);
  P2PVG_REQUIRE(smem <= 48 * 1024, P2PVG_ERR_UNSUPPORTED, "moving_mnist: T = %d too long for %d digits", T, num_digits);
  dim3 grid(B, (T + MM_FRAMES - 1) / MM_FRAMES);
  moving_mnist_kernel<<<grid, MM_THREADS, smem, st>>>(digits, n_digits, draws, draw_stride, out, T, B, S, num_digits,
                                                       deterministic, row_len);
  return p2pvg_check_launch("moving_mnist");
}
