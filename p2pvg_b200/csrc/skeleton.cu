// Human3.6M skeletons drawn as the reference's Skeleton3DVisualizer draws them (data/human36m/human36m.py:290-388): the
// mplot3d camera of p2pvg_b200/skeleton.py (its module docstring is the spec), limbs as 3-pt lines with projecting caps,
// 8 x 8 supersampled coverage, the 98 x 98 crop of the 128 x 128 figure.  One CTA per image: the joints are projected into
// shared memory, each limb becomes a rectangle with a bounding box, and each pixel tests only the limbs whose box covers it.
//
// Exactness: projection and coverage are evaluated in fp64 with one rounding per operation (__d*_rn, no contraction), in
// the order of tests/skeleton_ref.py, so every coverage count equals the oracle's.  A pixel whose centre lies deep inside or
// far outside a rectangle (margin 0.625 px, more than the 0.619 px a sample point lies from the centre) takes 64 or 0
// without the per-sample loop.  The blend and the quantisation are fp32 with one rounding per operation, as the oracle's
// NumPy float32 arithmetic.
#include "common.cuh"

#define SK_THREADS 256
#define SK_FIG 128                 // figure: 2 in x 64 dpi
#define SK_CROP 15                 // fig2img's crop
#define SK_OUT (SK_FIG - 2 * SK_CROP)
#define SK_PIX (SK_OUT * SK_OUT)
#define SK_MAXJ 32
#define SK_VIEWS 4

namespace {

struct SkelTables {
  float rows[SK_VIEWS * 12];        // per view rows 0, 1, 3 of M = P . View . W, row-major [3][4]
  float color[(SK_MAXJ - 1) * 3];   // per limb RGB
  int parent[SK_MAXJ];
};

constexpr double kHalf = 1.5 * 64.0 / 72.0;   // half the 3-pt line width in pixels
constexpr double kMargin = 0.625;             // > sqrt(2) * 7/16, the farthest a sample point lies from its pixel centre
constexpr double kFastRange = 1048576.0;      // the centre-only shortcut is taken for limbs within 2^20 px of the origin

__device__ __forceinline__ double dot2(double a, double b, double c, double d) {   // fl(fl(a b) + fl(c d))
  return __dadd_rn(__dmul_rn(a, b), __dmul_rn(c, d));
}

// Pixel column of a display x (columns cover [c, c + 1)) and row of a display y (row r covers [127 - r, 128 - r)), as crop
// coordinates clamped to [-1, SK_OUT]; d is finite and already clamped to a few thousand pixels.
__device__ __forceinline__ int crop_col(double x) { return max(-1, min(SK_OUT, (int)floor(x) - SK_CROP)); }
__device__ __forceinline__ int crop_row(double y) { return max(-1, min(SK_OUT, SK_FIG - 1 - (int)floor(y) - SK_CROP)); }

// Number of the 8 x 8 sample points of crop pixel (rr, cc) inside limb l's rectangle: along in [-h, len + h], |across| <= h.
__device__ __forceinline__ int coverage(double p0x, double p0y, double ux, double uy, double lenh, int rr, int cc) {
  const double X0 = (double)(cc + SK_CROP), Y0 = (double)(SK_FIG - 1 - (rr + SK_CROP));
  double ax[8], bx[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const double ex = __dsub_rn(X0 + (i + 0.5) * 0.125, p0x);   // the sample coordinate is exact
    ax[i] = __dmul_rn(ux, ex);
    bx[i] = __dmul_rn(uy, ex);
  }
  int k = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const double ey = __dsub_rn(Y0 + (j + 0.5) * 0.125, p0y);
    const double by = __dmul_rn(uy, ey), cy = __dmul_rn(ux, ey);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const double along = __dadd_rn(ax[i], by), across = __dsub_rn(cy, bx[i]);
      k += (along >= -kHalf) & (along <= lenh) & (fabs(across) <= kHalf);
    }
  }
  return k;
}

__global__ void __launch_bounds__(SK_THREADS) skeleton_kernel(const float* __restrict__ poses, const int32_t* __restrict__ views,
                                                              int J, const SkelTables tb, float* __restrict__ out_f,
                                                              uint8_t* __restrict__ out_u8) {
  __shared__ float s_rows[12], s_color[(SK_MAXJ - 1) * 3];
  __shared__ int s_parent[SK_MAXJ];
  __shared__ double s_jx[SK_MAXJ], s_jy[SK_MAXJ];
  __shared__ double s_p0x[SK_MAXJ], s_p0y[SK_MAXJ], s_ux[SK_MAXJ], s_uy[SK_MAXJ], s_lenh[SK_MAXJ];
  __shared__ int s_box[SK_MAXJ][4];   // crop columns c0..c1, rows r0..r1 of the limb's bounding box
  __shared__ int s_fast[SK_MAXJ];
  __shared__ uint32_t s_rowmask[SK_OUT];
  const int n = blockIdx.x, tid = threadIdx.x, L = J - 1;
  const int view = views[n];
  const bool view_ok = view >= 0 && view < SK_VIEWS;
  if (tid == 0) {   // static indices only, so the tables are read from the parameter bank without a local copy
#pragma unroll
    for (int v = 0; v < SK_VIEWS; ++v)
      if (v == view) {
#pragma unroll
        for (int k = 0; k < 12; ++k) s_rows[k] = tb.rows[v * 12 + k];
      }
#pragma unroll
    for (int k = 0; k < (SK_MAXJ - 1) * 3; ++k) s_color[k] = tb.color[k];
#pragma unroll
    for (int k = 0; k < SK_MAXJ; ++k) s_parent[k] = tb.parent[k];
  }
  __syncthreads();
  if (tid < J && view_ok) {
    const float* p = poses + ((size_t)n * J + tid) * 3;
    const double X = p[0], Y = p[2], Z = p[1];   // plotted (X, Y, Z) = (x, z, y)
    double m[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const float* R = s_rows + 4 * r;
      m[r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn((double)R[0], X), __dmul_rn((double)R[1], Y)), __dmul_rn((double)R[2], Z)),
                       (double)R[3]);
    }
    const double x2 = __ddiv_rn(m[0], m[2]), y2 = __ddiv_rn(m[1], m[2]);
    s_jx[tid] = __dmul_rn(__ddiv_rn(__dadd_rn(x2, 0.095), 0.185), 128.0);
    s_jy[tid] = __dmul_rn(__ddiv_rn(__dadd_rn(y2, 0.095), 0.185), 128.0);
  }
  __syncthreads();
  if (tid < L) {
    int box[4] = {1, 0, 1, 0}, fast = 0;
    double ux = 0., uy = 0., lenh = 0.;
    const double p0x = view_ok ? s_jx[tid + 1] : 0., p0y = view_ok ? s_jy[tid + 1] : 0.;
    const double p1x = view_ok ? s_jx[s_parent[tid + 1]] : 0., p1y = view_ok ? s_jy[s_parent[tid + 1]] : 0.;
    const double dx = __dsub_rn(p1x, p0x), dy = __dsub_rn(p1y, p0y);
    const double len = __dsqrt_rn(dot2(dx, dx, dy, dy));
    // nothing for a limb shorter than 1e-6 px (the zero poses of skipped frames) or with a non-finite end
    if (view_ok && len >= 1e-6 && isfinite(len) && isfinite(p0x) && isfinite(p0y) && isfinite(p1x) && isfinite(p1y)) {
      ux = __ddiv_rn(dx, len);
      uy = __ddiv_rn(dy, len);
      lenh = __dadd_rn(len, kHalf);
      const double lim = 4096.0, pad = 2.0 * kHalf;   // a conservative box: the caps reach sqrt(2) h past an end
      const double xlo = fmax(-lim, fmin(p0x, p1x) - pad), xhi = fmin(lim, fmax(p0x, p1x) + pad);
      const double ylo = fmax(-lim, fmin(p0y, p1y) - pad), yhi = fmin(lim, fmax(p0y, p1y) + pad);
      box[0] = max(0, crop_col(xlo));
      box[1] = min(SK_OUT - 1, crop_col(xhi));
      box[2] = max(0, crop_row(yhi));
      box[3] = min(SK_OUT - 1, crop_row(ylo));
      fast = fmax(fmax(fabs(p0x), fabs(p0y)), fmax(fabs(p1x), fabs(p1y))) < kFastRange;
    }
    s_p0x[tid] = p0x;
    s_p0y[tid] = p0y;
    s_ux[tid] = ux;
    s_uy[tid] = uy;
    s_lenh[tid] = lenh;
#pragma unroll
    for (int k = 0; k < 4; ++k) s_box[tid][k] = box[k];
    s_fast[tid] = fast;
  }
  __syncthreads();
  for (int r = tid; r < SK_OUT; r += SK_THREADS) {
    uint32_t mask = 0;
    for (int l = 0; l < L; ++l) mask |= (uint32_t)(s_box[l][0] <= s_box[l][1] && s_box[l][2] <= r && r <= s_box[l][3]) << l;
    s_rowmask[r] = mask;
  }
  __syncthreads();
  float* of = out_f ? out_f + (size_t)n * 3 * SK_PIX : nullptr;
  uint8_t* ou = out_u8 ? out_u8 + (size_t)n * 3 * SK_PIX : nullptr;
  for (int p = tid; p < SK_PIX; p += SK_THREADS) {
    const int rr = p / SK_OUT, cc = p - rr * SK_OUT;
    float c[3] = {1.f, 1.f, 1.f};   // white background
    uint32_t mask = s_rowmask[rr];
    while (mask) {   // ascending limb order: later limbs over earlier ones
      const int l = __ffs(mask) - 1;
      mask &= mask - 1;
      if (cc < s_box[l][0] || cc > s_box[l][1]) continue;
      const double p0x = s_p0x[l], p0y = s_p0y[l], ux = s_ux[l], uy = s_uy[l], lenh = s_lenh[l];
      int k = -1;
      if (s_fast[l]) {
        const double ex = (double)(cc + SK_CROP) + 0.5 - p0x, ey = (double)(SK_FIG - 1 - (rr + SK_CROP)) + 0.5 - p0y;
        const double along = ux * ex + uy * ey, across = fabs(ux * ey - uy * ex);
        if (along < -kHalf - kMargin || along > lenh + kMargin || across > kHalf + kMargin) k = 0;
        else if (along >= -kHalf + kMargin && along <= lenh - kMargin && across <= kHalf - kMargin) k = 64;
      }
      if (k < 0) k = coverage(p0x, p0y, ux, uy, lenh, rr, cc);
      if (k == 0) continue;
      const float w = (float)k * 0.015625f;
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) c[ch] = __fadd_rn(c[ch], __fmul_rn(__fsub_rn(s_color[3 * l + ch], c[ch]), w));
    }
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const int q = min(255, (int)floorf(__fadd_rn(__fmul_rn(255.f, c[ch]), 0.5f)));
      if (of) of[ch * SK_PIX + p] = __double2float_rn(__ddiv_rn((double)q, 255.0));   // float32(q / 255.) as NumPy rounds it
      if (ou) ou[3 * p + ch] = (uint8_t)q;
    }
  }
}

}  // namespace

extern "C" int p2pvg_skeleton_render(const float* poses, const int32_t* views, int n, int J, const int32_t* parents_host,
                                     const float* colors_host, const float* matrices_host, float* out_f, uint8_t* out_u8,
                                     void* stream) {
  P2PVG_REQUIRE(n >= 0, P2PVG_ERR_BAD_ARG, "skeleton_render: n = %d", n);
  P2PVG_REQUIRE(J >= 2 && J <= SK_MAXJ, P2PVG_ERR_BAD_ARG, "skeleton_render: J = %d joints (needs 2..%d)", J, SK_MAXJ);
  P2PVG_REQUIRE(parents_host && colors_host && matrices_host, P2PVG_ERR_BAD_ARG, "skeleton_render: null host table");
  P2PVG_REQUIRE(n == 0 || (poses && views && (out_f || out_u8)), P2PVG_ERR_BAD_ARG,
                "skeleton_render: null poses, views or both outputs");
  P2PVG_REQUIRE(((uintptr_t)poses & 3) == 0 && ((uintptr_t)views & 3) == 0 && ((uintptr_t)out_f & 3) == 0, P2PVG_ERR_BAD_ARG,
                "skeleton_render: misaligned poses, views or fp32 output");
  P2PVG_REQUIRE(parents_host[0] == -1, P2PVG_ERR_BAD_ARG, "skeleton_render: parents[0] = %d (needs -1)", parents_host[0]);
  SkelTables tb;
  tb.parent[0] = 0;
  for (int j = 1; j < SK_MAXJ; ++j) {
    if (j < J) {
      P2PVG_REQUIRE(parents_host[j] >= 0 && parents_host[j] < j, P2PVG_ERR_BAD_ARG,
                    "skeleton_render: parents[%d] = %d (needs 0 <= parents[j] < j)", j, parents_host[j]);
    }
    tb.parent[j] = j < J ? parents_host[j] : 0;
  }
  for (int k = 0; k < (SK_MAXJ - 1) * 3; ++k) {
    const float v = k < (J - 1) * 3 ? colors_host[k] : 0.f;
    P2PVG_REQUIRE(v >= 0.f && v <= 1.f, P2PVG_ERR_BAD_ARG, "skeleton_render: colour value %d = %g (needs 0..1)", k, (double)v);
    tb.color[k] = v;
  }
  for (int k = 0; k < SK_VIEWS * 12; ++k) {
    P2PVG_REQUIRE(isfinite(matrices_host[k]), P2PVG_ERR_BAD_ARG, "skeleton_render: matrix value %d not finite", k);
    tb.rows[k] = matrices_host[k];
  }
  if (n == 0) return P2PVG_OK;
  skeleton_kernel<<<n, SK_THREADS, 0, (cudaStream_t)stream>>>(poses, views, J, tb, out_f, out_u8);
  return p2pvg_check_launch("skeleton_render");
}
