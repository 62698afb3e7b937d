// Split-level totals of generation scores (include/p2pvg_b200.h): one launch folds one batch's per-pair scores, as
// p2pvg_frame_metrics / p2pvg_pose_metrics wrote them, into device-resident fp64 bins.
//
// Phase 1, one thread per (segment k, row b, metric m): the mean over the segment's F scored frames of every sample s
// (fixed order: frame 0 first, then / F) picks the best sample -- the first NaN mean if there is one, else the first
// maximum (metric in higher_mask) or minimum, i.e. torch's argmax / argmin of metrics.best_of.  Per scored column the
// thread stores the best sample's value, the sum of the samples' finite values and their +-inf / NaN counts.
// Phase 2, the CTA that finishes last (integer ticket): one thread per (bin, metric) walks the columns that map to its bin
// in column order and their rows in row order, sums in fp64 with explicitly rounded adds and multiplies (no contraction
// into FMA), and adds the batch's sums to the totals.  No float atomics: the totals are bit-identical from run to run and
// do not depend on the grid or on which other bins share the launch.  The ticket counter is left zero.
#include "common.cuh"

#include <math.h>

#define MF_THREADS 128

namespace {

__device__ __forceinline__ double score_at(const double* __restrict__ scores, int nm, long long p, int m) {
  return __ldg(scores + p * nm + m);
}

__global__ void __launch_bounds__(MF_THREADS) metrics_fold_kernel(const double* __restrict__ scores, int nm, int higher_mask, int B,
                                                                   int ns, const int32_t* __restrict__ segs, int n_seg,
                                                                   const int32_t* __restrict__ col_bin, int n_cols, int n_bins,
                                                                   double* __restrict__ part_v, int32_t* __restrict__ part_c,
                                                                   unsigned int* __restrict__ counter, double* __restrict__ sums,
                                                                   unsigned long long* __restrict__ counts,
                                                                   unsigned long long* __restrict__ rows) {
  __shared__ bool last;
  const long long task = (long long)blockIdx.x * MF_THREADS + threadIdx.x;
  if (task < (long long)n_seg * B * nm) {
    const int m = (int)(task % nm), b = (int)(task / nm % B), k = (int)(task / nm / B);
    const long long off = segs[3 * k];
    const int c0 = segs[3 * k + 1], F = segs[3 * k + 2];
    const bool higher = (higher_mask >> m) & 1;
    // pair of (frame j, row b, sample s): off + (j * B + b) * ns + s
    int best = 0;
    double bm = 0.0;
    for (int s = 0; s < ns; ++s) {
      double acc = 0.0;
      for (int j = 0; j < F; ++j) acc = __dadd_rn(acc, score_at(scores, nm, off + ((long long)j * B + b) * ns + s, m));
      const double mean = __ddiv_rn(acc, (double)F);
      if (s == 0) {
        bm = mean;
      } else if (!isnan(bm) && (isnan(mean) || (higher ? mean > bm : mean < bm))) {
        best = s;
        bm = mean;
      }
    }
    for (int j = 0; j < F; ++j) {
      const long long p0 = off + ((long long)j * B + b) * ns;
      double all = 0.0;
      int n_inf = 0, n_nan = 0;
      for (int s = 0; s < ns; ++s) {
        const double v = score_at(scores, nm, p0 + s, m);
        if (isnan(v)) n_nan++;
        else if (isinf(v)) n_inf++;
        else all = __dadd_rn(all, v);
      }
      const long long q = (((long long)(c0 + j) * B + b) * nm + m);
      part_v[2 * q] = score_at(scores, nm, p0 + best, m);
      part_v[2 * q + 1] = all;
      part_c[2 * q] = n_inf;
      part_c[2 * q + 1] = n_nan;
    }
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(counter, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  for (int t = threadIdx.x; t < n_cols * nm; t += MF_THREADS) {
    const int c = t / nm, m = t % nm, u = col_bin[c];
    bool first = u >= 0 && u < n_bins;
    for (int cc = 0; cc < c && first; ++cc) first = col_bin[cc] != u;
    if (!first) continue;   // the bin's first column owns it
    double s_best = 0.0, s_sq = 0.0, s_all = 0.0;
    unsigned long long b_inf = 0, b_nan = 0, a_inf = 0, a_nan = 0, n_rows = 0;
    for (int cc = c; cc < n_cols; ++cc) {
      if (col_bin[cc] != u) continue;
      n_rows += B;
      for (int b = 0; b < B; ++b) {
        const long long q = ((long long)cc * B + b) * nm + m;
        const double v = __ldcg(part_v + 2 * q);
        if (isnan(v)) b_nan++;
        else if (isinf(v)) b_inf++;
        else {
          s_best = __dadd_rn(s_best, v);
          s_sq = __dadd_rn(s_sq, __dmul_rn(v, v));
        }
        s_all = __dadd_rn(s_all, __ldcg(part_v + 2 * q + 1));
        a_inf += (unsigned long long)__ldcg(part_c + 2 * q);
        a_nan += (unsigned long long)__ldcg(part_c + 2 * q + 1);
      }
    }
    double* S = sums + ((long long)u * nm + m) * 3;
    S[0] = __dadd_rn(S[0], s_best);
    S[1] = __dadd_rn(S[1], s_sq);
    S[2] = __dadd_rn(S[2], s_all);
    unsigned long long* N = counts + ((long long)u * nm + m) * 4;
    N[0] += b_inf;
    N[1] += b_nan;
    N[2] += a_inf;
    N[3] += a_nan;
    if (m == 0) rows[u] += n_rows;
  }
  if (threadIdx.x == 0) *counter = 0u;
}

}  // namespace

extern "C" int p2pvg_metrics_fold(const double* scores, int n_metrics, int higher_mask, int B, int nsample, const int32_t* segs, int n_seg,
                                  const int32_t* col_bin, int n_cols, int n_bins, double* part_v, int32_t* part_c, uint32_t* counter,
                                  double* sums, uint64_t* counts, uint64_t* rows, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  P2PVG_REQUIRE(scores && segs && col_bin && part_v && part_c && counter && sums && counts && rows, P2PVG_ERR_BAD_ARG,
                "metrics_fold: null pointer");
  P2PVG_REQUIRE(((uintptr_t)scores & 7) == 0 && ((uintptr_t)part_v & 7) == 0 && ((uintptr_t)sums & 7) == 0 &&
                    ((uintptr_t)counts & 7) == 0 && ((uintptr_t)rows & 7) == 0 && ((uintptr_t)segs & 3) == 0 &&
                    ((uintptr_t)col_bin & 3) == 0 && ((uintptr_t)part_c & 3) == 0 && ((uintptr_t)counter & 3) == 0,
                P2PVG_ERR_BAD_ARG, "metrics_fold: misaligned pointer");
  P2PVG_REQUIRE(n_metrics >= 1 && n_metrics <= 8 && B >= 1 && nsample >= 1 && n_seg >= 1 && n_cols >= n_seg && n_bins >= 1,
                P2PVG_ERR_BAD_ARG, "metrics_fold: n_metrics %d, B %d, nsample %d, n_seg %d, n_cols %d, n_bins %d", n_metrics, B,
                nsample, n_seg, n_cols, n_bins);
  const long long tasks = (long long)n_seg * B * n_metrics;
  P2PVG_REQUIRE((long long)n_cols * B * n_metrics < (1LL << 31) && tasks < (1LL << 31), P2PVG_ERR_UNSUPPORTED,
                "metrics_fold: too many (column, row, metric) values");
  const unsigned grid = (unsigned)((tasks + MF_THREADS - 1) / MF_THREADS);
  metrics_fold_kernel<<<grid, MF_THREADS, 0, st>>>(scores, n_metrics, higher_mask, B, nsample, segs, n_seg, col_bin, n_cols, n_bins,
                                                   part_v, part_c, counter, sums, (unsigned long long*)counts,
                                                   (unsigned long long*)rows);
  return p2pvg_check_launch("metrics_fold");
}
