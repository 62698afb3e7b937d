// The four terms of P2PModel.forward's objective split by batch row, for held-out scoring (P2PModel.p2p_losses): one launch
// reads the decoded frames, the Gaussian heads and the predicted latents of an eval-mode forward and writes per-row values
// and the four scalars (include/p2pvg_b200.h).
//
// One CTA per (executed step s, row b), s in [0, S]: step s < S contributes the squared reconstruction error of decode s
// against frame tgt[s], the KL sum of (mu, logvar) against (mu_p, logvar_p) and, for s < S - 1, the squared distance of
// h_pred[s] to row 0 of the latent of frame in_idx[s]; step S (the CPC decode) contributes the squared error against
// frame tgt[S] = x_cp.  Every thread accumulates its elements in fp64 in a fixed order, the CTA reduces in a fixed order
// and stores its three partials.  The CTA that finishes last (integer ticket) sums each row over s in step order and the
// rows in row order, and rearms the ticket counter for the next launch.  No float atomics: two launches on the same data
// give bit-identical results.  The kernel streams each decoded and target element once (HBM-bound).
#include "common.cuh"

#define SL_THREADS 256

namespace {

__device__ __forceinline__ double block_sum_d(double v, double* red /* [SL_THREADS / 32] */) {
  v = warp_sum_d(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) red[w] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int i = 0; i < SL_THREADS / 32; i++) s += red[i];
  return s;   // valid on thread 0
}

template <typename T>
__global__ void __launch_bounds__(SL_THREADS) seq_losses_kernel(const T* __restrict__ rec, int sigmoid, int vec, const float* __restrict__ x,
                                                                const int* __restrict__ tgt, int S, int B, long long E,
                                                                const float* __restrict__ mu, const float* __restrict__ lv,
                                                                const float* __restrict__ mu_p, const float* __restrict__ lv_p, int z,
                                                                const float* __restrict__ H, const int* __restrict__ in_idx,
                                                                const float* __restrict__ h_pred, int g, int has_cpc,
                                                                double batch_size, double seq_len, double* __restrict__ partial,
                                                                unsigned int* __restrict__ counter, double* __restrict__ per_seq,
                                                                double* __restrict__ out) {
  __shared__ double red[SL_THREADS / 32];
  __shared__ bool last;
  const int s = blockIdx.x / B, b = blockIdx.x % B, tid = threadIdx.x;
  double e2 = 0.0, kl = 0.0, al = 0.0;
  if (s < S || has_cpc) {
    const T* r = rec + ((long long)s * B + b) * E;
    const float* xt = x + ((long long)tgt[s] * B + b) * E;
    if (vec) {
      for (long long i = 4 * tid; i < E; i += 4 * SL_THREADS) {
        const f4 v = ld_f4<T>(r + i), t = ld_f4<float>(xt + i);
#pragma unroll
        for (int k = 0; k < 4; k++) {
          const float d = (sigmoid ? sigmoidf_(v.v[k]) : v.v[k]) - t.v[k];
          e2 += (double)d * d;
        }
      }
    } else {
      for (long long i = tid; i < E; i += SL_THREADS) {
        const float v = ld_f<T>(r + i);
        const float d = (sigmoid ? sigmoidf_(v) : v) - xt[i];
        e2 += (double)d * d;
      }
    }
  }
  if (s < S) {
    const long long o = ((long long)s * B + b) * z;
    for (int k = tid; k < z; k += SL_THREADS) {   // misc/criterion.py:10-15 with log(sigma2 / sigma1) = (lv_p - lv) / 2
      const double l1 = lv[o + k], l2 = lv_p[o + k], d = (double)mu[o + k] - (double)mu_p[o + k];
      kl += 0.5 * (l2 - l1) + (exp(l1) + d * d) / (2.0 * exp(l2)) - 0.5;
    }
  }
  if (s < S - 1) {   // models/p2p_model.py:224-225: h[0] is row 0 of the previous step's latent, broadcast over the batch
    const float* h0 = H + (long long)in_idx[s] * B * g;
    const float* hp = h_pred + ((long long)s * B + b) * g;
    for (int k = tid; k < g; k += SL_THREADS) {
      const double d = (double)h0[k] - (double)hp[k];
      al += d * d;
    }
  }
  e2 = block_sum_d(e2, red);
  kl = block_sum_d(kl, red);
  al = block_sum_d(al, red);
  if (tid == 0) {
    double* p = partial + 3LL * blockIdx.x;
    p[0] = e2;
    p[1] = kl;
    p[2] = al;
    __threadfence();
    last = atomicAdd(counter, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  const double inv_e = 1.0 / ((double)E * seq_len), inv_kl = 1.0 / (batch_size * seq_len), inv_g = 1.0 / ((double)g * seq_len);
  for (int bb = tid; bb < B; bb += SL_THREADS) {
    double m = 0.0, k = 0.0, a = 0.0;
    for (int t = 0; t < S; t++) {
      const double* p = partial + 3LL * ((long long)t * B + bb);
      m += __ldcg(p);
      k += __ldcg(p + 1);
      if (t < S - 1) a += __ldcg(p + 2);
    }
    per_seq[bb] = m * inv_e;
    per_seq[B + bb] = k * inv_kl;
    per_seq[2 * B + bb] = has_cpc ? __ldcg(partial + 3LL * ((long long)S * B + bb)) * inv_e : 0.0;
    per_seq[3 * B + bb] = a * inv_g;
  }
  __syncthreads();
  if (tid < 4) {   // row order; mse / cpc / align are means over the rows, kld (already / opt.batch_size) their sum
    double v = 0.0;
    for (int bb = 0; bb < B; bb++) v += per_seq[tid * B + bb];
    out[tid] = tid == 1 ? v : v / B;
  }
  if (tid == 0) *counter = 0u;
}

}  // namespace

extern "C" int p2pvg_seq_losses(const void* rec, int dtype, int sigmoid, const float* x, const int* tgt, int S, int B, int64_t E,
                                const float* mu, const float* lv, const float* mu_p, const float* lv_p, int z, const float* H,
                                const int* in_idx, const float* h_pred, int g, int has_cpc, double batch_size, double seq_len,
                                double* partial, uint32_t* counter, double* per_seq, double* out, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  P2PVG_REQUIRE(rec && x && tgt && mu && lv && mu_p && lv_p && H && in_idx && h_pred && partial && counter && per_seq && out,
                P2PVG_ERR_BAD_ARG, "seq_losses: null pointer");
  P2PVG_REQUIRE(S >= 1 && B >= 1 && E >= 1 && z >= 1 && g >= 1 && batch_size > 0.0 && seq_len > 0.0, P2PVG_ERR_BAD_ARG,
                "seq_losses: bad shape (S %d, B %d, E %lld, z %d, g %d)", S, B, (long long)E, z, g);
  // 4-wide loads when every row starts on a vector boundary (16 B for fp32, 8 B for bf16)
  const int vec = (E & 3) == 0 && ((uintptr_t)x & 15) == 0 && ((uintptr_t)rec & (dtype == P2PVG_BF16 ? 7 : 15)) == 0;
  const long long grid = (long long)(S + 1) * B;
  P2PVG_REQUIRE(grid < (1LL << 31), P2PVG_ERR_BAD_ARG, "seq_losses: too many (step, row) pairs");
  DISPATCH_DTYPE(dtype, T, (seq_losses_kernel<T><<<(unsigned)grid, SL_THREADS, 0, st>>>(
      (const T*)rec, sigmoid, vec, x, tgt, S, B, E, mu, lv, mu_p, lv_p, z, H, in_idx, h_pred, g, has_cpc, batch_size, seq_len, partial,
      counter, per_seq, out)));
  return p2pvg_check_launch("seq_losses");
}
