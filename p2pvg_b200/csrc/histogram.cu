// TensorBoard histograms of many device ranges in one launch (include/p2pvg_b200.h, p2pvg_histograms): per segment the
// np.histogram counts over a caller's fp64 edge table, and min, max, num, sum and sum of squares in fp64.
//
// The launch is persistent: each CTA loads the edge table (padded to a power of two with +inf) into shared memory once and
// walks the global list of fixed-size chunks (HIST_CHUNK elements of one segment) with a grid stride.  A value's bin is found
// by a branchless binary search in fp64 (fp32 inputs are widened exactly: nothing here is built with -ftz or fast math), and
// counted in a shared-memory histogram with warp-aggregated increments (__match_any_sync), since the default edges put most
// weights of a layer in a few dozen bins and an all-zero gradient in one.  The shared counts go to the int64 output with
// global atomics whenever the CTA's next chunk belongs to another segment.
//
// The fp64 statistics of a chunk are a fixed-order reduction (each thread a strided sequence, then a shuffle tree, then the
// warps in order) written to a partials row of its own; the CTA that finishes a segment's last chunk (a per-segment counter)
// combines that segment's rows in chunk order.  A segment's results therefore depend on the segment alone: not on the grid,
// the other segments of the launch or the order in which chunks finish.
#include "common.cuh"

#include <math.h>
#include <vector>

#define HIST_THREADS 256
#define HIST_UNROLL 8                                        // elements in flight per thread
#define HIST_CHUNK (HIST_THREADS * HIST_UNROLL * 8)          // elements per chunk: 16384 (P2PVG_HIST_CHUNK in the header)
#define HIST_MAX_EDGES 4096
#define HIST_CTAS_PER_SM 4

static_assert(HIST_CHUNK == 16384, "the header documents the chunk size");

namespace {

struct Seg {   // device copy of one segment-table row, plus the index of its first chunk
  long long addr, count, dtype, first_chunk;
};

// NaN-propagating min / max (numpy's): fmin / fmax return the non-NaN operand
__device__ __forceinline__ double nmin(double a, double b) { return (a != a || b != b) ? __longlong_as_double(0x7ff8000000000000LL) : fmin(a, b); }
__device__ __forceinline__ double nmax(double a, double b) { return (a != a || b != b) ? __longlong_as_double(0x7ff8000000000000LL) : fmax(a, b); }

__device__ __forceinline__ int find_seg(const Seg* __restrict__ segs, int n_seg, long long chunk) {
  int lo = 0, hi = n_seg - 1;   // last segment whose first chunk <= chunk
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (segs[mid].first_chunk <= chunk) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(HIST_THREADS, HIST_CTAS_PER_SM)
histogram_kernel(const double* __restrict__ edges_g, int n_edges, int log2p, const Seg* __restrict__ segs, int n_seg,
                 long long n_chunks, unsigned* __restrict__ done, double* __restrict__ partial,
                 unsigned long long* __restrict__ counts, double* __restrict__ stats) {
  extern __shared__ __align__(16) unsigned char hsm[];
  __shared__ double red[4][HIST_THREADS / 32];
  __shared__ int last;
  const int P = 1 << log2p, n_bins = n_edges - 1, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  double* edges = reinterpret_cast<double*>(hsm);            // [P], +inf past n_edges
  unsigned* hist = reinterpret_cast<unsigned*>(edges + P);   // [n_bins]
  for (int i = tid; i < P; i += HIST_THREADS) edges[i] = edges_g[i];
  for (int i = tid; i < n_bins; i += HIST_THREADS) hist[i] = 0u;
  __syncthreads();
  const double e_lo = edges[0], e_hi = edges[n_edges - 1];

  for (long long c = blockIdx.x; c < n_chunks; c += gridDim.x) {
    const int s = find_seg(segs, n_seg, c);
    const Seg sg = segs[s];
    const long long c0 = (c - sg.first_chunk) * HIST_CHUNK;
    const int n = (int)min((long long)HIST_CHUNK, sg.count - c0);
    const bool f64 = sg.dtype == P2PVG_F64;
    const float* pf = reinterpret_cast<const float*>(sg.addr) + c0;
    const double* pd = reinterpret_cast<const double*>(sg.addr) + c0;
    double mn = INFINITY, mx = -INFINITY, sum = 0.0, sq = 0.0;
    for (int base = 0; base < n; base += HIST_THREADS * HIST_UNROLL) {
      double v[HIST_UNROLL];
#pragma unroll
      for (int u = 0; u < HIST_UNROLL; ++u) {
        const int i = base + u * HIST_THREADS + tid;
        v[u] = i < n ? (f64 ? __ldcs(pd + i) : (double)__ldcs(pf + i)) : 0.0;
      }
#pragma unroll
      for (int u = 0; u < HIST_UNROLL; ++u) {
        const bool in = base + u * HIST_THREADS + tid < n;
        int bin = -1;
        if (in) {
          const double x = v[u];
          mn = nmin(mn, x);
          mx = nmax(mx, x);
          sum += x;
          sq += x * x;
          if (x >= e_lo && x <= e_hi) {   // false for NaN
            if (x == e_hi) {
              bin = n_bins - 1;           // the last bin is closed
            } else {                      // largest k with edges[k] <= x (edges[0] <= x < e_hi <= the +inf padding)
              int k = 0;
              for (int step = P >> 1; step > 0; step >>= 1) k = edges[k + step] <= x ? k + step : k;
              bin = k;
            }
          }
        }
        const unsigned peers = __match_any_sync(0xffffffffu, bin);
        if (bin >= 0 && lane == __ffs(peers) - 1) atomicAdd(hist + bin, (unsigned)__popc(peers));
      }
    }
    // fixed-order statistics of this chunk
    mn = -mn;   // reduce as max(-min) and max so that one NaN-propagating max serves both
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mn = nmax(mn, __shfl_xor_sync(0xffffffffu, mn, o));
      mx = nmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      sum += __shfl_xor_sync(0xffffffffu, sum, o);
      sq += __shfl_xor_sync(0xffffffffu, sq, o);
    }
    if (lane == 0) {
      red[0][wid] = mn;
      red[1][wid] = mx;
      red[2][wid] = sum;
      red[3][wid] = sq;
    }
    __syncthreads();
    if (tid == 0) {
      double a = red[0][0], b = red[1][0], d = red[2][0], e = red[3][0];
#pragma unroll
      for (int w = 1; w < HIST_THREADS / 32; ++w) {
        a = nmax(a, red[0][w]);
        b = nmax(b, red[1][w]);
        d += red[2][w];
        e += red[3][w];
      }
      double* pr = partial + 4 * c;
      pr[0] = -a;
      pr[1] = b;
      pr[2] = d;
      pr[3] = e;
      __threadfence();
      const long long n_seg_chunks = (sg.count + HIST_CHUNK - 1) / HIST_CHUNK;
      last = atomicAdd(done + s, 1u) == (unsigned)(n_seg_chunks - 1);
    }
    // flush the shared counts when the next chunk of this CTA is in another segment (or there is none)
    const long long cn = c + gridDim.x;
    const bool flush = cn >= n_chunks || cn >= sg.first_chunk + (sg.count + HIST_CHUNK - 1) / HIST_CHUNK;
    __syncthreads();   // red[] consumed, `last` and every shared increment visible
    if (flush) {
      unsigned long long* out = counts + (size_t)s * n_bins;
      for (int i = tid; i < n_bins; i += HIST_THREADS) {
        const unsigned h = hist[i];
        if (h) {
          atomicAdd(out + i, (unsigned long long)h);
          hist[i] = 0u;
        }
      }
    }
    if (last && wid == 0) {   // this CTA finished the segment's last chunk: combine its partial rows in chunk order
      __threadfence();
      const long long nc = (sg.count + HIST_CHUNK - 1) / HIST_CHUNK;
      const double* pr = partial + 4 * sg.first_chunk;
      double a = -INFINITY, b = -INFINITY, d = 0.0, e = 0.0;
      for (long long k = lane; k < nc; k += 32) {
        a = nmax(a, -__ldcg(pr + 4 * k));
        b = nmax(b, __ldcg(pr + 4 * k + 1));
        d += __ldcg(pr + 4 * k + 2);
        e += __ldcg(pr + 4 * k + 3);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        a = nmax(a, __shfl_xor_sync(0xffffffffu, a, o));
        b = nmax(b, __shfl_xor_sync(0xffffffffu, b, o));
        d += __shfl_xor_sync(0xffffffffu, d, o);
        e += __shfl_xor_sync(0xffffffffu, e, o);
      }
      if (lane == 0) {
        double* o = stats + 5 * (size_t)s;
        o[0] = -a;
        o[1] = b;
        o[2] = (double)sg.count;
        o[3] = d;
        o[4] = e;
      }
    }
    __syncthreads();   // hist zeroed and `last` read before the next chunk
  }
}

// workspace layout: edges [P] fp64 | segment table [n_seg] Seg | done counters [n_seg] u32 | partials [n_chunks][4] fp64,
// each region 16-byte aligned; the first three are staged on the host and uploaded in one copy
struct Layout {
  int log2p;
  long long n_chunks;
  size_t off_segs, off_done, off_partial, staged, total;
};

size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }

Layout layout(const int64_t* segs, int n_seg, int n_edges) {
  Layout L{};
  L.log2p = 1;
  while ((1 << L.log2p) < n_edges) ++L.log2p;
  for (int s = 0; s < n_seg; ++s) L.n_chunks += (segs[3 * s + 1] + HIST_CHUNK - 1) / HIST_CHUNK;
  L.off_segs = align16(sizeof(double) << L.log2p);
  L.off_done = L.off_segs + align16(sizeof(Seg) * (size_t)n_seg);
  L.off_partial = L.off_done + align16(sizeof(unsigned) * (size_t)n_seg);
  L.staged = L.off_partial;
  L.total = L.off_partial + sizeof(double) * 4 * (size_t)L.n_chunks;
  return L;
}

int check_args(const int64_t* segs, int n_seg, const double* edges, int n_edges) {
  P2PVG_REQUIRE(n_seg >= 0, P2PVG_ERR_BAD_ARG, "histograms: n_seg = %d", n_seg);
  P2PVG_REQUIRE(n_seg == 0 || (segs && edges), P2PVG_ERR_BAD_ARG, "histograms: null segment or edge table");
  P2PVG_REQUIRE(n_seg == 0 || n_edges >= 2, P2PVG_ERR_BAD_ARG, "histograms: n_edges = %d (needs at least 2)", n_edges);
  P2PVG_REQUIRE(n_edges <= HIST_MAX_EDGES, P2PVG_ERR_UNSUPPORTED, "histograms: n_edges = %d (at most %d)", n_edges, HIST_MAX_EDGES);
  for (int i = 0; n_seg > 0 && i < n_edges; ++i)
    P2PVG_REQUIRE(isfinite(edges[i]) && (i == 0 || edges[i] > edges[i - 1]), P2PVG_ERR_BAD_ARG,
                  "histograms: edge %d = %g is not finite or not above the previous edge", i, edges[i]);
  for (int s = 0; s < n_seg; ++s) {
    const long long addr = segs[3 * s], count = segs[3 * s + 1], dt = segs[3 * s + 2];
    P2PVG_REQUIRE(dt == P2PVG_F32 || dt == P2PVG_F64, P2PVG_ERR_BAD_ARG, "histograms: segment %d dtype %lld (needs F32 or F64)", s, dt);
    P2PVG_REQUIRE(addr != 0 && addr % (dt == P2PVG_F64 ? 8 : 4) == 0, P2PVG_ERR_BAD_ARG,
                  "histograms: segment %d address 0x%llx is null or not aligned to its element size", s, (unsigned long long)addr);
    P2PVG_REQUIRE(count >= 1, P2PVG_ERR_BAD_ARG, "histograms: segment %d count %lld", s, count);
    P2PVG_REQUIRE(count < (1LL << 40), P2PVG_ERR_UNSUPPORTED, "histograms: segment %d count %lld (below 2^40)", s, count);
  }
  return P2PVG_OK;
}

}  // namespace

extern "C" size_t p2pvg_histograms_workspace_bytes(const int64_t* segs, int n_seg, int n_edges) {
  if (n_seg <= 0 || !segs || n_edges < 2 || n_edges > HIST_MAX_EDGES) return 0;
  return layout(segs, n_seg, n_edges).total;
}

extern "C" int p2pvg_histograms(const int64_t* segs, int n_seg, const double* edges, int n_edges, void* ws, size_t ws_bytes,
                                int64_t* counts, double* stats, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const int rc = check_args(segs, n_seg, edges, n_edges);
  if (rc != P2PVG_OK) return rc;
  if (n_seg == 0) return P2PVG_OK;
  P2PVG_REQUIRE(ws && counts && stats, P2PVG_ERR_BAD_ARG, "histograms: null workspace or output");
  P2PVG_REQUIRE(((uintptr_t)ws & 15) == 0 && ((uintptr_t)counts & 7) == 0 && ((uintptr_t)stats & 7) == 0, P2PVG_ERR_BAD_ARG,
                "histograms: workspace must be 16-byte, counts and stats 8-byte aligned");
  const Layout L = layout(segs, n_seg, n_edges);
  P2PVG_REQUIRE(ws_bytes >= L.total, P2PVG_ERR_WORKSPACE, "histograms: workspace %zu bytes, needs %zu", ws_bytes, L.total);
  std::vector<unsigned char> host(L.staged, 0);
  double* e = reinterpret_cast<double*>(host.data());
  for (int i = 0; i < (1 << L.log2p); ++i) e[i] = i < n_edges ? edges[i] : INFINITY;
  Seg* tab = reinterpret_cast<Seg*>(host.data() + L.off_segs);
  long long first = 0;
  for (int s = 0; s < n_seg; ++s) {
    tab[s] = Seg{segs[3 * s], segs[3 * s + 1], segs[3 * s + 2], first};
    first += (segs[3 * s + 1] + HIST_CHUNK - 1) / HIST_CHUNK;
  }
  unsigned char* w = static_cast<unsigned char*>(ws);
  cudaError_t err = cudaMemcpyAsync(w, host.data(), L.staged, cudaMemcpyHostToDevice, st);
  if (err == cudaSuccess) err = cudaMemsetAsync(counts, 0, sizeof(int64_t) * (size_t)n_seg * (n_edges - 1), st);
  if (err != cudaSuccess) {
    p2pvg_set_error("histograms: table upload: %s", cudaGetErrorString(err));
    return P2PVG_ERR_CUDA;
  }
  const size_t smem = (sizeof(double) << L.log2p) + sizeof(unsigned) * (size_t)(n_edges - 1);
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  static unsigned long long attr_set = 0;   // per device; 64 KB covers the largest table: 4096 edges + 4095 bins = 48 KB
  if (dev >= 64 || !((attr_set >> dev) & 1ULL)) {
    err = cudaFuncSetAttribute(histogram_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 << 10);
    if (err != cudaSuccess) {
      p2pvg_set_error("histograms: shared-memory attribute: %s", cudaGetErrorString(err));
      return P2PVG_ERR_CUDA;
    }
    if (dev < 64) attr_set |= 1ULL << dev;
  }
  const long long grid = min(L.n_chunks, (long long)HIST_CTAS_PER_SM * (sms > 0 ? sms : 1));
  histogram_kernel<<<(unsigned)grid, HIST_THREADS, smem, st>>>(
      reinterpret_cast<const double*>(w), n_edges, L.log2p, reinterpret_cast<const Seg*>(w + L.off_segs), n_seg, L.n_chunks,
      reinterpret_cast<unsigned*>(w + L.off_done), reinterpret_cast<double*>(w + L.off_partial),
      reinterpret_cast<unsigned long long*>(counts), stats);
  return p2pvg_check_launch("histograms");
}
