// PNG files of a batch of fp32 / uint8 images (include/p2pvg_b200.h, p2pvg_png_encode), every stage on the device.
//
//   1. filter_kernel (one CTA per image row): quantise the row and the row above to 8-bit RGB with the call's rule, pick
//      the PNG filter (0-4, bpp 3) whose residual has the smallest sum of |signed byte| (libpng's heuristic, lowest filter
//      on ties) and write the filter byte and residuals into the image's filtered stream.
//   2. deflate_kernel (one CTA per PNG_SEG bytes of a filtered stream): LZ77 over the segment with the 32 KB before it as
//      history (never before the image's first byte), one dynamic-Huffman block or stored blocks when those are no larger,
//      then an empty stored block (sync flush) unless the segment ends the image, so segments concatenate byte-aligned.
//      Also the segment's Adler-32 parts.
//   3. scan_kernel (one CTA): exclusive scan of the pieces' sizes; pieces are packed back to back, file after file.
//   4. container_kernel (one CTA per segment): the segment's IDAT chunk with its CRC-32, plus the signature and IHDR in
//      front of an image's first segment and the Adler-32 and IEND after its last.
//
// LZ77 in a CTA, deterministically: the segment is hashed in rounds of PNG_ROUND positions; a position's hash candidate is
// the nearest earlier position of its warp with the same 3-byte hash, else the most recent one before its round (a
// shared-memory head table updated with atomicMax after each round).  Each thread then parses its own PNG_SUB bytes
// greedily with one byte of lazy evaluation, trying distances 1, 3 (one pixel), the row stride and the hash candidate;
// matches stop at the end of the thread's bytes.  Every choice depends on the data alone, so
// the bytes of a file do not depend on the grid or on the other images of the call.
#include "common.cuh"

#include <algorithm>
#include <vector>

#define PNG_SEG 65536          // filtered-stream bytes per segment (P2PVG_PNG_SEGMENT in the header)
#define PNG_HIST 32768         // deflate window
#define PNG_THREADS 256
#define PNG_SUB (PNG_SEG / PNG_THREADS)
#define PNG_HASH_BITS 14
#define PNG_ROUND 128         // positions hashed per round
#define PNG_WIN (PNG_HIST + PNG_SEG + 64)
#define PNG_U8 3               // P2PVG_PNG_U8
#define PNG_SLOT (PNG_SEG + 64)  // compressed bytes of a segment are at most its stored size, PNG_SEG + 15

static_assert(PNG_SUB == 256, "one thread parses 256 bytes: about one longest match");

namespace {

struct Img {   // device copy of one image-table row with its place in the call
  long long addr, dtype, C, H, W, off, row0, seg0, n_seg;
};
struct Seg {   // one segment: its image, its offset in that image's stream, its length and history
  long long img, start, len, hist;
};

__host__ __device__ inline long long stream_len(long long H, long long W) { return H * (1 + 3 * W); }

// ---- stage 1: quantise and filter -------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned quant(const Img& im, int rule, long long y, long long x, int c) {
  if (y < 0 || x < 0) return 0u;
  const long long ch = im.C == 1 ? 0 : c;
  const long long i = (ch * im.H + y) * im.W + x;
  if (im.dtype == PNG_U8) return reinterpret_cast<const uint8_t*>(im.addr)[i];
  const float v = reinterpret_cast<const float*>(im.addr)[i];
  float t = __fmul_rn(v, 255.f);
  if (rule == 0) t = __fadd_rn(t, 0.5f);
  t = fminf(fmaxf(t, 0.f), 255.f);
  return (unsigned)t;
}

__device__ __forceinline__ unsigned paeth(unsigned a, unsigned b, unsigned c) {
  const int p = (int)a + (int)b - (int)c, pa = abs(p - (int)a), pb = abs(p - (int)b), pc = abs(p - (int)c);
  return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

__device__ __forceinline__ unsigned residual(int f, unsigned x, unsigned a, unsigned b, unsigned c) {
  const unsigned pred = f == 0 ? 0u : f == 1 ? a : f == 2 ? b : f == 3 ? (a + b) >> 1 : paeth(a, b, c);
  return (x - pred) & 255u;
}

__device__ __forceinline__ int find_row(const Img* __restrict__ imgs, int n, long long row) {
  int lo = 0, hi = n - 1;   // last image whose first row <= row
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (imgs[mid].row0 <= row) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(PNG_THREADS) filter_kernel(const Img* __restrict__ imgs, int n, int rule,
                                                             uint8_t* __restrict__ stream) {
  __shared__ unsigned red[5][PNG_THREADS / 32];
  __shared__ int best;
  const Img im = imgs[find_row(imgs, n, blockIdx.x)];
  const long long y = blockIdx.x - im.row0, rb = 3 * im.W;
  uint8_t* out = stream + im.off + y * (1 + rb);
  unsigned s[5] = {0u, 0u, 0u, 0u, 0u};
  for (long long i = threadIdx.x; i < rb; i += PNG_THREADS) {
    const long long x = i / 3;
    const int c = (int)(i - 3 * x);
    const unsigned v = quant(im, rule, y, x, c), a = quant(im, rule, y, x - 1, c), b = quant(im, rule, y - 1, x, c),
                   d = quant(im, rule, y - 1, x - 1, c);
#pragma unroll
    for (int f = 0; f < 5; ++f) {
      const unsigned r = residual(f, v, a, b, d);
      s[f] += r < 128u ? r : 256u - r;
    }
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int f = 0; f < 5; ++f) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s[f] += __shfl_xor_sync(0xffffffffu, s[f], o);
    if (lane == 0) red[f][wid] = s[f];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long mins = ~0ull;
    int bf = 0;
    for (int f = 0; f < 5; ++f) {
      unsigned long long t = 0;
      for (int w = 0; w < PNG_THREADS / 32; ++w) t += red[f][w];
      if (t < mins) { mins = t; bf = f; }
    }
    best = bf;
    out[0] = (uint8_t)bf;
  }
  __syncthreads();
  const int f = best;
  for (long long i = threadIdx.x; i < rb; i += PNG_THREADS) {
    const long long x = i / 3;
    const int c = (int)(i - 3 * x);
    out[1 + i] = (uint8_t)residual(f, quant(im, rule, y, x, c), quant(im, rule, y, x - 1, c), quant(im, rule, y - 1, x, c),
                                   quant(im, rule, y - 1, x - 1, c));
  }
}

// ---- stage 2: deflate -------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned hash3(const uint8_t* p) {
  return (((unsigned)p[0] << 16 | (unsigned)p[1] << 8 | p[2]) * 2654435761u) >> (32 - PNG_HASH_BITS);
}

// deflate's length (257..285) and distance (0..29) codes with their extra bits
__device__ __forceinline__ void len_code(int l, int& code, int& nx, int& xv) {
  if (l == 258) { code = 285; nx = 0; xv = 0; return; }
  const int v = l - 3;
  if (v < 8) { code = 257 + v; nx = 0; xv = 0; return; }
  const int nb = 31 - __clz(v), hi = (v >> (nb - 2)) & 3;
  code = 257 + 4 * (nb - 1) + hi;
  nx = nb - 2;
  xv = v - ((4 | hi) << (nb - 2));
}
__device__ __forceinline__ void dist_code(int d, int& code, int& nx, int& xv) {
  const int v = d - 1;
  if (v < 4) { code = v; nx = 0; xv = 0; return; }
  const int nb = 31 - __clz(v), hi = (v >> (nb - 1)) & 1;
  code = 2 * nb + hi;
  nx = nb - 1;
  xv = v - ((2 | hi) << (nb - 1));
}

__device__ __forceinline__ void put_bits(unsigned* w, unsigned long long pos, unsigned v, int nb) {
  if (nb == 0) return;
  const unsigned sh = pos & 31;
  atomicOr(w + (pos >> 5), v << sh);
  if (sh + nb > 32) atomicOr(w + (pos >> 5) + 1, v >> (32 - sh));
}

struct HuffScratch {
  int A[320];
  short order[320];
  int used, cnt[16], next[16];
};

// Length-limited Huffman code lengths of freq[0..n) (n <= 320) into len[]; every thread of the CTA calls it.  Symbols are
// ranked by (freq, symbol); thread 0 runs Moffat and Katajainen's in-place construction on the sorted weights, then moves
// leaves deeper than `limit` up and lengthens the deepest shorter leaves until the code is complete again.
__device__ void huff_lengths(const unsigned* freq, int n, int limit, uint8_t* len, HuffScratch& h) {
  if (threadIdx.x == 0) h.used = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    len[i] = 0;
    if (freq[i] == 0) continue;
    int r = 0;
    for (int j = 0; j < n; ++j) r += freq[j] != 0 && (freq[j] < freq[i] || (freq[j] == freq[i] && j < i));
    h.order[r] = (short)i;
    h.A[r] = (int)freq[i];
    atomicAdd(&h.used, 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int* A = h.A;
    const int m = h.used;   // >= 2: the callers make sure of it
    A[0] += A[1];
    int root = 0, leaf = 2;
    for (int next = 1; next < m - 1; ++next) {
      if (leaf >= m || A[root] < A[leaf]) { A[next] = A[root]; A[root++] = next; } else A[next] = A[leaf++];
      if (leaf >= m || (root < next && A[root] < A[leaf])) { A[next] += A[root]; A[root++] = next; } else A[next] += A[leaf++];
    }
    A[m - 2] = 0;
    for (int next = m - 3; next >= 0; --next) A[next] = A[A[next]] + 1;
    int avbl = 1, used = 0, dpth = 0, next = m - 1;
    root = m - 2;
    while (avbl > 0) {
      while (root >= 0 && A[root] == dpth) { ++used; --root; }
      while (avbl > used) { A[next--] = dpth; --avbl; }
      avbl = 2 * used;
      ++dpth;
      used = 0;
    }
    int* cnt = h.cnt;
    for (int l = 0; l < 16; ++l) cnt[l] = 0;
    for (int k = 0; k < m; ++k) ++cnt[A[k] > limit ? limit : A[k]];
    unsigned total = 0;
    for (int l = 1; l <= limit; ++l) total += (unsigned)cnt[l] << (limit - l);
    while (total > (1u << limit)) {   // each round: one leaf fewer at `limit`, one leaf moved from l to l + 1 with a sibling
      --cnt[limit];
      for (int l = limit - 1; l > 0; --l)
        if (cnt[l]) { --cnt[l]; cnt[l + 1] += 2; break; }
      --total;
    }
    int k = 0;   // the least frequent symbols take the longest codes
    for (int l = limit; l >= 1; --l)
      for (int c = 0; c < cnt[l]; ++c) len[h.order[k++]] = (uint8_t)l;
  }
  __syncthreads();
}

// canonical codes (RFC 1951 3.2.2), bit-reversed for the LSB-first stream; thread 0 only
__device__ void huff_codes(const uint8_t* len, int n, uint16_t* code, HuffScratch& h) {
  int *cnt = h.cnt, *next = h.next;
  for (int l = 0; l < 16; ++l) cnt[l] = 0;
  for (int i = 0; i < n; ++i) ++cnt[len[i]];
  cnt[0] = 0;
  int c = 0;
  for (int l = 1; l < 16; ++l) { c = (c + cnt[l - 1]) << 1; next[l] = c; }
  for (int i = 0; i < n; ++i)
    code[i] = len[i] ? (uint16_t)(__brev((unsigned)next[len[i]]++) >> (32 - len[i])) : 0;
}

// at least two used symbols, so that every code is complete (a one-symbol code would be a 0-bit code)
__device__ void two_symbols(unsigned* freq, int n) {
  int used = 0;
  for (int i = 0; i < n; ++i) used += freq[i] != 0;
  for (int i = 0; used < 2 && i < n; ++i)
    if (!freq[i]) { freq[i] = 1; ++used; }
}

__device__ __forceinline__ int match_len(const uint8_t* w, int p, int d, int maxlen) {
  int l = 0;
  while (l < maxlen && w[p + l] == w[p - d + l]) ++l;
  return l;
}

// the longest match at segment byte i (window byte h + i) ending by e0, over distances 1, 3, the row stride and the hash
// candidate; 0 when there is none of 3 bytes or more (or only a 3-byte one further than 4 KB back)
__device__ __forceinline__ int best_match(const uint8_t* w, const uint16_t* cand, int h, int i, int e0, int stride, int& bd) {
  const int p = h + i, maxlen = min(258, e0 - i);
  int bl = 0;
  bd = 0;
  if (maxlen < 3) return 0;
  const int ds[4] = {1, 3, stride, (int)cand[i]};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int d = ds[k];
    if (d < 1 || d > p || d > PNG_HIST || bl == maxlen) continue;
    const int l = match_len(w, p, d, maxlen);
    if (l > bl) { bl = l; bd = d; }
  }
  return bl == 3 && bd > 4096 ? 0 : bl;
}

struct DeflateSmem {
  uint8_t win[PNG_WIN];                 // history + segment bytes; then the output bit buffer
  int head[1 << PNG_HASH_BITS];
  unsigned lfreq[286], dfreq[30], cfreq[19];
  uint8_t llen[286 + 30], clen[19];
  uint16_t lcode[286], dcode[30], ccode[19];
  uint16_t rle[286 + 30];               // code-length symbol | extra << 5
  uint8_t seq[286 + 30];
  int n_rle, hlit, hdist, hclen, use_stored;
  unsigned long long hdr_bits, tok_bits;
  unsigned tbits[PNG_THREADS], ntok[PNG_THREADS];
  unsigned long long wsum[PNG_THREADS / 32][2];
  HuffScratch hs;
};

__constant__ uint8_t kClOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

__global__ void __launch_bounds__(PNG_THREADS, 1)
deflate_kernel(const Img* __restrict__ imgs, const Seg* __restrict__ segs, const uint8_t* __restrict__ stream,
               uint16_t* __restrict__ cand_g, unsigned* __restrict__ tok_g, uint8_t* __restrict__ slots,
               long long* __restrict__ meta) {
  extern __shared__ __align__(16) unsigned char dsm[];
  DeflateSmem& S = *reinterpret_cast<DeflateSmem*>(dsm);
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const long long sidx = blockIdx.x;
  const Seg sg = segs[sidx];
  const Img im = imgs[sg.img];
  const int n = (int)sg.len, h = (int)sg.hist;
  const bool last = sg.start + sg.len == stream_len(im.H, im.W);
  const int stride = (int)min(3 * im.W + 1, (long long)PNG_HIST + 1);
  const uint8_t* src = stream + im.off + sg.start - h;
  uint16_t* cand = cand_g + sidx * PNG_SEG;
  unsigned* tok = tok_g + sidx * PNG_SEG;

  for (int i = tid; i < h + n; i += PNG_THREADS) S.win[i] = src[i];
  for (int i = h + n + tid; i < PNG_WIN; i += PNG_THREADS) S.win[i] = 0;
  for (int i = tid; i < (1 << PNG_HASH_BITS); i += PNG_THREADS) S.head[i] = -1;
  for (int i = tid; i < 286; i += PNG_THREADS) S.lfreq[i] = 0;
  if (tid < 30) S.dfreq[tid] = 0;
  if (tid < 19) S.cfreq[tid] = 0;
  __syncthreads();

  // Adler-32 parts of the segment: sum of bytes and sum of (bytes from here to the end) * byte
  {
    const int a = tid * PNG_SUB, e = min(a + PNG_SUB, n);
    unsigned long long s1 = 0, s2 = 0;
    for (int i = a; i < e; ++i) {
      s1 += S.win[h + i];
      s2 += (unsigned long long)(e - i) * S.win[h + i];
    }
    if (e > a) s2 += (unsigned long long)(n - e) * s1;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    if (lane == 0) { S.wsum[wid][0] = s1; S.wsum[wid][1] = s2; }
  }
  // hash candidates: the history first (any order: the head keeps the largest position), then rounds of the segment
  for (int q = tid; q + 2 < h; q += PNG_THREADS) atomicMax(&S.head[hash3(S.win + q)], q);
  __syncthreads();
  if (tid == 0) {
    unsigned long long s1 = 0, s2 = 0;
    for (int w = 0; w < PNG_THREADS / 32; ++w) { s1 += S.wsum[w][0]; s2 += S.wsum[w][1]; }
    meta[sidx * 4 + 1] = (long long)s1;
    meta[sidx * 4 + 2] = (long long)s2;
  }
  for (int r = 0; r < n; r += PNG_ROUND) {
    const int i = r + tid, p = h + i;
    const bool ok = tid < PNG_ROUND && i + 2 < n;
    const unsigned hv = ok ? hash3(S.win + p) : 0u;
    if (tid < PNG_ROUND) {   // whole warps: the nearest earlier lane of the warp with the same hash, else the head table
      const unsigned peers = __match_any_sync(0xffffffffu, ok ? hv : 0x80000000u | lane) & ((1u << lane) - 1u);
      int c = ok ? S.head[hv] : -1;
      if (ok && peers) c = p - (lane - (31 - __clz(peers)));
      if (i < n) cand[i] = (uint16_t)(c >= 0 && p - c <= PNG_HIST ? p - c : 0);   // 32768 is 0x8000, still nonzero
    }
    __syncthreads();
    if (ok) atomicMax(&S.head[hv], p);
    __syncthreads();
  }

  // greedy parse of this thread's bytes, deferring a match by one byte when the next byte starts a longer one
  const int a0 = tid * PNG_SUB, e0 = min(a0 + PNG_SUB, n);
  unsigned nt = 0;
  for (int i = a0; i < e0;) {
    int bd, bl = best_match(S.win, cand, h, i, e0, stride, bd);
    if (bl >= 3 && bl < 258 && i + 1 < e0) {
      int bd1;
      if (best_match(S.win, cand, h, i + 1, e0, stride, bd1) > bl) bl = 0;
    }
    if (bl >= 3) {
      tok[a0 + nt++] = (unsigned)bl << 16 | (unsigned)(bd - 1);
      int c, nx, xv;
      len_code(bl, c, nx, xv);
      atomicAdd(&S.lfreq[c], 1u);
      dist_code(bd, c, nx, xv);
      atomicAdd(&S.dfreq[c], 1u);
      i += bl;
    } else {
      tok[a0 + nt++] = S.win[h + i];
      atomicAdd(&S.lfreq[S.win[h + i]], 1u);
      ++i;
    }
  }
  S.ntok[tid] = nt;
  if (tid == 0) S.lfreq[256] = 1;
  __syncthreads();
  if (tid == 0) {
    two_symbols(S.lfreq, 286);
    two_symbols(S.dfreq, 30);
  }
  __syncthreads();
  huff_lengths(S.lfreq, 286, 15, S.llen, S.hs);
  huff_lengths(S.dfreq, 30, 15, S.llen + 286, S.hs);

  // the header's code lengths, run-length coded (16: repeat the previous 3-6 times, 17 / 18: 3-10 / 11-138 zeros)
  if (tid == 0) {
    huff_codes(S.llen, 286, S.lcode, S.hs);
    huff_codes(S.llen + 286, 30, S.dcode, S.hs);
    int hlit = 286, hdist = 30;
    while (hlit > 257 && !S.llen[hlit - 1]) --hlit;
    while (hdist > 1 && !S.llen[286 + hdist - 1]) --hdist;
    uint8_t* seq = S.seq;
    for (int i = 0; i < hlit; ++i) seq[i] = S.llen[i];
    for (int i = 0; i < hdist; ++i) seq[hlit + i] = S.llen[286 + i];
    const int m = hlit + hdist;
    int nr = 0;
    for (int i = 0; i < m;) {
      const int v = seq[i];
      int run = 1;
      while (i + run < m && seq[i + run] == v) ++run;
      if (v == 0 && run >= 3) {
        const int k = min(run, 138);
        S.rle[nr++] = k >= 11 ? (uint16_t)(18 | (k - 11) << 5) : (uint16_t)(17 | (k - 3) << 5);
        i += k;
      } else if (v != 0 && run >= 4) {
        S.rle[nr++] = (uint16_t)v;
        const int k = min(run - 1, 6);
        S.rle[nr++] = (uint16_t)(16 | (k - 3) << 5);
        i += 1 + k;
      } else {
        S.rle[nr++] = (uint16_t)v;
        i += 1;
      }
    }
    for (int i = 0; i < nr; ++i) ++S.cfreq[S.rle[i] & 31];
    two_symbols(S.cfreq, 19);
    S.n_rle = nr;
    S.hlit = hlit;
    S.hdist = hdist;
  }
  __syncthreads();
  huff_lengths(S.cfreq, 19, 7, S.clen, S.hs);

  // bits of this thread's tokens
  unsigned long long bits = 0;
  for (unsigned k = 0; k < nt; ++k) {
    const unsigned t = tok[a0 + k];
    if (t >> 16) {
      int c, nx, xv;
      len_code((int)(t >> 16), c, nx, xv);
      bits += S.llen[c] + nx;
      dist_code((int)(t & 0xffff) + 1, c, nx, xv);
      bits += S.llen[286 + c] + nx;
    } else {
      bits += S.llen[t];
    }
  }
  S.tbits[tid] = (unsigned)bits;   // at most 256 tokens of 48 bits
  if (tid == 0) {
    huff_codes(S.clen, 19, S.ccode, S.hs);
    int hclen = 19;
    while (hclen > 4 && !S.clen[kClOrder[hclen - 1]]) --hclen;
    S.hclen = hclen;
    unsigned long long hb = 3 + 5 + 5 + 4 + 3ull * hclen;
    for (int i = 0; i < S.n_rle; ++i) {
      const int s = S.rle[i] & 31;
      hb += S.clen[s] + (s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0);
    }
    S.hdr_bits = hb;
  }
  __syncthreads();
  if (tid == 0) {
    unsigned long long acc = S.hdr_bits;
    for (int t = 0; t < PNG_THREADS; ++t) {   // exclusive scan, in place
      const unsigned b = S.tbits[t];
      S.tbits[t] = (unsigned)(acc - S.hdr_bits);
      acc += b;
    }
    S.tok_bits = acc - S.hdr_bits;
    const unsigned long long dyn_bits = acc + S.llen[256];
    const long long dyn = last ? (long long)((dyn_bits + 7) >> 3) : (long long)((dyn_bits + 3 + 7) >> 3) + 4;
    const long long nblk = (n + 65534) / 65535;
    const long long stored = n + 5 * nblk + (last ? 0 : 5);
    S.use_stored = stored <= dyn;
    meta[sidx * 4 + 0] = S.use_stored ? stored : dyn;
    meta[sidx * 4 + 3] = S.use_stored;
  }
  __syncthreads();
  uint8_t* slot = slots + sidx * PNG_SLOT;
  if (S.use_stored) {
    const long long nblk = (n + 65534) / 65535;
    for (int i = tid; i < n; i += PNG_THREADS) {
      const long long b = i / 65535;
      slot[i + 5 * (b + 1)] = S.win[h + i];
    }
    if (tid < nblk) {
      const int b = tid, bl = min(65535, n - 65535 * b);
      uint8_t* o = slot + (long long)b * (65535 + 5);
      o[0] = (uint8_t)(last && b == nblk - 1);
      o[1] = (uint8_t)bl; o[2] = (uint8_t)(bl >> 8); o[3] = (uint8_t)~bl; o[4] = (uint8_t)(~bl >> 8);
    }
    if (!last && tid == 0) {
      uint8_t* o = slot + n + 5 * nblk;
      o[0] = 0; o[1] = 0; o[2] = 0; o[3] = 0xff; o[4] = 0xff;
    }
    return;
  }
  unsigned* wb = reinterpret_cast<unsigned*>(S.win);
  for (int i = tid; i < PNG_WIN / 4; i += PNG_THREADS) wb[i] = 0u;
  __syncthreads();
  if (tid == 0) {   // block header: BFINAL, BTYPE = 2, HLIT, HDIST, HCLEN, the code-length code and the coded lengths
    unsigned long long pos = 0;
    put_bits(wb, pos, (last ? 1u : 0u) | 2u << 1, 3); pos += 3;
    put_bits(wb, pos, S.hlit - 257, 5); pos += 5;
    put_bits(wb, pos, S.hdist - 1, 5); pos += 5;
    put_bits(wb, pos, S.hclen - 4, 4); pos += 4;
    for (int i = 0; i < S.hclen; ++i) { put_bits(wb, pos, S.clen[kClOrder[i]], 3); pos += 3; }
    for (int i = 0; i < S.n_rle; ++i) {
      const int s = S.rle[i] & 31, x = S.rle[i] >> 5;
      put_bits(wb, pos, S.ccode[s], S.clen[s]); pos += S.clen[s];
      const int nx = s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0;
      put_bits(wb, pos, x, nx); pos += nx;
    }
    const unsigned long long eob = S.hdr_bits + S.tok_bits;
    put_bits(wb, eob, S.lcode[256], S.llen[256]);
    if (!last) {   // empty stored block: 3 zero bits, padding, LEN 0, NLEN 0xffff
      const unsigned long long byte = (eob + S.llen[256] + 3 + 7) >> 3;
      put_bits(wb, 8 * byte + 16, 0xffffu, 16);
    }
  }
  {
    unsigned long long pos = S.hdr_bits + S.tbits[tid];
    for (unsigned k = 0; k < nt; ++k) {
      const unsigned t = tok[a0 + k];
      if (t >> 16) {
        int c, nx, xv;
        len_code((int)(t >> 16), c, nx, xv);
        put_bits(wb, pos, S.lcode[c] | (unsigned)xv << S.llen[c], S.llen[c] + nx);
        pos += S.llen[c] + nx;
        dist_code((int)(t & 0xffff) + 1, c, nx, xv);
        put_bits(wb, pos, S.dcode[c] | (unsigned)xv << S.llen[286 + c], S.llen[286 + c] + nx);
        pos += S.llen[286 + c] + nx;
      } else {
        put_bits(wb, pos, S.lcode[t], S.llen[t]);
        pos += S.llen[t];
      }
    }
  }
  __syncthreads();
  const long long nb = meta[sidx * 4 + 0];
  for (long long i = tid; i < nb; i += PNG_THREADS) slot[i] = S.win[i];
}

// ---- stages 3 and 4: packing and the container ------------------------------------------------------------------------
__device__ __forceinline__ long long piece_bytes(long long comp, bool first, bool last) {
  return 12 + comp + (first ? 8 + 25 + 2 : 0) + (last ? 4 + 12 : 0);
}

__global__ void __launch_bounds__(1024) scan_kernel(const Img* __restrict__ imgs, int n_img, const Seg* __restrict__ segs,
                                                    long long n_seg, const long long* __restrict__ meta,
                                                    long long* __restrict__ piece_off, long long* __restrict__ files) {
  __shared__ long long warp_tot[32];
  __shared__ long long carry;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) carry = 0;
  __syncthreads();
  for (long long base = 0; base < n_seg; base += 1024) {
    const long long s = base + tid;
    long long v = 0;
    if (s < n_seg) {
      const Seg sg = segs[s];
      const Img im = imgs[sg.img];
      v = piece_bytes(meta[s * 4], s == im.seg0, s == im.seg0 + im.n_seg - 1);
    }
    long long x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) warp_tot[wid] = x;
    __syncthreads();
    if (wid == 0) {
      long long t = warp_tot[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const long long y = __shfl_up_sync(0xffffffffu, t, o);
        if (lane >= o) t += y;
      }
      warp_tot[lane] = t;
    }
    __syncthreads();
    const long long incl = carry + x + (wid ? warp_tot[wid - 1] : 0);
    if (s < n_seg) piece_off[s] = incl - v;
    __syncthreads();
    if (tid == 1023) carry = incl;
    __syncthreads();
  }
  for (int i = tid; i < n_img; i += 1024) {
    const Img im = imgs[i];
    const long long e = im.seg0 + im.n_seg - 1;
    files[2 * i] = piece_off[im.seg0];
    files[2 * i + 1] = piece_off[e] + piece_bytes(meta[e * 4], im.n_seg == 1, true) - piece_off[im.seg0];
  }
}

__device__ unsigned crc_update(const unsigned* tab, unsigned c, const uint8_t* p, long long n) {
  for (long long i = 0; i < n; ++i) c = tab[(c ^ p[i]) & 255u] ^ (c >> 8);
  return c;
}

// a * b mod the CRC-32 polynomial, both in the reflected representation (x^0 is bit 31)
__device__ unsigned gf2_mul(unsigned a, unsigned b) {
  unsigned p = 0;
  for (int k = 0; k < 32; ++k) {
    if (a & (0x80000000u >> k)) p ^= b;
    b = (b & 1u) ? (b >> 1) ^ 0xedb88320u : b >> 1;
  }
  return p;
}

// the CRC register c advanced over n zero bytes: c * x^(8n)
__device__ unsigned crc_shift(unsigned c, unsigned long long n) {
  unsigned r = 0x80000000u, x = 0x00800000u;   // x^0, x^8
  for (; n; n >>= 1) {
    if (n & 1) r = gf2_mul(r, x);
    x = gf2_mul(x, x);
  }
  return gf2_mul(r, c);
}

__device__ __forceinline__ void be32(uint8_t* o, unsigned v) {
  o[0] = (uint8_t)(v >> 24); o[1] = (uint8_t)(v >> 16); o[2] = (uint8_t)(v >> 8); o[3] = (uint8_t)v;
}

__global__ void __launch_bounds__(PNG_THREADS) container_kernel(const Img* __restrict__ imgs, const Seg* __restrict__ segs,
                                                                const long long* __restrict__ meta,
                                                                const uint8_t* __restrict__ slots,
                                                                const long long* __restrict__ piece_off,
                                                                uint8_t* __restrict__ out) {
  __shared__ unsigned tab[256];
  __shared__ unsigned crc_part[PNG_THREADS / 32];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const long long s = blockIdx.x;
  const Seg sg = segs[s];
  const Img im = imgs[sg.img];
  const bool first = s == im.seg0, last = s == im.seg0 + im.n_seg - 1;
  {
    unsigned c = tid;
    for (int k = 0; k < 8; ++k) c = (c & 1u) ? (c >> 1) ^ 0xedb88320u : c >> 1;
    tab[tid] = c;
  }
  __syncthreads();
  const long long comp = meta[s * 4];
  uint8_t* o = out + piece_off[s];
  if (first) {
    if (tid == 0) {
      const uint8_t sig[8] = {137, 80, 78, 71, 13, 10, 26, 10};
      for (int i = 0; i < 8; ++i) o[i] = sig[i];
      uint8_t* c = o + 8;
      be32(c, 13);
      c[4] = 'I'; c[5] = 'H'; c[6] = 'D'; c[7] = 'R';
      be32(c + 8, (unsigned)im.W);
      be32(c + 12, (unsigned)im.H);
      c[16] = 8; c[17] = 2; c[18] = 0; c[19] = 0; c[20] = 0;   // 8-bit RGB, deflate, adaptive filtering, no interlace
      be32(c + 21, crc_update(tab, 0xffffffffu, c + 4, 17) ^ 0xffffffffu);
    }
    o += 33;
  }
  const long long data = comp + (first ? 2 : 0) + (last ? 4 : 0);
  uint8_t* d = o + 8 + (first ? 2 : 0);
  const uint8_t* slot = slots + s * PNG_SLOT;
  for (long long i = tid; i < comp; i += PNG_THREADS) d[i] = slot[i];
  if (tid == 0) {
    be32(o, (unsigned)data);
    o[4] = 'I'; o[5] = 'D'; o[6] = 'A'; o[7] = 'T';
    if (first) { o[8] = 0x78; o[9] = 0x9c; }   // zlib header: deflate, 32 KB window, default level, check bits
    if (last) {   // Adler-32 of the image's stream from its segments' parts (see the C header for the combination)
      const unsigned M = 65521u;
      const long long N = stream_len(im.H, im.W);
      unsigned long long A = 1, B = (unsigned long long)(N % M);
      for (long long k = im.seg0; k <= s; ++k) {
        const Seg q = segs[k];
        const unsigned long long S1 = (unsigned long long)meta[k * 4 + 1] % M, S2 = (unsigned long long)meta[k * 4 + 2] % M;
        const unsigned long long after = (unsigned long long)(N - q.start - q.len) % M;
        A = (A + S1) % M;
        B = (B + S2 + after * S1) % M;
      }
      be32(d + comp, (unsigned)(B << 16 | A));
    }
  }
  __syncthreads();
  // CRC over the type and data: per-thread slices combined by shifting each slice's register over the bytes after it
  const long long L = 4 + data, per = (L + PNG_THREADS - 1) / PNG_THREADS;
  const long long a = min(L, tid * per), e = min(L, a + per);
  unsigned c = crc_update(tab, 0u, o + 4 + a, e - a);
  c = crc_shift(c, (unsigned long long)(L - e));
  if (tid == 0) c ^= crc_shift(0xffffffffu, (unsigned long long)L);
#pragma unroll
  for (int k = 16; k > 0; k >>= 1) c ^= __shfl_xor_sync(0xffffffffu, c, k);
  if (lane == 0) crc_part[wid] = c;
  __syncthreads();
  if (tid == 0) {
    unsigned crc = 0xffffffffu;
    for (int w = 0; w < PNG_THREADS / 32; ++w) crc ^= crc_part[w];
    uint8_t* t = o + 8 + data;
    be32(t, crc);
    if (last) {
      const uint8_t iend[12] = {0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xae, 0x42, 0x60, 0x82};
      for (int i = 0; i < 12; ++i) t[4 + i] = iend[i];
    }
  }
}

struct Layout {
  long long n_seg, rows, stream;
  size_t off_segs, off_meta, off_piece, off_stream, off_cand, off_tok, off_slots, staged, total;
};

size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

int check_images(const int64_t* images, int n, int rule) {
  P2PVG_REQUIRE(n >= 0, P2PVG_ERR_BAD_ARG, "png_encode: n = %d", n);
  P2PVG_REQUIRE(rule == 0 || rule == 1, P2PVG_ERR_BAD_ARG, "png_encode: rule %d (0 save_image, 1 tensorboard)", rule);
  P2PVG_REQUIRE(n == 0 || images, P2PVG_ERR_BAD_ARG, "png_encode: null image table");
  for (int i = 0; i < n; ++i) {
    const int64_t* r = images + 5 * i;
    P2PVG_REQUIRE(r[0] != 0, P2PVG_ERR_BAD_ARG, "png_encode: image %d: null address", i);
    P2PVG_REQUIRE(r[1] == P2PVG_F32 || r[1] == PNG_U8, P2PVG_ERR_BAD_ARG, "png_encode: image %d: dtype %lld", i,
                  (long long)r[1]);
    P2PVG_REQUIRE(r[1] != P2PVG_F32 || (r[0] & 3) == 0, P2PVG_ERR_BAD_ARG, "png_encode: image %d: misaligned fp32", i);
    P2PVG_REQUIRE(r[2] == 1 || r[2] == 3, P2PVG_ERR_BAD_ARG, "png_encode: image %d: %lld channels (1 or 3)", i,
                  (long long)r[2]);
    P2PVG_REQUIRE(r[3] >= 1 && r[4] >= 1, P2PVG_ERR_BAD_ARG, "png_encode: image %d: %lld x %lld", i, (long long)r[3],
                  (long long)r[4]);
    P2PVG_REQUIRE(r[3] < (1LL << 24) && r[4] < (1LL << 24) && stream_len(r[3], r[4]) < (1LL << 40),
                  P2PVG_ERR_UNSUPPORTED, "png_encode: image %d: %lld x %lld is too large", i, (long long)r[3],
                  (long long)r[4]);
  }
  return P2PVG_OK;
}

Layout layout(const int64_t* images, int n) {
  Layout L{};
  for (int i = 0; i < n; ++i) {
    const long long N = stream_len(images[5 * i + 3], images[5 * i + 4]);
    L.n_seg += (N + PNG_SEG - 1) / PNG_SEG;
    L.rows += images[5 * i + 3];
    L.stream += N;
  }
  L.off_segs = align256(sizeof(Img) * n);
  L.staged = L.off_segs + sizeof(Seg) * L.n_seg;
  L.off_meta = align256(L.staged);
  L.off_piece = L.off_meta + align256(sizeof(long long) * 4 * L.n_seg);
  L.off_stream = L.off_piece + align256(sizeof(long long) * L.n_seg);
  L.off_cand = L.off_stream + align256(L.stream + 8);
  L.off_tok = L.off_cand + align256(sizeof(uint16_t) * PNG_SEG * L.n_seg);
  L.off_slots = L.off_tok + align256(sizeof(unsigned) * PNG_SEG * L.n_seg);
  L.total = L.off_slots + (size_t)PNG_SLOT * L.n_seg;
  return L;
}

size_t out_bound(const int64_t* images, int n) {
  size_t b = 0;
  for (int i = 0; i < n; ++i) {
    const long long N = stream_len(images[5 * i + 3], images[5 * i + 4]);
    b += (size_t)N + 64 * (size_t)((N + PNG_SEG - 1) / PNG_SEG) + 64;
  }
  return b;
}

}  // namespace

extern "C" size_t p2pvg_png_workspace_bytes(const int64_t* images, int n) {
  if (check_images(images, n, 0) != P2PVG_OK) return 0;
  return layout(images, n).total;
}

extern "C" size_t p2pvg_png_out_bytes(const int64_t* images, int n) {
  if (check_images(images, n, 0) != P2PVG_OK) return 0;
  return out_bound(images, n);
}

extern "C" int p2pvg_png_encode(const int64_t* images, int n, int rule, void* ws, size_t ws_bytes, uint8_t* out, size_t out_bytes,
                                int64_t* files, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const int rc = check_images(images, n, rule);
  if (rc != P2PVG_OK) return rc;
  if (n == 0) return P2PVG_OK;
  P2PVG_REQUIRE(ws && out && files, P2PVG_ERR_BAD_ARG, "png_encode: null workspace, output or file table");
  P2PVG_REQUIRE(((uintptr_t)ws & 255) == 0 && ((uintptr_t)files & 7) == 0, P2PVG_ERR_BAD_ARG,
                "png_encode: workspace must be 256-byte, files 8-byte aligned");
  const Layout L = layout(images, n);
  P2PVG_REQUIRE(ws_bytes >= L.total, P2PVG_ERR_WORKSPACE, "png_encode: workspace %zu bytes, needs %zu", ws_bytes, L.total);
  const size_t bound = out_bound(images, n);
  P2PVG_REQUIRE(out_bytes >= bound, P2PVG_ERR_WORKSPACE, "png_encode: output %zu bytes, needs %zu", out_bytes, bound);
  std::vector<unsigned char> host(L.staged, 0);
  Img* it = reinterpret_cast<Img*>(host.data());
  Seg* sg = reinterpret_cast<Seg*>(host.data() + L.off_segs);
  long long off = 0, row0 = 0, s = 0;
  for (int i = 0; i < n; ++i) {
    const int64_t* r = images + 5 * i;
    const long long N = stream_len(r[3], r[4]), ns = (N + PNG_SEG - 1) / PNG_SEG;
    it[i] = Img{r[0], r[1], r[2], r[3], r[4], off, row0, s, ns};
    for (long long k = 0; k < ns; ++k, ++s) {
      const long long start = k * PNG_SEG;
      sg[s] = Seg{i, start, std::min((long long)PNG_SEG, N - start), std::min((long long)PNG_HIST, start)};
    }
    off += N;
    row0 += r[3];
  }
  unsigned char* w = static_cast<unsigned char*>(ws);
  cudaError_t err = cudaMemcpyAsync(w, host.data(), L.staged, cudaMemcpyHostToDevice, st);
  if (err != cudaSuccess) {
    p2pvg_set_error("png_encode: table upload: %s", cudaGetErrorString(err));
    return P2PVG_ERR_CUDA;
  }
  const Img* d_img = reinterpret_cast<const Img*>(w);
  const Seg* d_seg = reinterpret_cast<const Seg*>(w + L.off_segs);
  long long* meta = reinterpret_cast<long long*>(w + L.off_meta);
  long long* piece = reinterpret_cast<long long*>(w + L.off_piece);
  uint8_t* filtered = w + L.off_stream;
  uint8_t* slots = w + L.off_slots;

  int dev = 0;
  cudaGetDevice(&dev);
  static unsigned long long attr_set = 0;   // per device
  if (dev >= 64 || !((attr_set >> dev) & 1ULL)) {
    err = cudaFuncSetAttribute(deflate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(DeflateSmem));
    if (err != cudaSuccess) {
      p2pvg_set_error("png_encode: shared-memory attribute: %s", cudaGetErrorString(err));
      return P2PVG_ERR_CUDA;
    }
    if (dev < 64) attr_set |= 1ULL << dev;
  }
  filter_kernel<<<(unsigned)L.rows, PNG_THREADS, 0, st>>>(d_img, n, rule, filtered);
  deflate_kernel<<<(unsigned)L.n_seg, PNG_THREADS, sizeof(DeflateSmem), st>>>(
      d_img, d_seg, filtered, reinterpret_cast<uint16_t*>(w + L.off_cand), reinterpret_cast<unsigned*>(w + L.off_tok), slots,
      meta);
  scan_kernel<<<1, 1024, 0, st>>>(d_img, n, d_seg, L.n_seg, meta, piece, reinterpret_cast<long long*>(files));
  container_kernel<<<(unsigned)L.n_seg, PNG_THREADS, 0, st>>>(d_img, d_seg, meta, slots, piece, out);
  return p2pvg_check_launch("png_encode");
}
