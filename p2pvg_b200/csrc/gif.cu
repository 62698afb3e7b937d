// GIF89a files of a batch of animations (include/p2pvg_b200.h, p2pvg_gif_encode), every per-pixel stage on the device.
//
//   1. colours_kernel (one CTA per GIF_CHUNK pixels of a frame): quantise each pixel to a 24-bit RGB key and count it in
//      the frame's open-addressing hash table (key << 32 | count); a warp counts equal keys once.
//   2. compact_kernel (one CTA per GIF_CHUNK hash slots): the frame's distinct colours as a list, in slot-claim order.
//   3. palette_kernel (one CTA per frame): at most 256 colours, those colours sorted by key; more, median cut (split the box
//      of largest count-weighted squared error along its widest channel at the count-weighted median, from a 256-bin
//      histogram) to 256 boxes, their rounded means, then GIF_LLOYD Lloyd iterations over the distinct colours.  Every sum
//      is an integer sum and every tie goes to the lower box / entry index, so the list's order never shows in the palette.
//   4. index_kernel (one CTA per GIF_CHUNK pixels): each pixel's nearest palette entry (squared RGB distance, lowest index
//      on ties).
//   5. lzw_kernel (one thread per segment of GIF_SEG pixels, its dictionary in shared memory): GIF LZW with minimum code size
//      8 from the post-clear state; the segment ends with a CLEAR (an EOI after the frame's last segment), so the bits of a
//      segment depend on its pixels alone.  A full table (4096 codes) emits a CLEAR at 12 bits.
//   6. plan_kernel (one CTA): the segments' bit offsets in their frame, the frames' byte counts and the packing offsets.
//   7. pack_kernel (one warp per segment): the codes LSB-first at their bit offsets.
//   8. container_kernel (one CTA per frame): header, logical screen and NETSCAPE2.0 loop block in front of an animation's
//      first frame; the graphic control extension, image descriptor, local colour table and data sub-blocks of every frame;
//      the trailer after the last.
#include "common.cuh"

#include <algorithm>
#include <vector>

#define GIF_SEG 65536            // pixels per LZW segment (P2PVG_GIF_SEGMENT in the header)
#define GIF_U8 3                 // P2PVG_PNG_U8
#define GIF_THREADS 256
#define GIF_PER 16
#define GIF_CHUNK (GIF_THREADS * GIF_PER)
#define GIF_LLOYD 3
#define GIF_TAB 8192             // LZW dictionary hash slots per segment
#define GIF_PAL_THREADS 512
#define GIF_HDR 32               // "GIF89a", logical screen descriptor, NETSCAPE2.0 block
#define GIF_FRAME_HDR (8 + 10 + 768 + 1)   // graphic control extension, image descriptor, colour table, LZW code size

namespace {

constexpr unsigned long long EMPTY = ~0ull;
constexpr unsigned NO_KEY = 0xffffffffu;   // keys are < 2^24

struct Frame {   // one frame with its place in the workspace and the output
  long long src, dtype, anim, t, T, H, W, N, hoff, hcap, coff, chunk0, hchunk0, seg0, n_seg, soff, delay, loop;
};
struct Seg {     // pixels [start, start + len) of a frame; its codes at coff
  long long frame, start, len, coff;
};

__host__ __device__ inline long long seg_codes(long long len) { return len + len / 3838 + 3; }

__device__ __forceinline__ unsigned quant(const Frame& f, int rule, long long i) {
  const float v = reinterpret_cast<const float*>(f.src)[i];
  float t = __fmul_rn(v, 255.f);
  if (rule == 0) t = __fadd_rn(t, 0.5f);
  t = fminf(fmaxf(t, 0.f), 255.f);
  return (unsigned)t;
}

__device__ __forceinline__ unsigned pixel_key(const Frame& f, int rule, long long p) {
  if (f.dtype == GIF_U8) {
    const uint8_t* s = reinterpret_cast<const uint8_t*>(f.src) + 3 * p;
    return (unsigned)s[0] << 16 | (unsigned)s[1] << 8 | s[2];
  }
  return quant(f, rule, p) << 16 | quant(f, rule, f.N + p) << 8 | quant(f, rule, 2 * f.N + p);
}

__device__ __forceinline__ int find_frame(const Frame* __restrict__ fr, int n, long long chunk, bool hash) {
  int lo = 0, hi = n - 1;   // last frame whose first chunk <= chunk
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if ((hash ? fr[mid].hchunk0 : fr[mid].chunk0) <= chunk) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ unsigned hash_key(unsigned key) { return key * 2654435761u; }   // use the high bits

__device__ __forceinline__ unsigned mix(unsigned k) {   // murmur3's finaliser: every bit of the key reaches the low bits
  k ^= k >> 16; k *= 0x85ebca6bu; k ^= k >> 13; k *= 0xc2b2ae35u; k ^= k >> 16;
  return k;
}

// ---- stage 1: colour counts -------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(GIF_THREADS) colours_kernel(const Frame* __restrict__ frames, int nf, int rule,
                                                              unsigned long long* __restrict__ hash, unsigned* __restrict__ ncol) {
  const int fi = find_frame(frames, nf, blockIdx.x, false);
  const Frame f = frames[fi];
  const long long base = (blockIdx.x - f.chunk0) * (long long)GIF_CHUNK;
  unsigned long long* tab = hash + f.hoff;
  const unsigned mask = (unsigned)(f.hcap - 1);
  const int lane = threadIdx.x & 31;
  for (int k = 0; k < GIF_PER; ++k) {
    const long long p = base + k * GIF_THREADS + threadIdx.x;
    const bool ok = p < f.N;
    const unsigned key = ok ? pixel_key(f, rule, p) : NO_KEY;
    const unsigned peers = __match_any_sync(0xffffffffu, key);
    if (!ok || lane != __ffs(peers) - 1) continue;
    const unsigned long long add = __popc(peers);
    unsigned h = mix(key) & mask;
    for (;;) {
      const unsigned long long s = *reinterpret_cast<volatile unsigned long long*>(tab + h);
      if ((unsigned)(s >> 32) == key) { atomicAdd(tab + h, add); break; }
      if (s == EMPTY) {
        const unsigned long long prev = atomicCAS(tab + h, EMPTY, (unsigned long long)key << 32 | add);
        if (prev == EMPTY) { atomicAdd(ncol + fi, 1u); break; }
        if ((unsigned)(prev >> 32) == key) { atomicAdd(tab + h, add); break; }
      }
      h = (h + 1) & mask;
    }
  }
}

// ---- stage 2: the distinct colours as a list ----------------------------------------------------------------------------
__global__ void __launch_bounds__(GIF_THREADS) compact_kernel(const Frame* __restrict__ frames, int nf,
                                                              const unsigned long long* __restrict__ hash,
                                                              unsigned* __restrict__ fill, unsigned long long* __restrict__ cols) {
  const int fi = find_frame(frames, nf, blockIdx.x, true);
  const Frame f = frames[fi];
  const long long base = (blockIdx.x - f.hchunk0) * (long long)GIF_CHUNK;
  const int lane = threadIdx.x & 31;
  for (int k = 0; k < GIF_PER; ++k) {
    const long long i = base + k * GIF_THREADS + threadIdx.x;
    const unsigned long long s = hash[f.hoff + i];
    const unsigned used = __ballot_sync(0xffffffffu, s != EMPTY);
    if (!used) continue;
    unsigned pos = 0;
    if (lane == __ffs(used) - 1) pos = atomicAdd(fill + fi, (unsigned)__popc(used));
    pos = __shfl_sync(0xffffffffu, pos, __ffs(used) - 1);
    if (s != EMPTY) cols[f.coff + pos + __popc(used & ((1u << lane) - 1u))] = s;
  }
}

// ---- stage 3: the palette ---------------------------------------------------------------------------------------------
struct Acc {   // count, per-channel sum and sum of squares (count-weighted), min and max of a set of colours
  unsigned long long c, s[3], q[3];
  int mn[3], mx[3];
};
struct Box {
  long long b, e;
  Acc a;
  double sse;
};

__device__ __forceinline__ int chan(unsigned long long col, int c) { return (int)(col >> (32 + 8 * (2 - c))) & 255; }

__device__ __forceinline__ void acc_init(Acc& a) {
  a.c = 0;
#pragma unroll
  for (int c = 0; c < 3; ++c) { a.s[c] = 0; a.q[c] = 0; a.mn[c] = 255; a.mx[c] = 0; }
}
__device__ __forceinline__ void acc_add(Acc& a, unsigned long long col) {
  const unsigned long long n = (unsigned)col;
  a.c += n;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int v = chan(col, c);
    a.s[c] += n * v;
    a.q[c] += n * (unsigned long long)(v * v);
    a.mn[c] = min(a.mn[c], v);
    a.mx[c] = max(a.mx[c], v);
  }
}
// a thread's partial into the shared total (initialised by acc_init), through a warp reduction
__device__ void acc_merge(Acc& a, Acc* tot) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a.c += __shfl_xor_sync(0xffffffffu, a.c, o);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      a.s[c] += __shfl_xor_sync(0xffffffffu, a.s[c], o);
      a.q[c] += __shfl_xor_sync(0xffffffffu, a.q[c], o);
      a.mn[c] = min(a.mn[c], __shfl_xor_sync(0xffffffffu, a.mn[c], o));
      a.mx[c] = max(a.mx[c], __shfl_xor_sync(0xffffffffu, a.mx[c], o));
    }
  }
  if ((threadIdx.x & 31) == 0 && a.c) {
    atomicAdd(&tot->c, a.c);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      atomicAdd(&tot->s[c], a.s[c]);
      atomicAdd(&tot->q[c], a.q[c]);
      atomicMin(&tot->mn[c], a.mn[c]);
      atomicMax(&tot->mx[c], a.mx[c]);
    }
  }
}

// count-weighted squared error about the mean: sum over channels of (c q - s^2) / c, the numerators exact
__device__ double box_sse(const Acc& a) {
  double e = 0.0;
  for (int c = 0; c < 3; ++c) {
    const unsigned __int128 num = (unsigned __int128)a.c * a.q[c] - (unsigned __int128)a.s[c] * a.s[c];
    e += (double)num;
  }
  return e / (double)a.c;
}

__device__ __forceinline__ int nearest(const int* pr, const int* pg, const int* pb, int r, int g, int b) {
  int best = 0, bd = 0x7fffffff;
  for (int j = 0; j < 256; ++j) {
    const int dr = r - pr[j], dg = g - pg[j], db = b - pb[j], d = dr * dr + dg * dg + db * db;
    if (d < bd) { bd = d; best = j; if (d == 0) break; }
  }
  return best;
}

struct PaletteSmem {
  Box box[256];
  unsigned long long hist[256];
  unsigned long long lc[256], ls[256][3];
  int pr[256], pg[256], pb[256];
  unsigned keys[256];
  Acc accL, accR;
  unsigned lcur, rcur;
  int sel, ch, thr, nbox;
};

__global__ void __launch_bounds__(GIF_PAL_THREADS, 1)
palette_kernel(const Frame* __restrict__ frames, const unsigned* __restrict__ ncol, unsigned long long* __restrict__ cols,
               unsigned long long* __restrict__ hash, unsigned* __restrict__ pal) {
  extern __shared__ __align__(16) unsigned char psm[];
  PaletteSmem& S = *reinterpret_cast<PaletteSmem*>(psm);
  const int fi = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const Frame f = frames[fi];
  const long long n = ncol[fi];
  unsigned long long* A = cols + f.coff;
  unsigned long long* tmp = hash + f.hoff;   // the hash table is no longer needed: partition scratch
  unsigned* out = pal + 256LL * fi;

  if (n <= 256) {   // lossless: the colours sorted by key, the rest of the table black
    if (tid < n) S.keys[tid] = (unsigned)(A[tid] >> 32);
    __syncthreads();
    if (tid < 256) out[tid] = 0u;
    __syncthreads();
    if (tid < n) {
      int r = 0;
      for (int j = 0; j < n; ++j) r += S.keys[j] < S.keys[tid];
      out[r] = S.keys[tid];
    }
    return;
  }

  if (tid == 0) { acc_init(S.accL); S.nbox = 1; }
  __syncthreads();
  {
    Acc a;
    acc_init(a);
    for (long long i = tid; i < n; i += GIF_PAL_THREADS) acc_add(a, A[i]);
    acc_merge(a, &S.accL);
  }
  __syncthreads();
  if (tid == 0) { S.box[0] = Box{0, n, S.accL, box_sse(S.accL)}; }
  __syncthreads();

  while (S.nbox < 256) {
    if (wid == 0) {   // the box of largest error that holds two colours or more, lowest index on ties
      double bs = -1.0;
      int bi = -1;
      for (int j = lane; j < S.nbox; j += 32)
        if (S.box[j].e - S.box[j].b > 1 && S.box[j].sse > bs) { bs = S.box[j].sse; bi = j; }
      for (int o = 16; o > 0; o >>= 1) {
        const double os = __shfl_xor_sync(0xffffffffu, bs, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (oi >= 0 && (os > bs || (os == bs && (bi < 0 || oi < bi)))) { bs = os; bi = oi; }
      }
      if (lane == 0) {
        S.sel = bi;
        if (bi >= 0) {
          const Acc& a = S.box[bi].a;
          int ch = 0;
          for (int c = 1; c < 3; ++c)
            if (a.mx[c] - a.mn[c] > a.mx[ch] - a.mn[ch]) ch = c;
          S.ch = ch;
        }
      }
    }
    if (tid < 256) S.hist[tid] = 0;
    __syncthreads();
    const int sel = S.sel;
    if (sel < 0) break;
    const int ch = S.ch;
    const long long bb = S.box[sel].b, be = S.box[sel].e;
    for (long long i = bb + tid; i < be; i += GIF_PAL_THREADS) atomicAdd(&S.hist[chan(A[i], ch)], (unsigned long long)(unsigned)A[i]);
    __syncthreads();
    if (tid == 0) {   // the count-weighted median, kept below the box's largest value so that both halves hold colours
      const Acc& a = S.box[sel].a;
      unsigned long long cum = 0;
      int t = a.mx[ch] - 1;
      for (int v = a.mn[ch]; v < a.mx[ch]; ++v) {
        cum += S.hist[v];
        if (2 * cum >= a.c) { t = v; break; }
      }
      S.thr = t;
      S.lcur = 0;
      S.rcur = 0;
      acc_init(S.accL);
      acc_init(S.accR);
    }
    __syncthreads();
    {
      const int t = S.thr;
      Acc l, r;
      acc_init(l);
      acc_init(r);
      for (long long i = bb + tid; i < be; i += GIF_PAL_THREADS) {
        const unsigned long long col = A[i];
        if (chan(col, ch) <= t) { tmp[bb + atomicAdd(&S.lcur, 1u)] = col; acc_add(l, col); }
        else { tmp[be - 1 - atomicAdd(&S.rcur, 1u)] = col; acc_add(r, col); }
      }
      acc_merge(l, &S.accL);
      acc_merge(r, &S.accR);
    }
    __syncthreads();
    for (long long i = bb + tid; i < be; i += GIF_PAL_THREADS) A[i] = tmp[i];
    if (tid == 0) {
      const long long m = bb + S.lcur;
      S.box[sel] = Box{bb, m, S.accL, box_sse(S.accL)};
      S.box[S.nbox] = Box{m, be, S.accR, box_sse(S.accR)};
      S.nbox += 1;
    }
    __syncthreads();
  }

  if (tid < 256) {   // box means, rounded; a table of fewer boxes repeats its last mean
    const Acc& a = S.box[min(tid, S.nbox - 1)].a;
    S.pr[tid] = (int)((a.s[0] + a.c / 2) / a.c);
    S.pg[tid] = (int)((a.s[1] + a.c / 2) / a.c);
    S.pb[tid] = (int)((a.s[2] + a.c / 2) / a.c);
  }
  __syncthreads();
  for (int it = 0; it < GIF_LLOYD; ++it) {
    if (tid < 256) { S.lc[tid] = 0; S.ls[tid][0] = 0; S.ls[tid][1] = 0; S.ls[tid][2] = 0; }
    __syncthreads();
    for (long long i = tid; i < n; i += GIF_PAL_THREADS) {
      const unsigned long long col = A[i], c = (unsigned)col;
      const int r = chan(col, 0), g = chan(col, 1), b = chan(col, 2);
      const int j = nearest(S.pr, S.pg, S.pb, r, g, b);
      atomicAdd(&S.lc[j], c);
      atomicAdd(&S.ls[j][0], c * r);
      atomicAdd(&S.ls[j][1], c * g);
      atomicAdd(&S.ls[j][2], c * b);
    }
    __syncthreads();
    if (tid < 256 && S.lc[tid]) {   // an entry no colour chose keeps its value
      const unsigned long long c = S.lc[tid];
      S.pr[tid] = (int)((S.ls[tid][0] + c / 2) / c);
      S.pg[tid] = (int)((S.ls[tid][1] + c / 2) / c);
      S.pb[tid] = (int)((S.ls[tid][2] + c / 2) / c);
    }
    __syncthreads();
  }
  if (tid < 256) out[tid] = (unsigned)S.pr[tid] << 16 | (unsigned)S.pg[tid] << 8 | (unsigned)S.pb[tid];
}

// ---- stage 4: the index map -------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(GIF_THREADS) index_kernel(const Frame* __restrict__ frames, int nf, int rule,
                                                            const unsigned* __restrict__ pal, uint8_t* __restrict__ idx) {
  __shared__ int pr[256], pg[256], pb[256];
  const int fi = find_frame(frames, nf, blockIdx.x, false);
  const Frame f = frames[fi];
  {
    const unsigned k = pal[256LL * fi + threadIdx.x];
    pr[threadIdx.x] = (int)(k >> 16);
    pg[threadIdx.x] = (int)(k >> 8) & 255;
    pb[threadIdx.x] = (int)k & 255;
  }
  __syncthreads();
  const long long base = (blockIdx.x - f.chunk0) * (long long)GIF_CHUNK;
  for (int k = 0; k < GIF_PER; ++k) {
    const long long p = base + k * GIF_THREADS + threadIdx.x;
    if (p >= f.N) break;
    const unsigned key = pixel_key(f, rule, p);
    idx[f.coff + p] = (uint8_t)nearest(pr, pg, pb, (int)(key >> 16), (int)(key >> 8) & 255, (int)key & 255);
  }
}

// ---- stage 5: LZW per segment -----------------------------------------------------------------------------------------
// A code is stored with its width: code | (width - 9) << 12.  The width of the j-th code after a CLEAR is the bit length
// of 257 + j (at most 12): the decoder's next free code when it reads that code.
__global__ void __launch_bounds__(32) lzw_kernel(const Frame* __restrict__ frames, const Seg* __restrict__ segs,
                                                 const uint8_t* __restrict__ idx, uint16_t* __restrict__ codes,
                                                 long long* __restrict__ meta) {
  extern __shared__ unsigned tab[];   // GIF_TAB slots: (prefix << 8 | byte) << 12 | code, 0 when free (codes are >= 258)
  const Seg s = segs[blockIdx.x];
  const Frame f = frames[s.frame];
  for (int i = threadIdx.x; i < GIF_TAB; i += 32) tab[i] = 0u;
  __syncwarp();
  if (threadIdx.x) return;
  const uint8_t* in = idx + f.coff + s.start;
  uint16_t* out = codes + s.coff;
  long long nc = 0, bits = 0;
  int j = 0, next = 258;
  auto emit = [&](unsigned code) {
    const int w = min(12, 32 - __clz(257 + j));
    out[nc++] = (uint16_t)(code | (unsigned)(w - 9) << 12);
    bits += w;
    ++j;
  };
  if (s.start == 0) { emit(256u); j = 0; }
  unsigned P = in[0];
  for (long long i = 1; i < s.len; ++i) {
    const unsigned k = in[i], key = P << 8 | k;
    unsigned h = (hash_key(key) >> 19) & (GIF_TAB - 1), e;
    while ((e = tab[h]) != 0u && (e >> 12) != key) h = (h + 1) & (GIF_TAB - 1);
    if (e) { P = e & 4095u; continue; }
    emit(P);
    tab[h] = key << 12 | (unsigned)next;
    if (++next == 4096) {
      emit(256u);
      j = 0;
      next = 258;
      for (int q = 0; q < GIF_TAB; ++q) tab[q] = 0u;
    }
    P = k;
  }
  emit(P);
  emit(s.start + s.len == f.N ? 257u : 256u);
  meta[2 * blockIdx.x] = nc;
  meta[2 * blockIdx.x + 1] = bits;
}

// ---- stages 6-8: offsets, bit packing and the container ---------------------------------------------------------------
__host__ __device__ inline long long data_bytes(long long B) { return B + (B + 254) / 255 + 1; }   // sub-blocks, terminator

__device__ __forceinline__ long long piece_bytes(const Frame& f, long long B) {
  return GIF_FRAME_HDR + data_bytes(B) + (f.t == 0 ? GIF_HDR : 0) + (f.t == f.T - 1 ? 1 : 0);
}

__global__ void __launch_bounds__(1024) plan_kernel(const Frame* __restrict__ frames, int nf, const long long* __restrict__ meta,
                                                    long long* __restrict__ sbit, long long* __restrict__ fbytes,
                                                    long long* __restrict__ poff, long long* __restrict__ files) {
  __shared__ long long warp_tot[32];
  __shared__ long long carry;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  for (int i = tid; i < nf; i += 1024) {
    const Frame f = frames[i];
    long long off = 0;
    for (long long s = f.seg0; s < f.seg0 + f.n_seg; ++s) { sbit[s] = off; off += meta[2 * s + 1]; }
    fbytes[i] = (off + 7) >> 3;
  }
  if (tid == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < nf; base += 1024) {
    const int i = base + tid;
    const long long v = i < nf ? piece_bytes(frames[i], fbytes[i]) : 0;
    long long x = v;
    for (int o = 1; o < 32; o <<= 1) {
      const long long y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) warp_tot[wid] = x;
    __syncthreads();
    if (wid == 0) {
      long long t = warp_tot[lane];
      for (int o = 1; o < 32; o <<= 1) {
        const long long y = __shfl_up_sync(0xffffffffu, t, o);
        if (lane >= o) t += y;
      }
      warp_tot[lane] = t;
    }
    __syncthreads();
    const long long incl = carry + x + (wid ? warp_tot[wid - 1] : 0);
    if (i < nf) poff[i] = incl - v;
    __syncthreads();
    if (tid == 1023) carry = incl;
    __syncthreads();
  }
  for (int i = tid; i < nf; i += 1024) {
    const Frame f = frames[i];
    if (f.t != f.T - 1) continue;
    const long long first = i - f.t;
    files[2 * f.anim] = poff[first];
    files[2 * f.anim + 1] = poff[i] + piece_bytes(f, fbytes[i]) - poff[first];
  }
}

__global__ void __launch_bounds__(32) pack_kernel(const Frame* __restrict__ frames, const Seg* __restrict__ segs,
                                                  const uint16_t* __restrict__ codes, const long long* __restrict__ meta,
                                                  const long long* __restrict__ sbit, uint8_t* __restrict__ streams) {
  const Seg s = segs[blockIdx.x];
  const Frame f = frames[s.frame];
  unsigned* w = reinterpret_cast<unsigned*>(streams + f.soff);
  const long long nc = meta[2 * blockIdx.x];
  const int lane = threadIdx.x;
  unsigned long long pos = sbit[blockIdx.x];
  for (long long b = 0; b < nc; b += 32) {
    const bool ok = b + lane < nc;
    const unsigned c = ok ? codes[s.coff + b + lane] : 0u, v = c & 4095u;
    const int nb = ok ? (int)(c >> 12) + 9 : 0;
    int x = nb;
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (ok) {
      const unsigned long long p = pos + (unsigned long long)(x - nb);
      const unsigned sh = p & 31;
      atomicOr(w + (p >> 5), v << sh);
      if (sh + nb > 32) atomicOr(w + (p >> 5) + 1, v >> (32 - sh));
    }
    pos += (unsigned long long)__shfl_sync(0xffffffffu, x, 31);
  }
}

__device__ __forceinline__ void le16(uint8_t* o, long long v) { o[0] = (uint8_t)v; o[1] = (uint8_t)(v >> 8); }

__global__ void __launch_bounds__(GIF_THREADS) container_kernel(const Frame* __restrict__ frames, const unsigned* __restrict__ pal,
                                                                const uint8_t* __restrict__ streams,
                                                                const long long* __restrict__ fbytes,
                                                                const long long* __restrict__ poff, uint8_t* __restrict__ out) {
  const int fi = blockIdx.x, tid = threadIdx.x;
  const Frame f = frames[fi];
  uint8_t* o = out + poff[fi];
  if (f.t == 0) {
    if (tid == 0) {
      const uint8_t head[GIF_HDR] = {'G', 'I', 'F', '8', '9', 'a', 0, 0, 0, 0, 0x70, 0, 0,   // no global table, 8-bit colour
                                     0x21, 0xff, 11, 'N', 'E', 'T', 'S', 'C', 'A', 'P', 'E', '2', '.', '0', 3, 1, 0, 0, 0};
      for (int i = 0; i < GIF_HDR; ++i) o[i] = head[i];
      le16(o + 6, f.W);
      le16(o + 8, f.H);
      le16(o + 29, f.loop);
    }
    o += GIF_HDR;
  }
  if (tid == 0) {
    const uint8_t gce[8] = {0x21, 0xf9, 4, 0, 0, 0, 0, 0};   // no disposal method, no transparency
    for (int i = 0; i < 8; ++i) o[i] = gce[i];
    le16(o + 4, f.delay);
    uint8_t* d = o + 8;
    d[0] = 0x2c;
    le16(d + 1, 0);
    le16(d + 3, 0);
    le16(d + 5, f.W);
    le16(d + 7, f.H);
    d[9] = 0x87;   // local colour table of 2^(7 + 1) entries, not interlaced
    o[GIF_FRAME_HDR - 1] = 8;   // LZW minimum code size
  }
  {
    const unsigned k = pal[256LL * fi + tid];
    uint8_t* t = o + 18 + 3 * tid;
    t[0] = (uint8_t)(k >> 16); t[1] = (uint8_t)(k >> 8); t[2] = (uint8_t)k;
  }
  const long long B = fbytes[fi], nblk = (B + 254) / 255;
  const uint8_t* src = streams + f.soff;
  uint8_t* d = o + GIF_FRAME_HDR;
  for (long long i = tid; i < B + nblk; i += GIF_THREADS) {
    const long long b = i >> 8, r = i & 255;
    d[i] = r == 0 ? (uint8_t)min(255LL, B - 255 * b) : src[255 * b + r - 1];
  }
  if (tid == 0) {
    d[B + nblk] = 0;
    if (f.t == f.T - 1) d[B + nblk + 1] = 0x3b;
  }
}

struct Layout {
  long long nf, n_seg, px, chunks, hslots, hchunks, codes, stream;
  size_t off_segs, staged, off_hash, off_cols, off_ncol, off_pal, off_idx, off_codes, off_meta, off_sbit, off_fbytes, off_poff,
      off_stream, total;
};

size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

long long hash_cap(long long N) {
  long long c = GIF_CHUNK;
  while (c < 2 * N && c < (1LL << 25)) c <<= 1;
  return c;
}

// a frame's stream bound: every segment's codes at 12 bits, rounded up to whole 8-byte words
long long stream_bound(long long N) {
  long long codes = 0;
  for (long long s = 0; s < N; s += GIF_SEG) codes += seg_codes(std::min((long long)GIF_SEG, N - s));
  return (12 * codes + 63) / 64 * 8;
}

int check_anims(const int64_t* anims, int n, int rule) {
  P2PVG_REQUIRE(n >= 0, P2PVG_ERR_BAD_ARG, "gif_encode: n = %d", n);
  P2PVG_REQUIRE(rule == 0 || rule == 1, P2PVG_ERR_BAD_ARG, "gif_encode: rule %d (0 save_image, 1 tensorboard)", rule);
  P2PVG_REQUIRE(n == 0 || anims, P2PVG_ERR_BAD_ARG, "gif_encode: null animation table");
  long long px = 0, nf = 0, hslots = 0;
  for (int i = 0; i < n; ++i) {
    const int64_t* r = anims + 7 * i;
    P2PVG_REQUIRE(r[0] != 0, P2PVG_ERR_BAD_ARG, "gif_encode: animation %d: null address", i);
    P2PVG_REQUIRE(r[1] == P2PVG_F32 || r[1] == GIF_U8, P2PVG_ERR_BAD_ARG, "gif_encode: animation %d: dtype %lld", i,
                  (long long)r[1]);
    P2PVG_REQUIRE(r[1] != P2PVG_F32 || (r[0] & 3) == 0, P2PVG_ERR_BAD_ARG, "gif_encode: animation %d: misaligned fp32", i);
    for (int k = 2; k < 5; ++k)
      P2PVG_REQUIRE(r[k] >= 1 && r[k] <= 65535, P2PVG_ERR_BAD_ARG, "gif_encode: animation %d: T, H, W = %lld, %lld, %lld "
                    "(1..65535 each)", i, (long long)r[2], (long long)r[3], (long long)r[4]);
    P2PVG_REQUIRE(r[5] >= 0 && r[5] <= 65535 && r[6] >= 0 && r[6] <= 65535, P2PVG_ERR_BAD_ARG,
                  "gif_encode: animation %d: delay %lld cs, loop %lld (0..65535 each)", i, (long long)r[5], (long long)r[6]);
    px += r[2] * r[3] * r[4];
    nf += r[2];
    hslots += r[2] * hash_cap(r[3] * r[4]);
  }
  P2PVG_REQUIRE(px < (1LL << 40) && nf < (1LL << 24) && hslots / GIF_CHUNK < (1LL << 31), P2PVG_ERR_UNSUPPORTED,
                "gif_encode: %lld frames of %lld pixels in all are too many for one call", nf, px);
  return P2PVG_OK;
}

Layout layout(const int64_t* anims, int n) {
  Layout L{};
  for (int i = 0; i < n; ++i) {
    const int64_t* r = anims + 7 * i;
    const long long N = r[3] * r[4];
    L.nf += r[2];
    L.px += r[2] * N;
    L.chunks += r[2] * ((N + GIF_CHUNK - 1) / GIF_CHUNK);
    L.hslots += r[2] * hash_cap(N);
    L.n_seg += r[2] * ((N + GIF_SEG - 1) / GIF_SEG);
    long long codes = 0;
    for (long long s = 0; s < N; s += GIF_SEG) codes += seg_codes(std::min((long long)GIF_SEG, N - s));
    L.codes += r[2] * codes;
    L.stream += r[2] * stream_bound(N);
  }
  L.hchunks = L.hslots / GIF_CHUNK;
  L.off_segs = align256(sizeof(Frame) * L.nf);
  L.staged = L.off_segs + sizeof(Seg) * L.n_seg;
  L.off_hash = align256(L.staged);
  L.off_cols = L.off_hash + align256(8 * L.hslots);
  L.off_ncol = L.off_cols + align256(8 * L.px);
  L.off_pal = L.off_ncol + align256(2 * 4 * L.nf);   // distinct colours, then list fill counters
  L.off_idx = L.off_pal + align256(4 * 256 * L.nf);
  L.off_codes = L.off_idx + align256(L.px);
  L.off_meta = L.off_codes + align256(2 * L.codes);
  L.off_sbit = L.off_meta + align256(16 * L.n_seg);
  L.off_fbytes = L.off_sbit + align256(8 * L.n_seg);
  L.off_poff = L.off_fbytes + align256(8 * L.nf);
  L.off_stream = L.off_poff + align256(8 * L.nf);
  L.total = L.off_stream + (size_t)L.stream;
  return L;
}

size_t out_bound(const int64_t* anims, int n) {
  size_t b = 0;
  for (int i = 0; i < n; ++i) {
    const int64_t* r = anims + 7 * i;
    b += GIF_HDR + 1 + (size_t)r[2] * (GIF_FRAME_HDR + data_bytes(stream_bound(r[3] * r[4])));
  }
  return b;
}

}  // namespace

extern "C" size_t p2pvg_gif_workspace_bytes(const int64_t* anims, int n) {
  if (check_anims(anims, n, 1) != P2PVG_OK) return 0;
  return layout(anims, n).total;
}

extern "C" size_t p2pvg_gif_out_bytes(const int64_t* anims, int n) {
  if (check_anims(anims, n, 1) != P2PVG_OK) return 0;
  return out_bound(anims, n);
}

extern "C" int p2pvg_gif_encode(const int64_t* anims, int n, int rule, void* ws, size_t ws_bytes, uint8_t* out, size_t out_bytes,
                                int64_t* files, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const int rc = check_anims(anims, n, rule);
  if (rc != P2PVG_OK) return rc;
  if (n == 0) return P2PVG_OK;
  P2PVG_REQUIRE(ws && out && files, P2PVG_ERR_BAD_ARG, "gif_encode: null workspace, output or file table");
  P2PVG_REQUIRE(((uintptr_t)ws & 255) == 0 && ((uintptr_t)files & 7) == 0, P2PVG_ERR_BAD_ARG,
                "gif_encode: workspace must be 256-byte, files 8-byte aligned");
  const Layout L = layout(anims, n);
  P2PVG_REQUIRE(ws_bytes >= L.total, P2PVG_ERR_WORKSPACE, "gif_encode: workspace %zu bytes, needs %zu", ws_bytes, L.total);
  const size_t bound = out_bound(anims, n);
  P2PVG_REQUIRE(out_bytes >= bound, P2PVG_ERR_WORKSPACE, "gif_encode: output %zu bytes, needs %zu", out_bytes, bound);

  std::vector<unsigned char> host(L.staged, 0);
  Frame* fr = reinterpret_cast<Frame*>(host.data());
  Seg* sg = reinterpret_cast<Seg*>(host.data() + L.off_segs);
  long long f = 0, s = 0, px = 0, chunk = 0, hoff = 0, code = 0, soff = 0;
  for (int i = 0; i < n; ++i) {
    const int64_t* r = anims + 7 * i;
    const long long T = r[2], H = r[3], W = r[4], N = H * W, hc = hash_cap(N);
    const long long frame_bytes = r[1] == GIF_U8 ? 3 * N : 12 * N, ns = (N + GIF_SEG - 1) / GIF_SEG;
    for (long long t = 0; t < T; ++t, ++f) {
      fr[f] = Frame{r[0] + t * frame_bytes, r[1], i, t, T, H, W, N, hoff, hc, px, chunk, hoff / GIF_CHUNK, s, ns, soff, r[5], r[6]};
      for (long long k = 0; k < N; k += GIF_SEG, ++s) {
        const long long len = std::min((long long)GIF_SEG, N - k);
        sg[s] = Seg{f, k, len, code};
        code += seg_codes(len);
      }
      px += N;
      chunk += (N + GIF_CHUNK - 1) / GIF_CHUNK;
      hoff += hc;
      soff += stream_bound(N);
    }
  }
  unsigned char* w = static_cast<unsigned char*>(ws);
  cudaError_t err = cudaMemcpyAsync(w, host.data(), L.staged, cudaMemcpyHostToDevice, st);
  if (err == cudaSuccess) err = cudaMemsetAsync(w + L.off_hash, 0xff, 8 * L.hslots, st);
  if (err == cudaSuccess) err = cudaMemsetAsync(w + L.off_ncol, 0, 8 * L.nf, st);
  if (err == cudaSuccess) err = cudaMemsetAsync(w + L.off_stream, 0, L.stream, st);
  if (err != cudaSuccess) {
    p2pvg_set_error("gif_encode: table upload: %s", cudaGetErrorString(err));
    return P2PVG_ERR_CUDA;
  }
  const Frame* d_fr = reinterpret_cast<const Frame*>(w);
  const Seg* d_sg = reinterpret_cast<const Seg*>(w + L.off_segs);
  auto* hash = reinterpret_cast<unsigned long long*>(w + L.off_hash);
  auto* cols = reinterpret_cast<unsigned long long*>(w + L.off_cols);
  auto* ncol = reinterpret_cast<unsigned*>(w + L.off_ncol);
  auto* pal = reinterpret_cast<unsigned*>(w + L.off_pal);
  uint8_t* idx = w + L.off_idx;
  auto* codes = reinterpret_cast<uint16_t*>(w + L.off_codes);
  auto* meta = reinterpret_cast<long long*>(w + L.off_meta);
  auto* sbit = reinterpret_cast<long long*>(w + L.off_sbit);
  auto* fbytes = reinterpret_cast<long long*>(w + L.off_fbytes);
  auto* poff = reinterpret_cast<long long*>(w + L.off_poff);
  uint8_t* streams = w + L.off_stream;
  const int nf = (int)L.nf;

  int dev = 0;
  cudaGetDevice(&dev);
  static unsigned long long attr_set = 0;   // per device
  if (dev >= 64 || !((attr_set >> dev) & 1ULL)) {
    err = cudaFuncSetAttribute(palette_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(PaletteSmem));
    if (err != cudaSuccess) {
      p2pvg_set_error("gif_encode: shared-memory attribute: %s", cudaGetErrorString(err));
      return P2PVG_ERR_CUDA;
    }
    if (dev < 64) attr_set |= 1ULL << dev;
  }
  colours_kernel<<<(unsigned)L.chunks, GIF_THREADS, 0, st>>>(d_fr, nf, rule, hash, ncol);
  compact_kernel<<<(unsigned)L.hchunks, GIF_THREADS, 0, st>>>(d_fr, nf, hash, ncol + nf, cols);
  palette_kernel<<<(unsigned)nf, GIF_PAL_THREADS, sizeof(PaletteSmem), st>>>(d_fr, ncol, cols, hash, pal);
  index_kernel<<<(unsigned)L.chunks, GIF_THREADS, 0, st>>>(d_fr, nf, rule, pal, idx);
  lzw_kernel<<<(unsigned)L.n_seg, 32, GIF_TAB * sizeof(unsigned), st>>>(d_fr, d_sg, idx, codes, meta);
  plan_kernel<<<1, 1024, 0, st>>>(d_fr, nf, meta, sbit, fbytes, poff, reinterpret_cast<long long*>(files));
  pack_kernel<<<(unsigned)L.n_seg, 32, 0, st>>>(d_fr, d_sg, codes, meta, sbit, streams);
  container_kernel<<<(unsigned)nf, GIF_THREADS, 0, st>>>(d_fr, pal, streams, fbytes, poff, out);
  return p2pvg_check_launch("gif_encode");
}
