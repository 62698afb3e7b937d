// Implicit-GEMM 4x4 / stride-2 / pad-1 convolution family on NHWC bf16 tensors (no im2col / col2im buffers).
// The persistent wgmma skeleton of tc_common.cuh, shared with gemm_tc.cu (TMA -> 128B-swizzled smem -> wgmma.mma_async in
// one MMA warpgroup -> shared-memory staging buffer -> epilogue warps); what changes is how an operand tile is fetched:
//
//   "pixel box" tiles: P consecutive NHW pixels of the SMALL map (H x W per image) are a rectangular box
//   {bw = W, bh, bn}; the operand rows for filter tap (kh,kw) are the BIG-map pixels (2y+kh-1, 2x+kw-1), i.e. one
//   4-D TMA load with elementStrides {1,2,2,1} whose out-of-bounds part (the conv padding) is zero-filled by the
//   hardware.  For the transposed direction the rows are SMALL-map pixels (y+dy, x+dx): a stride-1 4-D box.
//
// kind 0  y_small[N,H,W,Cn] = conv_s2(x_big[N,2H,2W,Ck]) . W[Cn, (tap, Ck)]           Conv forward, ConvT data-gradient
// kind 1  g[Cm, (tap, Cn)]  = sum_pix a_small[pix, Cm]^T . gather_s2(b_big)[pix, tap, Cn]   weight gradients (split-K)
// kind 2  y_big[N,2H,2W,Cn] = convT_s2(x_small[N,H,W,Ck]) . W[Ck, (tap, Cn)] + bias + addend   ConvT forward, Conv data-gradient
//         (4 output-parity phases, each a 2x2 stride-1 convolution; `addend` holds the skip-connection half of
//          torch.cat([d, skip]) computed once per distinct source call and is indexed through grp_src)
// kind 3  y[N,H,W,Cn] = conv3x3_s1_p1(x[N,H,W,Ck]) . W[Cn, (tap, Ck)] + bias + addend      vgg layer forward (kind 0 geometry, 9 taps)
// kind 4  g[Cm, (tap, Cn)] = sum_pix a[pix, Cm]^T . gather_3x3(b)[pix, tap, Cn]             vgg weight gradients (kind 1 geometry)
// kind 5  kind 3 with mirrored tap offsets (pixel - (kh-1, kw-1)): the data gradient of a 3x3 convolution

#include "tc_common.cuh"

namespace {

using namespace tc;

struct Geom {
  int N, H, W;          // images, small-map height / width
  int Ck, Cn;           // reduction channels / output channels (kind 0,2);  kind 1: Cm = M extent, Cn = gathered channels
  int M;                // GEMM M: kind 0/2: N*H*W pixels; kind 1: Cm
  int Ntot;             // GEMM N: kind 0/2: Cn; kind 1: 16*Cn
  int bhm, bnm;         // pixel box of one M tile (BM = 128 or 256 pixels, kinds 0 / 2): {W, bhm, bnm}
  int bh64, bn64;       // pixel box of 64 pixels (kind 1 K-blocks): {bw64, bh64, bn64}; bw64 = 64 < W for 128-wide maps
  int bw64;
  int imgs_per_group;   // addend indexing
  int add_bf16;         // the addend tensor is bf16 (half the epilogue read traffic of the fp32 form)
  int bres;             // kind 0, BN = 64, one channel chunk, <= 9 taps: ALL weight tiles stay resident in shared memory for the whole
                        // kernel (72 KB) and only the A boxes stream through a 7-slot ring -- the 64 -> 64 channel 3x3 layers re-fetched
                        // their 73 KB of weights for every 128-pixel tile (43 FLOP per filled byte -> 65)
  int swap;             // kind 1 with the operand roles swapped: M = taps*Cn (gathered map), N = Cm (few output channels would waste
                        // half of a 128-row MMA tile otherwise); the partial sums are [taps*Cn][Cm] and the reduce kernel transposes
  int ks, st, sgn;      // filter taps per side (4 | 3), stride between the two maps (2 | 1), tap-offset sign (+1 | -1)
};

__device__ __forceinline__ void pix_block(int pb, int P, int H, int W, int bh, int bn, int& n0, int& y0) {
  const int HW = H * W;
  if (HW >= P) {
    const int bpi = HW / P;
    n0 = pb / bpi;
    y0 = (pb - n0 * bpi) * bh;
  } else {
    n0 = pb * bn;
    y0 = 0;
  }
}

// 64 addend columns of one output row into 16-byte registers: 16 loads for fp32, 8 for bf16
__device__ __forceinline__ void addend_load64(float4 (&a4)[16], const float* base, long long elem_off, bool is_bf16) {
  if (is_bf16) {
    const uint4* p = reinterpret_cast<const uint4*>(reinterpret_cast<const bf16*>(base) + elem_off);
#pragma unroll
    for (int j = 0; j < 8; j++) {
      const uint4 r = p[j];
      a4[j] = make_float4(__uint_as_float(r.x), __uint_as_float(r.y), __uint_as_float(r.z), __uint_as_float(r.w));
    }
  } else {
    const float4* p = reinterpret_cast<const float4*>(base + elem_off);
#pragma unroll
    for (int j = 0; j < 16; j++) a4[j] = p[j];
  }
}
// f[0..31] += columns [32 h, 32 h + 32) of what addend_load64 fetched
__device__ __forceinline__ void addend_add32(float (&f)[32], const float4 (&a4)[16], int h, bool is_bf16) {
  if (is_bf16) {
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const float4 r = a4[4 * h + j];
      float v[8];
      unpack16<bf16>(make_uint4(__float_as_uint(r.x), __float_as_uint(r.y), __float_as_uint(r.z), __float_as_uint(r.w)), v);
#pragma unroll
      for (int i = 0; i < 8; i++) f[8 * j + i] += v[i];
    }
  } else {
#pragma unroll
    for (int j = 0; j < 8; j++) {
      const float4 x4 = a4[8 * h + j];
      f[4 * j] += x4.x; f[4 * j + 1] += x4.y; f[4 * j + 2] += x4.z; f[4 * j + 3] += x4.w;
    }
  }
}

// EVAL: eval-mode BatchNorm + activation in the epilogue, y = act(eval_scale[c] * (acc + bias + addend) + eval_shift[c]) (kinds 0 / 2;
// kind 3 runs as kind 0)
// BM = 256 (kind 2, BN = 64, no statistics or eval epilogue): 256-pixel tiles, twice the MMA work per filled K block
template <int KIND, int BM, int BN, bool STAT, bool EVAL>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, void* __restrict__ Cv, int c_bf16,
                 long long ldc, Geom g, int accumulate, const float* __restrict__ bias, const float* __restrict__ addend,
                 const int* __restrict__ grp_src, float* __restrict__ partial, int kb_per_split, int splits,
                 float2* __restrict__ stat_partial, const float* __restrict__ eval_scale, const float* __restrict__ eval_shift, int act) {
  static_assert(BM == 128 || (KIND == 2 && !STAT && !EVAL), "256-row tiles: kind 2 without statistics or eval epilogue");
  using C_ = Cfg<BN, BM>;
  constexpr bool A_MN = (KIND == 1), B_MN = (KIND != 0);
  extern __shared__ uint8_t smem_raw[];
  const Smem sm = smem_setup<BN, BM>(smem_raw);
  const bool bres = (KIND == 0) && (BN == 64) && g.bres != 0;   // resident weights (tc_common.cuh BRES_*)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_m = (g.M + BM - 1) / BM, tiles_n = (g.Ntot + BN - 1) / BN;
  const int tiles_mn = tiles_m * tiles_n;
  const int phases = (KIND == 2) ? 4 : 1;
  const int num_tiles = tiles_mn * splits * phases;
  const int cchunks = g.Ck / 64;
  // K blocks: kind 0: 16 taps x Ck/64; kind 2: 4 taps x Ck/64; kind 1: pixel blocks of 64
  const int nkb_total = (KIND == 0) ? g.ks * g.ks * cchunks : (KIND == 2) ? 4 * cchunks : (g.N * g.H * g.W + 63) / 64;

  if (warp >= 8) {
    // ===================== TMA producer =====================
    regs_producer();
    if (warp == 8 && lane == 0) {
      uint32_t it = 0;
      if (bres) {   // all weight taps once: [tap][64 output channels][64 input channels]
        mbar_expect_tx(sm.bres_bar, (uint32_t)(g.ks * g.ks) * 64 * 128);
        for (int tap = 0; tap < g.ks * g.ks; tap++) tma_load_2d(&tmB, sm.bres_bar, sm.ring + tap * 64 * 128, tap * 64, 0);
      }
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        // tile decode with as few integer divisions as possible: the producer thread is the latency-critical one
        // kind 2: the output-parity phase is the FASTEST tile index, so that the four phases of one pixel tile run on four
        // CTAs at the same time and share the A tile through L2 (in phase-major order every phase would re-read A from
        // DRAM).  Kinds 0 / 2 never split K.
        const int ph = (KIND == 2) ? (t & 3) : 0;
        const int t2 = (KIND == 2) ? (t >> 2) : t;
        const int z = (splits == 1) ? 0 : t2 / tiles_mn, r = t2 - z * tiles_mn;
        const int mt = (tiles_n == 1) ? r : r / tiles_n, nt = (tiles_n == 1) ? 0 : r - mt * tiles_n;
        const int n0 = nt * BN;
        const int kb0 = z * kb_per_split, kb1 = min(kb0 + kb_per_split, nkb_total);
        int pn0 = 0, py0 = 0;
        if (KIND != 1) pix_block(mt, BM, g.H, g.W, g.bhm, g.bnm, pn0, py0);
        const int pa = ph >> 1, pb_ = ph & 1;
        // kind 1: everything that does not depend on the K-block is computed once per tile, the pixel-box coordinates
        // advance incrementally -- the single producer thread must not spend its K-block budget on integer divisions
        int kn0 = 0, ky0 = 0, kx0 = 0;
        int t_kh = 0, t_kw = 0, t_cc = 0;
        int qc0[BN / 64], qdx[BN / 64], qdy[BN / 64];
        int mc0[2] = {0, 0}, mdx[2] = {0, 0}, mdy[2] = {0, 0};
        if (KIND == 1) {
          if (g.bw64 < g.W) {  // a 64-pixel K-block is a fraction of one row
            const int per_row = g.W / g.bw64;
            const int rowi = kb0 / per_row;
            kx0 = (kb0 - rowi * per_row) * g.bw64;
            kn0 = rowi / g.H;
            ky0 = rowi - kn0 * g.H;
          } else {
            pix_block(kb0, 64, g.H, g.W, g.bh64, g.bn64, kn0, ky0);
          }
#pragma unroll
          for (int q = 0; q < BN / 64; q++) {
            const int nb = n0 + 64 * q;
            const int tap = nb / g.Cn;
            const int kh = tap / g.ks;
            qc0[q] = nb - tap * g.Cn;
            qdx[q] = tap - kh * g.ks - 1;
            qdy[q] = kh - 1;
          }
          if (g.swap) {   // the gathered map is the A operand: (tap, channel) of the two 64-row halves of the M tile
#pragma unroll
            for (int q = 0; q < 2; q++) {
              const int mb = mt * BM + 64 * q;
              int tap = mb / g.Cn;
              if (tap >= g.ks * g.ks) tap = g.ks * g.ks - 1;   // rows past M are discarded by the epilogue: any in-bounds tap will do
              const int kh = tap / g.ks;
              mc0[q] = mb < g.M ? mb - tap * g.Cn : 0;
              mdx[q] = tap - kh * g.ks - 1;
              mdy[q] = kh - 1;
            }
          }
        }
        for (int kb = kb0; kb < kb1; kb++, it++) {
          // (both divisors are compile-time constants: no runtime division in the single producer / issuer threads)
          const int s = bres ? (int)(it % BRES_STAGES) : (int)(it % C_::STAGES);
          const uint32_t par = (bres ? (it / BRES_STAGES) : (it / C_::STAGES)) & 1;
          mbar_wait(&sm.empty_bar[s], par ^ 1);
          uint8_t* sa = bres ? sm.ring + BRES_B_BYTES + s * A_STAGE_BYTES : sm.ring + s * C_::STAGE_BYTES;
          uint8_t* sb = sa + C_::A_STAGE_BYTES;
          mbar_expect_tx(&sm.full_bar[s], bres ? A_STAGE_BYTES : C_::STAGE_BYTES);
          if (KIND == 0) {
            // (kh, kw, channel chunk) advance incrementally (kinds 0 / 2 never split K: kb starts at 0)
            tma_load_4d(&tmA, &sm.full_bar[s], sa, t_cc * 64, g.sgn * (t_kw - 1), g.st * py0 + g.sgn * (t_kh - 1), pn0);
            if (!bres) tma_load_2d(&tmB, &sm.full_bar[s], sb, kb * 64, n0);   // (tap * Ck + c0) == kb * 64
            if (++t_cc == cchunks) { t_cc = 0; if (++t_kw == g.ks) { t_kw = 0; t_kh++; } }
          } else if (KIND == 2) {
            const int tq = t_kh, c0 = t_cc * 64;   // t_kh doubles as the 2x2 tap index of this phase
            if (++t_cc == cchunks) { t_cc = 0; t_kh++; }
            const int i = tq >> 1, j = tq & 1;
            // phase a: taps (dy=0, ky=a+1) and (dy = a ? +1 : -1, ky = a ? 0 : 3); same along x
            const int dy = i == 0 ? 0 : (pa ? 1 : -1), ky = i == 0 ? pa + 1 : (pa ? 0 : 3);
            const int dx = j == 0 ? 0 : (pb_ ? 1 : -1), kx = j == 0 ? pb_ + 1 : (pb_ ? 0 : 3);
            tma_load_4d(&tmA, &sm.full_bar[s], sa, c0, dx, py0 + dy, pn0);
#pragma unroll
            for (int q = 0; q < BN / 64; q++)
              tma_load_2d(&tmB, &sm.full_bar[s], sb + q * 64 * 128, (ky * 4 + kx) * g.Cn + n0 + 64 * q, c0);
          } else {
            const int m0 = mt * BM;
            if (g.swap) {
              tma_load_4d(&tmA, &sm.full_bar[s], sa, mc0[0], g.st * kx0 + mdx[0], g.st * ky0 + mdy[0], kn0);
              tma_load_4d(&tmA, &sm.full_bar[s], sa + 64 * 128, mc0[1], g.st * kx0 + mdx[1], g.st * ky0 + mdy[1], kn0);
#pragma unroll
              for (int q = 0; q < BN / 64; q++) tma_load_2d(&tmB, &sm.full_bar[s], sb + q * 64 * 128, n0 + 64 * q, kb * 64);
            } else {
              tma_load_2d(&tmA, &sm.full_bar[s], sa, m0, kb * 64);
              tma_load_2d(&tmA, &sm.full_bar[s], sa + 64 * 128, m0 + 64, kb * 64);
#pragma unroll
              for (int q = 0; q < BN / 64; q++)
                tma_load_4d(&tmB, &sm.full_bar[s], sb + q * 64 * 128, qc0[q], g.st * kx0 + qdx[q], g.st * ky0 + qdy[q], kn0);
            }
            // next 64-pixel box
            if (g.bw64 < g.W) {
              kx0 += g.bw64;
              if (kx0 >= g.W) { kx0 = 0; if (++ky0 >= g.H) { ky0 = 0; kn0++; } }
            } else if (g.H * g.W >= 64) {
              ky0 += g.bh64;
              if (ky0 >= g.H) { ky0 = 0; kn0++; }
            } else {
              kn0 += g.bn64;
            }
          }
        }
      }
    }
  } else if (warp >= 4) {
    regs_worker();
    mma_loop<false, BN, A_MN, B_MN, BM>(sm, num_tiles, tiles_mn, splits, kb_per_split, nkb_total, bres);
  } else {
    // ===================== epilogue =====================
    regs_worker();
    const int q = warp;
    __shared__ float bias_s[2 * BN];
    // BatchNorm forward statistics fused into the epilogue: per-warp column sums (sum y, sum y^2) of the tile, double-
    // buffered by tile parity so that tile t+1 may write while the sums of tile t are still being combined
    __shared__ float2 stat_s[STAT ? 2 * 4 * BN : 1];
    constexpr bool do_stat = STAT;   // a separate instantiation: the statistics cost ~50 registers in this epilogue
    // eval-mode BatchNorm coefficients of the tile's columns, double-buffered by tile parity like bias_s: [parity][scale | shift][BN]
    __shared__ float ev_s[EVAL ? 2 * 2 * BN : 1];
    // plain bf16 stores of kinds 0 / 2 (no statistics, no eval epilogue, no accumulation; a bf16 addend if any) take the
    // row-cooperative path
    const bool row_major_store = !STAT && !EVAL && KIND != 1 && c_bf16 && !accumulate && (addend == nullptr || g.add_bf16);
    uint32_t lt = 0, lh = 0;   // tiles / staging-buffer hand-overs (BM / 128 per tile) so far
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x, lt++) {
      const int ph = (KIND == 2) ? (t & 3) : 0;
      const int t2 = (KIND == 2) ? (t >> 2) : t;
      const int z = (splits == 1) ? 0 : t2 / tiles_mn, r = t2 - z * tiles_mn;
      const int mt = (tiles_n == 1) ? r : r / tiles_n, nt = (tiles_n == 1) ? 0 : r - mt * tiles_n;
      const int n0 = nt * BN;
      const uint32_t acc = lt & 1;   // bias_s / stat_s half of this tile
      int pn0 = 0, py0 = 0;
      if (KIND == 2) pix_block(mt, BM, g.H, g.W, g.bhm, g.bnm, pn0, py0);
      // tile row rt -> output row, addend row (through grp_src), whether the row exists
      auto row_of = [&](int rt, long long& out_row, long long& add_row, bool& row_ok) {
        out_row = (long long)mt * BM + rt;
        add_row = 0;
        row_ok = out_row < g.M;
        if (KIND == 2) {
          // tile row -> small-map pixel -> big-map output pixel of this parity phase
          const int HW = g.H * g.W;
          int nn, yy, xx;
          if (HW >= BM) { nn = 0; yy = rt / g.W; xx = rt - yy * g.W; }
          else { nn = rt / HW; const int rem = rt - nn * HW; yy = rem / g.W; xx = rem - yy * g.W; }
          const int n = pn0 + nn, y = py0 + yy;
          row_ok = (n < g.N) && (y < g.H);
          const int oy = 2 * y + (ph >> 1), ox = 2 * xx + (ph & 1);
          out_row = ((long long)n * (2 * g.H) + oy) * (2 * g.W) + ox;
          if (addend && row_ok) {
            const int n2 = grp_src[n / g.imgs_per_group] * g.imgs_per_group + (n % g.imgs_per_group);
            add_row = ((long long)n2 * (2 * g.H) + oy) * (2 * g.W) + ox;
          }
        }
        if (KIND == 0 && addend && row_ok) {
          const int HW = g.H * g.W;
          const int n = (int)(out_row / HW);
          const int n2 = grp_src[n / g.imgs_per_group] * g.imgs_per_group + (n % g.imgs_per_group);
          add_row = (long long)n2 * HW + (out_row - (long long)n * HW);
        }
      };
      if (EVAL) {
        stage_cols<BN>(ev_s + acc * 2 * BN, eval_scale, n0, g.Ntot);
        stage_cols<BN>(ev_s + acc * 2 * BN + BN, eval_shift, n0, g.Ntot);
        if (bias == nullptr) epi_bar_sync();
      }
      if (bias != nullptr) {
        stage_cols<BN>(bias_s + acc * BN, bias, n0, g.Ntot);
        epi_bar_sync();
      }
      const bool abf = g.add_bf16 != 0;
      if (row_major_store) {
        // Row-cooperative bf16 stores: LPR lanes share one output row, 16 B (8 columns) each, so one warp instruction writes
        // RPI whole rows instead of 32 scattered 16-byte pieces of 32 rows.  The row addresses come from the lane that owns
        // the row.  The addend of every row the lane writes in this tile (BN = 64: 8 per 128 rows; BN = 128: 16) is
        // requested before the accumulator is waited for.  Same arithmetic per element as the thread-per-row path:
        // (acc + bias) + addend, rounded once to bf16.
        constexpr int LPR = BN / 8, RPI = 32 / LPR, STEPS = 32 / RPI, HALVES = BM / 128;
        const int sub = lane / LPR, cl = (lane % LPR) * 8;
        const bool col_ok = n0 + cl < g.Ntot;   // Ntot is a multiple of 32: 8-column groups are all in or all out
        bf16* cbase = reinterpret_cast<bf16*>(Cv) + n0 + cl;
        long long orow_h[HALVES];
        bool ok_h[HALVES];
        uint4 av[HALVES * STEPS];   // 8 bf16 addend values per step
#pragma unroll
        for (int hf = 0; hf < HALVES; hf++) {
          long long arow_h;
          row_of(hf * 128 + q * 32 + lane, orow_h[hf], arow_h, ok_h[hf]);
          if (addend != nullptr) {
            const bf16* abase = reinterpret_cast<const bf16*>(addend) + n0 + cl;
#pragma unroll
            for (int i = 0; i < STEPS; i++) {
              const int src = i * RPI + sub;
              const long long arow = __shfl_sync(0xffffffffu, arow_h, src);
              const bool aok = __shfl_sync(0xffffffffu, (int)ok_h[hf], src) != 0;
              av[hf * STEPS + i] = (aok && col_ok) ? *reinterpret_cast<const uint4*>(abase + arow * g.Ntot) : make_uint4(0, 0, 0, 0);
            }
          }
        }
        // the staging reads of CH steps are taken before their stores, which wait for the addend: the warp releases the
        // staging buffer (the MMA warpgroup's second half of a 256-row tile waits for it) without waiting for the addend
        constexpr int CH = STEPS < 8 ? STEPS : 8;
#pragma unroll
        for (int hf = 0; hf < HALVES; hf++, lh++) {
          mbar_wait(sm.acc_full_bar, lh & 1);
#pragma unroll
          for (int c0 = 0; c0 < STEPS; c0 += CH) {
            float4 x[CH][2];
#pragma unroll
            for (int k = 0; k < CH; k++) {
              const float* s = sm.accs + (q * 32 + (c0 + k) * RPI + sub) * C_::ACC_LD + cl;
              x[k][0] = *reinterpret_cast<const float4*>(s);
              x[k][1] = *reinterpret_cast<const float4*>(s + 4);
            }
            if (c0 + CH == STEPS) {   // the warp's last staging read of this hand-over
              __syncwarp();
              if (lane == 0) mbar_arrive(sm.acc_empty_bar);
            }
#pragma unroll
            for (int k = 0; k < CH; k++) {
              const int i = c0 + k, src = i * RPI + sub;   // the warp row this lane writes in step i
              const long long orow = __shfl_sync(0xffffffffu, orow_h[hf], src);
              const bool ok = __shfl_sync(0xffffffffu, (int)ok_h[hf], src) != 0;
              if (!ok || !col_ok) continue;
              const float4 x0 = x[k][0], x1 = x[k][1];
              float f[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
              if (bias) {
#pragma unroll
                for (int j = 0; j < 8; j++) f[j] += bias_s[acc * BN + cl + j];
              }
              if (addend != nullptr) {
                float a[8];
                unpack16<bf16>(av[hf * STEPS + i], a);
#pragma unroll
                for (int j = 0; j < 8; j++) f[j] += a[j];
              }
              *reinterpret_cast<uint4*>(cbase + orow * ldc) = pack16<bf16>(f);
            }
          }
        }
        continue;
      }
      // thread-per-row path: one tile row per thread, BM / 128 hand-overs of the staging buffer per tile
#pragma unroll 1
      for (int hf = 0; hf < BM / 128; hf++, lh++) {
        const int rs = q * 32 + lane;  // staging-buffer row
        long long out_row, add_row;
        bool row_ok;
        row_of(hf * 128 + rs, out_row, add_row, row_ok);
        const bool use_add = (KIND != 1) && addend != nullptr && row_ok;
        const long long aoff0 = add_row * g.Ntot + n0;   // element offset of this row's first addend column
        float4 a4[16];  // addend of the next 64 columns, requested before the accumulator is waited for
        if (use_add) addend_load64(a4, addend, aoff0, abf);
        mbar_wait(sm.acc_full_bar, lh & 1);
#pragma unroll 1
        for (int pr = 0; pr < BN / 64; pr++) {
          if (pr > 0 && use_add) addend_load64(a4, addend, aoff0 + pr * 64, abf);
#pragma unroll
          for (int h = 0; h < 2; h++) {
            const int c = pr * 2 + h;
            float f[32];
            read_chunk<BN>(sm, rs, c, f);
            const int nbase = n0 + c * 32;
            if (nbase >= g.Ntot) continue;             // warp-uniform
            if (!row_ok && !do_stat) continue;         // rows past the end only matter as zeros of the column sums
            if (KIND == 1 && partial != nullptr) {
              float* dst = partial + ((long long)z * g.M + out_row) * g.Ntot + nbase;
#pragma unroll
              for (int j = 0; j < 32; j += 8)   // partial workspace rows are 32-byte aligned (Ntot and nbase are multiples of 32)
                st_global_256(dst + j, __float_as_uint(f[j]), __float_as_uint(f[j + 1]), __float_as_uint(f[j + 2]), __float_as_uint(f[j + 3]),
                              __float_as_uint(f[j + 4]), __float_as_uint(f[j + 5]), __float_as_uint(f[j + 6]), __float_as_uint(f[j + 7]));
              continue;
            }
            if (bias) add_staged32(f, bias_s + acc * BN + c * 32);
            if (use_add) addend_add32(f, a4, h, abf);
            if (EVAL) {
              const float* sc = ev_s + acc * 2 * BN + c * 32;
#pragma unroll
              for (int j = 0; j < 32; j++) {
                float y = fmaf(f[j], sc[j], sc[BN + j]);
                if (act == P2PVG_ACT_LRELU) y = y > 0.f ? y : 0.2f * y;
                else if (act == P2PVG_ACT_TANH) y = tanhf(y);
                f[j] = y;
              }
            }
            if (STAT) {
              // statistics of the tensor AS STORED (bf16-rounded when the output is bf16); all 32 lanes take part
              float s1[32], s2[32];
#pragma unroll
              for (int j = 0; j < 32; j++) {
                const float r = row_ok ? (c_bf16 ? bf16_round(f[j]) : f[j]) : 0.f;
                s1[j] = r;
                s2[j] = r * r;
              }
              const float cs = warp_colsum32(s1, lane), cq = warp_colsum32(s2, lane);
              stat_s[(acc * 4 + q) * BN + c * 32 + lane] = make_float2(cs, cq);
              if (!row_ok) continue;
            }
            if (c_bf16) store_row32<bf16, false>(reinterpret_cast<bf16*>(Cv) + out_row * ldc + nbase, f, accumulate, 32);
            else store_row32<float, false>(reinterpret_cast<float*>(Cv) + out_row * ldc + nbase, f, accumulate, 32);
          }
        }
      }
      if (STAT) {
        // combine the four warps' column sums in a fixed order (deterministic) -> one partial row per (pixel tile, phase)
        epi_bar_sync();
        float2* dst = stat_partial + ((long long)mt * phases + ph) * g.Ntot + n0;
        for (int i = q * 32 + lane; i < BN; i += 128) {
          if (n0 + i >= g.Ntot) continue;
          const float2 a = stat_s[(acc * 4 + 0) * BN + i], b = stat_s[(acc * 4 + 1) * BN + i];
          const float2 c2 = stat_s[(acc * 4 + 2) * BN + i], d = stat_s[(acc * 4 + 3) * BN + i];
          dst[i] = make_float2((a.x + b.x) + (c2.x + d.x), (a.y + b.y) + (c2.y + d.y));
        }
      }
    }
  }
}

// NHWC [N, Hm, Wm, C] pixel-box map: box {64 ch, bw*s, bh*s, bn} traversed with stride s in x and y
int map4d(CUtensorMap* m, const void* base, int N, int Hm, int Wm, int C, int bw, int bh, int bn, int s) {
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)Wm, (cuuint64_t)Hm, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)Wm * C * 2, (cuuint64_t)Hm * Wm * C * 2};
  cuuint32_t box[4] = {64, (cuuint32_t)(bw * s), (cuuint32_t)(bh * s), (cuuint32_t)bn};
  cuuint32_t es[4] = {1, (cuuint32_t)s, (cuuint32_t)s, 1};
  CUresult r = driver().encode(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    p2pvg_set_error("conv_gemm: 4-D tensor map failed (%d): N=%d H=%d W=%d C=%d box=(%d,%d,%d) s=%d", (int)r, N, Hm, Wm, C, bw, bh, bn, s);
    return P2PVG_ERR_CUDA;
  }
  return P2PVG_OK;
}

bool box_for(int P, int H, int W, int& bh, int& bn) {
  const int HW = H * W;
  if (HW >= P) {
    if (P % W != 0 || (H % (P / W)) != 0) return false;
    bh = P / W;
    bn = 1;
  } else {
    if (P % HW != 0) return false;
    bh = H;
    bn = P / HW;
  }
  return bh * 2 <= 256 && W * 2 <= 256 && bn <= 256;
}

// eval-mode BatchNorm epilogue operands (all NULL / 0: no such epilogue)
struct EvalEpi {
  const float* scale = nullptr;
  const float* shift = nullptr;
  int act = 0;
};

template <int KIND, int BM, int BN, bool STAT, bool EVAL>
int launch_t(const CUtensorMap& ta, const CUtensorMap& tb, void* C, int c_dtype, long long ldc, const Geom& g, int accumulate,
             const float* bias, const float* addend, const int* grp_src, float* partial, int splits, int kb_per_split, cudaStream_t st,
             float2* stat_partial, const EvalEpi& ev) {
  const long long tiles = (long long)cdiv(g.M, BM) * cdiv(g.Ntot, BN) * splits * (KIND == 2 ? 4 : 1);
  return launch_persistent<conv_gemm_kernel<KIND, BM, BN, STAT, EVAL>, BN, BM>(tiles, st, "conv_gemm", ta, tb, C, (int)(c_dtype == P2PVG_BF16),
                                                                               ldc, g, accumulate, bias, addend, grp_src, partial, kb_per_split,
                                                                               splits, stat_partial, ev.scale, ev.shift, ev.act);
}

// BM = 256 tiles have no statistics or eval-epilogue instances (the caller does not choose them for such launches)
template <int KIND, int BN, int BM = BLOCK_M>
int launch(const CUtensorMap& ta, const CUtensorMap& tb, void* C, int c_dtype, long long ldc, const Geom& g, int accumulate,
           const float* bias, const float* addend, const int* grp_src, float* partial, int splits, int kb_per_split, cudaStream_t st,
           float2* stat_partial = nullptr, const EvalEpi& ev = EvalEpi()) {
  if constexpr (KIND != 1 && BM == 128) {
    if (ev.scale != nullptr) return launch_t<KIND, BM, BN, false, true>(ta, tb, C, c_dtype, ldc, g, accumulate, bias, addend, grp_src, partial, splits, kb_per_split, st, nullptr, ev);
    if (stat_partial != nullptr) return launch_t<KIND, BM, BN, true, false>(ta, tb, C, c_dtype, ldc, g, accumulate, bias, addend, grp_src, partial, splits, kb_per_split, st, stat_partial, ev);
  }
  return launch_t<KIND, BM, BN, false, false>(ta, tb, C, c_dtype, ldc, g, accumulate, bias, addend, grp_src, partial, splits, kb_per_split, st, nullptr, ev);
}

}  // namespace

// a, b: see the kind table at the top.  H, W: SMALL-map size.  Returns P2PVG_ERR_UNSUPPORTED when the shape does not
// fit the pixel-box tiling (the caller then uses the explicit im2col / col2im path).
extern "C" int p2pvg_conv_gemm(int kind, const void* a, const void* b, int64_t ldb, void* c, int c_dtype, int64_t ldc, int N, int H, int W,
                               int Ck, int Cn, int Cm, const float* bias, const void* addend_v, const int* grp_src, int imgs_per_group,
                               int accumulate, void* ws, size_t ws_bytes, const p2pvg_conv_fusion_t* fusion, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  P2PVG_REQUIRE(a && b && c, P2PVG_ERR_BAD_ARG, "conv_gemm: null operand");
  float2* stat_partial = fusion ? reinterpret_cast<float2*>(fusion->fwd_stat_partial) : nullptr;
  P2PVG_REQUIRE(!(stat_partial && accumulate), P2PVG_ERR_BAD_ARG, "conv_gemm: statistics of an accumulating GEMM are not defined");
  const int addend_dtype = fusion ? fusion->addend_dtype : P2PVG_F32;
  P2PVG_REQUIRE(addend_dtype == P2PVG_F32 || addend_dtype == P2PVG_BF16, P2PVG_ERR_BAD_ARG, "conv_gemm: bad addend dtype %d", addend_dtype);
  const float* addend = reinterpret_cast<const float*>(addend_v);
  const float* eval_scale = fusion ? fusion->eval_scale : nullptr;
  const float* eval_shift = fusion ? fusion->eval_shift : nullptr;
  const int act = fusion ? fusion->act : 0;
  EvalEpi ev;
  ev.scale = eval_scale; ev.shift = eval_shift; ev.act = act;
  P2PVG_REQUIRE(driver().encode != nullptr, P2PVG_ERR_UNSUPPORTED, "conv_gemm: cuTensorMapEncodeTiled unavailable");
  P2PVG_REQUIRE(kind >= 0 && kind <= 5, P2PVG_ERR_BAD_ARG, "conv_gemm: bad kind %d", kind);
  if (eval_scale != nullptr) {
    P2PVG_REQUIRE(kind == 0 || kind == 2 || kind == 3, P2PVG_ERR_BAD_ARG, "conv_gemm: the eval-BatchNorm epilogue belongs to kinds 0, 2 and 3");
    P2PVG_REQUIRE(eval_shift != nullptr, P2PVG_ERR_BAD_ARG, "conv_gemm: eval_scale without eval_shift");
    P2PVG_REQUIRE(stat_partial == nullptr, P2PVG_ERR_BAD_ARG, "conv_gemm: the eval-BatchNorm epilogue excludes fwd_stat_partial");
    P2PVG_REQUIRE(!accumulate, P2PVG_ERR_BAD_ARG, "conv_gemm: the eval-BatchNorm epilogue does not accumulate");
    P2PVG_REQUIRE(act == P2PVG_ACT_LRELU || act == P2PVG_ACT_TANH, P2PVG_ERR_BAD_ARG, "conv_gemm: eval epilogue act %d", act);
  }
  if (N <= 0) return P2PVG_OK;
  Geom g;
  g.N = N; g.H = H; g.W = W; g.Ck = Ck; g.Cn = Cn; g.imgs_per_group = imgs_per_group > 0 ? imgs_per_group : 1;
  g.add_bf16 = (addend != nullptr && addend_dtype == P2PVG_BF16) ? 1 : 0;
  g.swap = 0;
  g.bres = 0;
  g.ks = kind >= 3 ? 3 : 4; g.st = kind >= 3 ? 1 : 2; g.sgn = kind == 5 ? -1 : 1;
  const int taps = g.ks * g.ks;
  if (kind == 3 || kind == 5) kind = 0;
  if (kind == 4) kind = 1;
  // kinds 0 / 2 tile the output in 128-pixel boxes, kind 1 reduces over 64-pixel boxes
  g.bhm = g.bnm = g.bh64 = g.bn64 = 1;
  g.bw64 = W;
  bool ok;
  if (kind == 1) {
    if (W > 64 && W % 64 == 0 && W * g.st <= 256) { g.bw64 = 64; ok = true; }
    else ok = box_for(64, H, W, g.bh64, g.bn64);
  } else {
    ok = box_for(128, H, W, g.bhm, g.bnm);
  }
  ok = ok && (((uintptr_t)a | (uintptr_t)b | (uintptr_t)c) & 15) == 0;
  if (kind == 1) ok = ok && (Cn % 64 == 0) && (Cm % 8 == 0);
  else ok = ok && (Ck % 64 == 0) && (Cn % 32 == 0) && (ldb % 8 == 0);
  if (kind == 2 || addend != nullptr) ok = ok && (Cn % 64 == 0);
  if (!ok) {
    p2pvg_set_error("conv_gemm: shape not supported by the pixel-box tiling (kind=%d N=%d H=%d W=%d Ck=%d Cn=%d)", kind, N, H, W, Ck, Cn);
    return P2PVG_ERR_UNSUPPORTED;
  }
  CUtensorMap ta, tb;
  int rc;
  const long long pix = (long long)N * H * W;
  if (kind == 0) {
    g.M = (int)pix; g.Ntot = Cn;
    rc = map4d(&ta, a, N, g.st * H, g.st * W, Ck, W, g.bhm, g.bnm, g.st);
    if (rc) return rc;
    const int BN = Cn > 64 ? 128 : 64;
    rc = map2d(&tb, b, (long long)taps * Ck, Cn, ldb, BN);
    if (rc) return rc;
    const int nkb = taps * (Ck / 64);
    // 64 -> 64 channel 3x3 layers: weights resident in shared memory
    g.bres = (BN == 64 && Cn == 64 && Ck == 64 && taps <= 9) ? 1 : 0;
    if (BN == 128) return launch<0, 128>(ta, tb, c, c_dtype, ldc, g, accumulate, bias, addend, grp_src, nullptr, 1, nkb, st, stat_partial, ev);
    return launch<0, 64>(ta, tb, c, c_dtype, ldc, g, accumulate, bias, addend, grp_src, nullptr, 1, nkb, st, stat_partial, ev);
  }
  if (kind == 2) {
    g.M = (int)pix; g.Ntot = Cn;
    // 64 output channels: 256-pixel tiles, so that a filled K block (32 KB of pixels + 8 KB of weights) feeds twice the
    // MMA work of a 128 x 64 one (51 instead of 43 FLOP per filled byte).  Launches with fused statistics (partials are
    // laid out per 128-row tile) or the eval-BatchNorm epilogue keep 128 rows, as does a map that 256-pixel boxes do not tile.
    int bh256 = 1, bn256 = 1;
    const bool tall = Cn == 64 && stat_partial == nullptr && eval_scale == nullptr && box_for(256, H, W, bh256, bn256);
    if (tall) { g.bhm = bh256; g.bnm = bn256; }
    rc = map4d(&ta, a, N, H, W, Ck, W, g.bhm, g.bnm, 1);
    if (rc) return rc;
    rc = map2d(&tb, b, 16LL * Cn, Ck, ldb, 64);  // MN-major weight [Ck rows][16*Cn]
    if (rc) return rc;
    const int nkb = 4 * (Ck / 64);
    const int BN = Cn > 64 ? 128 : 64;
    if (tall) return launch<2, 64, 256>(ta, tb, c, c_dtype, ldc, g, accumulate, bias, addend, grp_src, nullptr, 1, nkb, st);
    if (BN == 128) return launch<2, 128>(ta, tb, c, c_dtype, ldc, g, accumulate, bias, addend, grp_src, nullptr, 1, nkb, st, stat_partial, ev);
    return launch<2, 64>(ta, tb, c, c_dtype, ldc, g, accumulate, bias, addend, grp_src, nullptr, 1, nkb, st, stat_partial, ev);
  }
  // kind 1: weight gradient
  P2PVG_REQUIRE(c_dtype == P2PVG_F32, P2PVG_ERR_BAD_ARG, "conv_gemm kind 1 writes fp32");
  P2PVG_REQUIRE(stat_partial == nullptr, P2PVG_ERR_BAD_ARG, "conv_gemm: BatchNorm statistics belong to the forward / data-gradient kinds");
  g.Ck = 64;
  // 64 output channels would fill only half of a 128-row MMA tile: swap the operand roles (M = taps*Cn from the gathered map,
  // N = Cm); the partial sums are then [taps*Cn][Cm] and the split-K reduce kernel writes the transposed result
  const int nkb = (int)((pix + 63) / 64);
  g.swap = (Cm == 64 && nkb >= 16 && ws != nullptr && (size_t)2 * taps * Cn * Cm * sizeof(float) <= ws_bytes) ? 1 : 0;
  if (g.swap) {
    g.M = taps * Cn; g.Ntot = Cm;
    rc = map4d(&ta, b, N, g.st * H, g.st * W, Cn, g.bw64, g.bh64, g.bn64, g.st);
    if (rc) return rc;
    rc = map2d(&tb, a, Cm, pix, Cm, 64);
    if (rc) return rc;
  } else {
    g.M = Cm; g.Ntot = taps * Cn;
    rc = map2d(&ta, a, Cm, pix, Cm, 64);  // a_small [pix][Cm] as MN-major A
    if (rc) return rc;
    rc = map4d(&tb, b, N, g.st * H, g.st * W, Cn, g.bw64, g.bh64, g.bn64, g.st);
    if (rc) return rc;
  }
  const int BN = (g.Ntot % 128 == 0) ? 128 : 64;
  const long long tiles = (long long)cdiv(g.M, BLOCK_M) * cdiv(g.Ntot, BN);
  // split-K chosen by a small cost model (units: time of one 128x128x64 k-block on one SM, ~0.22 us): the persistent grid
  // processes ceil(items / SMs) rounds of (k-blocks per item + fixed per-item cost); partial sums cost a write + read
  int splits = g.swap ? 2 : 1;
  {
    double best = 1e300;
    const int maxs = nkb / 8 < 64 ? nkb / 8 : 64;
    const int smin = g.swap ? 2 : 1;
    for (int s = smin; s <= (maxs < smin ? smin : maxs); s++) {
      const int kb = cdiv(nkb, s), se = cdiv(nkb, kb);
      if (se > 1 && (ws == nullptr || (size_t)se * g.M * g.Ntot * sizeof(float) > ws_bytes)) continue;
      const long long rounds = cdiv((long long)tiles * se, driver().sms);
      double cost = (double)rounds * (kb + 8.0);
      if (se > 1) cost += (double)se * g.M * g.Ntot * 8.0 / 6.0e12 / (0.22e-6 * BN / 128);
      if (cost < best) { best = cost; splits = se; }
    }
  }
  int kbps = cdiv(nkb, splits);
  splits = cdiv(nkb, kbps);
  float* partial = splits > 1 ? reinterpret_cast<float*>(ws) : nullptr;
  if (BN == 128) rc = launch<1, 128>(ta, tb, c, c_dtype, ldc, g, accumulate, nullptr, nullptr, nullptr, partial, splits, kbps, st);
  else rc = launch<1, 64>(ta, tb, c, c_dtype, ldc, g, accumulate, nullptr, nullptr, nullptr, partial, splits, kbps, st);
  if (rc) return rc;
  if (splits > 1)
    return p2pvg_splitk_reduce(partial, splits, c, P2PVG_F32, ldc, Cm, taps * Cn, accumulate, nullptr, nullptr, 0, g.swap, st);
  P2PVG_REQUIRE(!g.swap, P2PVG_ERR_UNSUPPORTED, "conv_gemm kind 1 (swapped roles) needs the split-K workspace");
  return P2PVG_OK;
}
