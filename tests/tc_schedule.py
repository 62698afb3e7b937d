"""Host-side launch decisions of the persistent tensor-core kernels, mirrored in Python, plus the float64 references and the
error bound the multi-round tests (tests/test_tc_schedule_gpu.py) and the launch tests share.

The persistent kernels (gemm_tc.cu, conv_gemm.cu) launch grid = min(tiles, SMs) CTAs and every CTA walks the tiles
t = blockIdx.x, blockIdx.x + gridDim.x, ...  `gemm_tc_tiles` and `conv_tiles` transcribe the launchers' choices (tile width,
split-K, resident weights, swapped operand roles, phases) so that a test can state, and assert, how many rounds its launch runs
and which tiles each CTA visits.  They are literal transcriptions: when a launcher changes, the line references below say what to
re-read.
"""
from dataclasses import dataclass

import torch
import torch.nn.functional as F

BLOCK_M = 128
GEMM_WS_BYTES = 256 << 20   # CudaKernels.gemm_workspace(): the split-K / kind-1 partial-sum workspace


def cdiv(a, b):
    return (a + b - 1) // b


def sm_count(dev=None):
    """What the launchers read through cudaDevAttrMultiProcessorCount (tc_common.cuh driver(), :383-397)."""
    return torch.cuda.get_device_properties(dev if dev is not None else torch.cuda.current_device()).multi_processor_count


@dataclass
class Schedule:
    tiles: int            # tiles of the launch, split-K slices and phases included
    splits: int
    phases: int
    BN: int
    tiles_m: int
    tiles_n: int
    grid: int
    sms: int
    kb_per_split: int = 0
    bres: bool = False
    swap: bool = False
    BM: int = BLOCK_M     # rows (pixels) of one M tile: 256 for the tall kind-2 tiles, else 128

    def decode(self, t):
        """(z, mt, nt, ph) of tile t, as the producer and epilogue decode it (conv_gemm.cu:127-130, :242-245; gemm_tc.cu:49-51)."""
        ph = t & 3 if self.phases == 4 else 0
        t2 = t >> 2 if self.phases == 4 else t
        tiles_mn = self.tiles_m * self.tiles_n
        z = t2 // tiles_mn
        r = t2 - z * tiles_mn
        mt = r // self.tiles_n
        return z, mt, r - mt * self.tiles_n, ph

    def tile_index(self, z, mt, nt, ph=0):
        t2 = (z * self.tiles_m + mt) * self.tiles_n + nt
        return t2 * 4 + ph if self.phases == 4 else t2

    def seq(self, cta):
        """The tiles CTA `cta` runs, in order, as (z, mt, nt, ph)."""
        return [self.decode(t) for t in range(cta, self.tiles, self.grid)]

    @property
    def rounds(self):
        return cdiv(self.tiles, self.grid)

    def n0_changes(self):
        """Some CTA runs two consecutive tiles with different n0 (the epilogue's bias / eval-coefficient halves then hold different
        columns).  For kinds 0 / 1 and gemm_tc that needs tiles_n not dividing gridDim; kind 2 decodes nt from t >> 2."""
        for c in range(self.grid):
            s = self.seq(c)
            if any(a[2] != b[2] for a, b in zip(s, s[1:])):
                return True
        return False

    def where(self, z, mt, nt, ph=0):
        t = self.tile_index(z, mt, nt, ph)
        return f"tile (z={z}, mt={mt}, nt={nt}, ph={ph}) = t {t}: CTA {t % self.grid}, its tile #{t // self.grid}"


def assert_multi_round(s, need_n_change=True, min_tiles=None):
    """The invariants every multi-round case states at run time: at least three rounds of tiles with a partial last round, and
    (unless the output has a single column tile, so every tile's n0 is 0) a CTA whose consecutive tiles change n0."""
    need = 3 * s.sms if min_tiles is None else min_tiles
    assert s.grid == s.sms, f"grid {s.grid} < {s.sms} SMs: not a persistent multi-round launch"
    assert s.tiles >= need, f"{s.tiles} tiles < {need}: the case does not reach the rounds it is meant to test"
    assert s.tiles % s.sms != 0, f"{s.tiles} tiles fill every round: no partial last round"
    if need_n_change:
        assert s.tiles_n > 1 and s.n0_changes(), f"tiles_n={s.tiles_n} on {s.sms} SMs: every CTA keeps one n0"


def fit(cands, sched, need_n_change=True, min_tiles=None):
    """The first candidate shape whose schedule meets the multi-round invariants (fails loudly if none does)."""
    for shape in cands:
        s = sched(*shape)
        try:
            assert_multi_round(s, need_n_change, min_tiles)
        except AssertionError:
            continue
        return shape, s
    raise AssertionError("no candidate shape reaches the rounds this case is meant to test on this device")


def gemm_tc_tiles(M, N, K, sms, tf32=False, ws_bytes=GEMM_WS_BYTES):
    """p2pvg_gemm_tc (gemm_tc.cu:214-241) and p2pvg_gemm_tf32 (gemm_tc.cu:190-198); grid: launch() (gemm_tc.cu:157) and
    launch_persistent() (tc_common.cuh:429-430)."""
    BN = 128 if N > 64 else 64
    tiles_m, tiles_n = cdiv(M, BLOCK_M), cdiv(N, BN)
    if tf32:   # no split-K on the tf32 path
        nkb = cdiv(K, 32)
        return Schedule(tiles_m * tiles_n, 1, 1, BN, tiles_m, tiles_n, min(tiles_m * tiles_n, sms), sms, nkb)
    nkb = cdiv(K, 64)
    tiles = tiles_m * tiles_n
    splits = 1
    if tiles < 120 and nkb >= 16:
        want = (2 * sms + tiles - 1) // tiles
        maxs = nkb // 8
        splits = max(1, min(want, maxs))
        while splits > 1 and splits * M * N * 4 > ws_bytes:
            splits //= 2
    kbps = cdiv(nkb, splits)
    splits = cdiv(nkb, kbps)
    total = tiles * splits
    return Schedule(total, splits, 1, BN, tiles_m, tiles_n, min(total, sms), sms, kbps)


def box_for(P, H, W):
    """conv_gemm.cu box_for (:454-466): whether P consecutive small-map pixels form one TMA pixel box."""
    HW = H * W
    if HW >= P:
        if P % W != 0 or H % (P // W) != 0:
            return False
        bh, bn = P // W, 1
    else:
        if P % HW != 0:
            return False
        bh, bn = H, P // HW
    return bh * 2 <= 256 and W * 2 <= 256 and bn <= 256


def conv_tiles(kind, N, H, W, Ck, Cn, Cm, sms, ws_bytes=GEMM_WS_BYTES, bres_enabled=True, swap_enabled=True, stat=False,
               eval_epi=False):
    """p2pvg_conv_gemm (conv_gemm.cu:501-636); grid: launch_t() (conv_gemm.cu:479) and launch_persistent()
    (tc_common.cuh:429-430).  H, W: small-map size.  stat / eval_epi: the launch has fused statistics / the eval-BatchNorm
    epilogue (kind 2 then keeps 128-row tiles)."""
    taps = 9 if kind >= 3 else 16
    k = 0 if kind in (3, 5) else 1 if kind == 4 else kind
    pix = N * H * W
    if k == 0:
        BN = 128 if Cn > 64 else 64
        bres = BN == 64 and Cn == 64 and Ck == 64 and taps <= 9 and bres_enabled
        tm, tn = cdiv(pix, BLOCK_M), cdiv(Cn, BN)
        return Schedule(tm * tn, 1, 1, BN, tm, tn, min(tm * tn, sms), sms, taps * (Ck // 64), bres=bres)
    if k == 2:
        BN = 128 if Cn > 64 else 64
        # conv_gemm.cu:574-576: 64 output channels run on 256-pixel tiles unless the launch has statistics (partials are per
        # 128-row tile) or the eval epilogue, or 256-pixel boxes do not tile the map
        BM = 256 if Cn == 64 and not stat and not eval_epi and box_for(256, H, W) else BLOCK_M
        tm, tn = cdiv(pix, BM), cdiv(Cn, BN)
        return Schedule(tm * tn * 4, 1, 4, BN, tm, tn, min(tm * tn * 4, sms), sms, 4 * (Ck // 64), BM=BM)
    # kind 1 / 4: weight gradient, split-K by the cost model
    nkb = cdiv(pix, 64)
    swap = Cm == 64 and swap_enabled and nkb >= 16 and 2 * taps * Cn * Cm * 4 <= ws_bytes
    M, Ntot = (taps * Cn, Cm) if swap else (Cm, taps * Cn)
    BN = 128 if Ntot % 128 == 0 else 64
    tiles = cdiv(M, BLOCK_M) * cdiv(Ntot, BN)
    splits = 2 if swap else 1
    best = 1e300
    maxs = min(nkb // 8, 64)
    smin = 2 if swap else 1
    for s in range(smin, (smin if maxs < smin else maxs) + 1):
        kb = cdiv(nkb, s)
        se = cdiv(nkb, kb)
        if se > 1 and se * M * Ntot * 4 > ws_bytes:
            continue
        rounds = cdiv(tiles * se, sms)
        cost = rounds * (kb + 8.0)
        if se > 1:
            cost += se * M * Ntot * 8.0 / 6.0e12 / (0.22e-6 * BN / 128)
        if cost < best:
            best, splits = cost, se
    kbps = cdiv(nkb, splits)
    splits = cdiv(nkb, kbps)
    tm, tn = cdiv(M, BLOCK_M), cdiv(Ntot, BN)
    total = tm * tn * splits
    return Schedule(total, splits, 1, BN, tm, tn, min(total, sms), sms, kbps, swap=swap)


def image_slices(N, HW, unit, s, sms):
    """Three tile-aligned image ranges (first, middle, last round) whose launch has at most `sms` tiles."""
    tiles_per_img = lambda n: cdiv(n * HW, s.BM) * s.tiles_n * s.phases
    ni = unit
    while ni + unit <= N and tiles_per_img(ni + unit) <= sms:
        ni += unit
    mid = (N // 2) // unit * unit
    last = -(-(N - ni) // unit) * unit
    return [(0, ni), (mid, min(N, mid + ni)), (last, N)]


def rows_by_tile(out, kind, N, H, Cn, tiles_m):
    """The stored output as [tiles_m * phases, 128, Cn] float64: the rows each statistics partial row covers (rows past the
    end are zeros).  Kind 2: partial row (mt, ph) covers phase ph's output pixels of the small-map pixels of tile mt."""
    o = out.double()
    if kind == 2:
        o = o.view(N, H, 2, H, 2, Cn).permute(2, 4, 0, 1, 3, 5).reshape(4, N * H * H, Cn)
    else:
        o = o.reshape(1, N * H * H, Cn)
    P = o.shape[0]
    pad = torch.zeros(P, tiles_m * 128, Cn, dtype=torch.float64, device=o.device)
    pad[:, :o.shape[1]] = o
    return pad.view(P, tiles_m, 128, Cn).transpose(0, 1).reshape(tiles_m * P, 128, Cn)


# ------------------------------------------------------------------ float64 references on the kernels' own (bf16-rounded) operands

def _f64(t):
    return t.double()


def ref64(A, B, a_mn=False, b_mn=False, bias=None, addend=None, c0=None):
    """C = opA(A) opB(B) + bias + addend + c0 in float64, and the same expression over absolute values: the per-element magnitude
    sum_k |a_k b_k| + |bias| + |addend| + |c0| that bounds the fp32 rounding of the kernel's sums.  A: [M,K] (K-major) or
    [K,M] (MN-major); B: [N,K] or [K,N]."""
    a = _f64(A)
    b = _f64(B)
    a = a.t() if a_mn else a
    b = b if b_mn else b.t()
    ref = a @ b
    absref = a.abs() @ b.abs()
    for extra in (bias, addend, c0):
        if extra is not None:
            e = _f64(extra)
            ref += e
            absref += e.abs()
    return ref, absref


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def conv_ref64(kind, a, b, N, H, W, Ck, Cn, Cm=0):
    """Float64 reference (and magnitude) of p2pvg_conv_gemm kind 0..5 on the operands the kernel reads (see the kind table in
    conv_gemm.cu).  Returns NHWC [.., C] outputs; kinds 1 / 4 return [Cm, taps * Cn]."""
    def run(x, w):
        if kind == 0:     # x big [N,2H,2W,Ck]; w [Cn, (4,4,Ck)]
            return _nhwc(F.conv2d(_nchw(x), w.view(Cn, 4, 4, Ck).permute(0, 3, 1, 2), stride=2, padding=1))
        if kind == 2:     # x small [N,H,W,Ck]; w [Ck, (4,4,Cn)]
            return _nhwc(F.conv_transpose2d(_nchw(x), w.view(Ck, 4, 4, Cn).permute(0, 3, 1, 2), stride=2, padding=1))
        if kind == 3:     # w [Cn, (3,3,Ck)]
            return _nhwc(F.conv2d(_nchw(x), w.view(Cn, 3, 3, Ck).permute(0, 3, 1, 2), padding=1))
        if kind == 5:     # taps mirrored: y[p] = sum x[p - (kh-1, kw-1)] w[Cn, kh, kw, Ck] = conv_transpose2d with weight [Ck, Cn, kh, kw]
            return _nhwc(F.conv_transpose2d(_nchw(x), w.view(Cn, 3, 3, Ck).permute(3, 0, 1, 2), padding=1))
        ks, st = (4, 2) if kind == 1 else (3, 1)   # a = x [N,H,W,Cm] (small), b = w [N,st*H,st*W,Cn] (gathered map)
        g = torch.nn.grad.conv2d_weight(_nchw(w), (Cm, Cn, ks, ks), _nchw(x), stride=st, padding=1)
        return g.permute(0, 2, 3, 1).reshape(Cm, ks * ks * Cn)
    a64, b64 = _f64(a), _f64(b)
    return run(a64, b64), run(a64.abs(), b64.abs())


# ------------------------------------------------------------------ the bound

ALPHA_BF16 = 2.0 ** -14
BETA = {torch.bfloat16: 2.0 ** -8, torch.float32: 2.0 ** -22}


def alpha_for(K, tf32=False):
    """Relative bound (to sum_k |a_k b_k|) of the fp32 accumulation of a K-long reduction.  The products of bf16 operands are
    exact in fp32; the accumulator takes one fp32 add per MMA-K step (K/16 for bf16, K/8 for tf32) plus the adds inside one
    MMA, each off by at most 2^-23 of a partial sum no larger than sum |a_k b_k|.  2^-14 covers that up to K ~ 8000; beyond it
    the worst case grows linearly.  tf32 operands keep 10 explicit mantissa bits; the hardware's conversion of an fp32 operand
    is not documented as rounding, so each operand may be off by 2^-10 (truncation) and a product by 2^-9."""
    steps = K / (8 if tf32 else 16) + 16
    acc = max(ALPHA_BF16, steps * 2.0 ** -23)
    return acc + (2.0 ** -9 if tf32 else 0.0)


def assert_within(got, ref, absref, K, out_dtype, name="", locate=None, alpha=None, quiet=False):
    """|got - ref| <= alpha * absref + beta * |ref|: alpha covers the fp32 accumulation (alpha_for), beta the rounding of the
    stored output.  On failure: the worst ratio, its index and (via `locate(index) -> str`) its tile.  Returns the worst ratio."""
    a = alpha_for(K) if alpha is None else alpha
    beta = BETA[out_dtype]
    diff = (got.double() - ref).abs()
    bound = a * absref + beta * ref.abs()
    ratio = torch.where(bound > 0, diff / bound.clamp_min(1e-300), torch.where(diff > 0, torch.inf, 0.0))
    ratio = torch.nan_to_num(ratio, nan=torch.inf)
    worst = ratio.max().item()
    if worst > 1.0:
        idx = tuple(int(i) for i in torch.unravel_index(ratio.argmax(), ratio.shape))
        bad = int((ratio > 1.0).sum().item())
        where = locate(idx) if locate is not None else ""
        raise AssertionError(f"{name}: {bad}/{ratio.numel()} elements out of bound, worst ratio {worst:.3g} at {idx} "
                             f"(got {got[idx].item():.6g}, ref {ref[idx].item():.6g}, bound {bound[idx].item():.3g}) {where}")
    if not quiet:
        print(f"[bound] {name}: worst error/bound {worst:.3g}")
    return worst
