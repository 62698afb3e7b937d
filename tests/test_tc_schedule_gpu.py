"""The persistent tensor-core kernels (gemm_tc.cu, conv_gemm.cu) on launches where every CTA runs several tiles, against float64.

A CTA of these kernels walks tiles t = blockIdx.x, +gridDim.x, ...  What crosses from one tile to the next -- the operand-ring
parity, the staging-buffer hand-off, the bias / statistics / eval-coefficient shared-memory halves chosen by tile parity, the
resident weights of the 64-channel 3x3 layers, the phase-fastest tile decode of the transposed convolution -- is only exercised
when tiles > SMs.  Every case here states its schedule with tests/tc_schedule.py and asserts at run time that it runs at least
three rounds with a partial last round and (where the output has more than one column tile) that some CTA changes n0 between
consecutive tiles.  Shapes are searched from a starting point so that the invariants also hold on a device with another SM count.

Three kinds of check:
  * float64 references on the kernels' own bf16 operands, with |got - ref| <= alpha * sum|a b| + beta * |ref|;
  * every fused BatchNorm-statistics row on its own, against the float64 sums of the stored rows it covers;
  * bit-exact slice invariance: kinds 0 / 2 and the non-split gemm_tc fix the accumulation order inside a tile, so rows taken
    from a multi-round launch equal (torch.equal) a launch of just those rows, in which every CTA runs one tile.
"""
import math

import pytest
import torch

from tests.tc_schedule import (alpha_for, assert_multi_round, assert_within, cdiv, conv_ref64, conv_tiles, fit, gemm_tc_tiles,
                               image_slices, ref64, rows_by_tile, sm_count)

pytestmark = pytest.mark.gpu

ACT_LRELU, ACT_TANH = 1, 2
NAN = float("nan")


@pytest.fixture(scope="module")
def K():
    from p2pvg_b200._lib import CudaKernels
    return CudaKernels("cuda")


@pytest.fixture(scope="module")
def sms():
    return sm_count()


def randn(*shape, scale=1.0, dtype=torch.float32):
    return (torch.randn(*shape, device="cuda") * scale).to(dtype)


# ------------------------------------------------------------------ gemm_tc (bf16)

def gemm_locate(s):
    return lambda idx: s.where(0, idx[0] // 128, idx[1] // s.BN)


GEMM_CASES = [
    # id, a_mn, b_mn, N candidates, K, starting M.  Tails: M % 128, N % 32 (scalar store path), K % 64.
    ("kk_bn128_tails", False, False, (1000, 1256), 328, 7000),
    ("mnmn_bn128", True, True, (2048, 2304), 1024, 2560),
    ("kmn_bn64_tails", False, True, (40,), 200, 50000),     # N <= 64: BN 64, a single column tile
    ("mnk_bn128_tails", True, False, (600, 856), 136, 9608),
]


@pytest.mark.parametrize("case", GEMM_CASES, ids=[c[0] for c in GEMM_CASES])
def test_gemm_tc_multi_round(K, sms, case):
    name, a_mn, b_mn, ncands, Kd, M0 = case
    (M, N), s = fit(((M0 + 128 * j, N) for N in ncands for j in range(400)), lambda M, N: gemm_tc_tiles(M, N, Kd, sms),
                    need_n_change=ncands[0] > 64)
    assert s.splits == 1
    assert_multi_round(s, need_n_change=s.BN == 128)
    torch.manual_seed(11)
    A = randn(*((Kd, M) if a_mn else (M, Kd)), dtype=torch.bfloat16)
    B = randn(*((Kd, N) if b_mn else (N, Kd)), dtype=torch.bfloat16)
    bias = randn(N)
    lda = M if a_mn else Kd
    # slices of whole 128-row blocks from the first, a middle and the last round; each sub-launch runs one tile per CTA and
    # must not switch to split-K (K < 16 * 64, or >= 120 tiles)
    per = sms // s.tiles_n
    assert Kd < 16 * 64 or per * s.tiles_n >= 120
    starts = (0, s.tiles_m // 2, s.tiles_m - per)
    K.set_gemm_impl("tc")
    try:
        for cdt in (torch.float32, torch.bfloat16):
            C = torch.full((M, N), NAN, device="cuda", dtype=cdt)   # every element must be written
            K.gemm(A, B, C, M, N, Kd, a_mn=a_mn, b_mn=b_mn)
            ref, absref = ref64(A, B, a_mn, b_mn)
            assert_within(C, ref, absref, Kd, cdt, name=f"gemm_tc {name} {cdt} plain", locate=gemm_locate(s))
            add, C0 = randn(M, N, dtype=cdt), randn(M, N, dtype=cdt)
            C = C0.clone()
            K.gemm(A, B, C, M, N, Kd, a_mn=a_mn, b_mn=b_mn, accumulate=True, bias=bias, addend=add)
            ref, absref = ref64(A, B, a_mn, b_mn, bias, add, C0)
            assert_within(C, ref, absref, Kd, cdt, name=f"gemm_tc {name} {cdt} acc+bias+addend", locate=gemm_locate(s))
            del ref, absref
            for mt0 in starts:
                r0, r1 = mt0 * 128, min((mt0 + per) * 128, M)
                sub = gemm_tc_tiles(r1 - r0, N, Kd, sms)
                assert sub.splits == 1 and sub.tiles <= sms
                Asub = A[:, r0:r1] if a_mn else A[r0:r1]
                Cs = C0[r0:r1].clone()
                K.gemm(Asub, B, Cs, r1 - r0, N, Kd, a_mn=a_mn, b_mn=b_mn, lda=lda, accumulate=True, bias=bias, addend=add[r0:r1])
                assert torch.equal(Cs, C[r0:r1]), f"gemm_tc {name} {cdt}: rows [{r0}, {r1}) differ from a launch of just those rows"
    finally:
        K.set_gemm_impl("auto")


def test_gemm_tc_splitk_multi_round(K, sms):
    """Split-K (few output tiles, long K) with bias + addend + accumulate applied by splitk_reduce_kernel.  The split rule
    targets 2 * SMs work items, so tiles * splits stays below 2 * SMs + 120: the launch spans three rounds, the last partial."""
    Kd = 1536
    cands = ((128 * tm - 28, N) for tm in range(17, 8, -1) for N in (833, 705, 961))
    (M, N), s = fit(cands, lambda M, N: gemm_tc_tiles(M, N, Kd, sms), min_tiles=2 * sms + 1)
    assert s.splits > 1 and s.rounds >= 3
    torch.manual_seed(12)
    A, B = randn(M, Kd, dtype=torch.bfloat16), randn(N, Kd, dtype=torch.bfloat16)
    bias = randn(N)
    K.set_gemm_impl("tc")
    try:
        for cdt in (torch.float32, torch.bfloat16):
            add, C0 = randn(M, N, dtype=cdt), randn(M, N, dtype=cdt)
            C = C0.clone()
            K.gemm(A, B, C, M, N, Kd, accumulate=True, bias=bias, addend=add)
            ref, absref = ref64(A, B, False, False, bias, add, C0)
            # each split accumulates kb_per_split K blocks; the reduce adds `splits` fp32 partials
            assert_within(C, ref, absref, s.kb_per_split * 64 + 16 * s.splits, cdt, name=f"gemm_tc split-K x{s.splits} {cdt}",
                          locate=gemm_locate(s))
    finally:
        K.set_gemm_impl("auto")


# ------------------------------------------------------------------ tf32 gemm (fp32 operands, K-major)

@pytest.mark.parametrize("M,N,Kd", [(30 * 256, 4 * 256, 144), (60 * 256, 4 * 512, 264)], ids=["C2_lstm_input", "C5_lstm_input"])
def test_tf32_gemm_multi_round(K, sms, M, N, Kd):
    """The LSTM input GEMMs, (S*B) x 4R x in_pitch, at the C2 and C5 sizes."""
    s = gemm_tc_tiles(M, N, Kd, sms, tf32=True)
    assert_multi_round(s)
    torch.manual_seed(13)
    A, B, bias = randn(M, Kd), randn(N, Kd), randn(N)
    add, C0 = randn(M, N), randn(M, N)
    C = C0.clone()
    Kc = K.with_mode(tf32=True)
    Kc.gemm(A, B, C, M, N, Kd, accumulate=True, bias=bias, addend=add)
    for r0 in range(0, M, 2048):   # float64 reference in row blocks
        r1 = min(M, r0 + 2048)
        ref, absref = ref64(A[r0:r1], B, bias=bias, addend=add[r0:r1], c0=C0[r0:r1])
        assert_within(C[r0:r1], ref, absref, Kd, torch.float32, name=f"tf32 {M}x{N}x{Kd} rows {r0}", alpha=alpha_for(Kd, tf32=True),
                      locate=lambda idx, r0=r0: s.where(0, (r0 + idx[0]) // 128, idx[1] // s.BN))
        del ref, absref
    diff = (C[:2048].double() - ref64(A[:2048], B, bias=bias, addend=add[:2048], c0=C0[:2048])[0]).abs().max().item()
    assert diff > 1e-4, "the tf32 mode gave fp32-exact results: it did not run on the tensor cores"


# ------------------------------------------------------------------ implicit-GEMM convolutions, kinds 0 / 2 / 3 / 5

def conv_operands(kind, N, H, Ck, Cn):
    """a: the kernel's A operand (NHWC), b: its packed weight.  Scales keep outputs O(1)."""
    taps = 9 if kind >= 3 else 16
    Ha = 2 * H if kind == 0 else H
    a = randn(N, Ha, Ha, Ck, scale=0.5, dtype=torch.bfloat16)
    b = randn(Ck if kind == 2 else Cn, taps * (Cn if kind == 2 else Ck), scale=1.0 / math.sqrt(taps * Ck), dtype=torch.bfloat16)
    return a, b


def out_shape(kind, N, H, Cn):
    return (N, 2 * H, 2 * H, Cn) if kind == 2 else (N, H, H, Cn)


def conv_locate(kind, H, s):
    def loc(idx):
        n, y, x, c = idx
        if kind == 2:
            row, ph = (n * H + y // 2) * H + x // 2, (y & 1) * 2 + (x & 1)
        else:
            row, ph = (n * H + y) * H + x, 0
        return s.where(0, row // s.BM, c // s.BN, ph)
    return loc


CONV_CASES = [
    # id, kind, H (small map), Ck, Cn candidates, starting N, image step, kind-2 images per addend group
    ("k0_hw256_cn576", 0, 16, 128, (576, 640), 40, 1, 0),        # 2 tiles per image; Cn tail: the last column tile is half
    ("k0_hw16_cn576", 0, 4, 256, (576, 640), 657, 1, 0),         # 8 images per tile; ragged last tile
    ("k0_bn64", 0, 8, 128, (64,), 800, 1, 0),                    # BN 64: a single column tile
    ("k2_hw256_cn256", 2, 16, 128, (256, 640), 25, 5, 5),
    ("k2_hw16_bn64", 2, 4, 256, (64,), 800, 16, 16),
    ("k3_bres", 3, 32, 64, (64,), 50, 1, 0),                     # resident weights must survive every tile of the CTA
    ("k3_cn576", 3, 32, 128, (576, 640), 10, 1, 0),
    ("k5_bres", 5, 32, 64, (64,), 50, 1, 0),
    ("k5_ck128", 5, 32, 128, (128,), 50, 1, 0),
]


def conv_fit(kind, H, Ck, Cn_cands, N0, step, sms, **kw):
    # Cn <= 128 is a single column tile (BN = 64 or 128), n0 = 0 on every tile: no n0 change to ask for.  Kind 2 decodes nt from
    # t >> 2 and the phase from t & 3; on 132 SMs the phase of a CTA never changes (132 % 4 == 0).  kw: stat / eval_epi.
    cands = ((N0 + step * j, Cn) for Cn in Cn_cands for j in range(200))
    return fit(cands, lambda N, Cn: conv_tiles(kind, N, H, H, Ck, Cn, 0, sms, **kw), need_n_change=Cn_cands[0] > 128)


@pytest.mark.parametrize("case", CONV_CASES, ids=[c[0] for c in CONV_CASES])
def test_conv_gemm_multi_round(K, sms, case):
    name, kind, H, Ck, Cn_cands, N0, step, B = case
    (N, Cn), s = conv_fit(kind, H, Ck, Cn_cands, N0, step, sms)
    assert s.bres == name.endswith("bres")
    assert s.BM == (256 if kind == 2 and Cn == 64 else 128)
    torch.manual_seed(14)
    a, b = conv_operands(kind, N, H, Ck, Cn)
    bias = randn(Cn) if kind != 5 else None
    taps = 9 if kind >= 3 else 16
    ref_c, abs_c = conv_ref64(kind, a, b, N, H, H, Ck, Cn)
    combos = [(cdt, None) for cdt in (torch.float32, torch.bfloat16)]
    add = src = None
    if kind == 2:
        G, nsrc = N // B, 3
        src = torch.tensor([(3 * g + 1) % nsrc for g in range(G)], dtype=torch.int32, device="cuda")
        idx = torch.tensor([int(src[n // B]) * B + n % B for n in range(N)], device="cuda")
        add = randn(nsrc * B, 2 * H, 2 * H, Cn)
        combos = [(torch.float32, torch.float32), (torch.bfloat16, torch.float32), (torch.float32, torch.bfloat16),
                  (torch.bfloat16, torch.bfloat16)]
    HW = H * H
    unit = math.lcm(step, max(1, s.BM // HW))
    for cdt, adt in combos:
        out = torch.full(out_shape(kind, N, H, Cn), NAN, device="cuda", dtype=cdt)
        kw = dict(bias=bias)
        ref, absref = ref_c.clone(), abs_c.clone()
        if bias is not None:
            ref += bias.double()
            absref += bias.double().abs()
        if adt is not None:
            a_ = add.to(adt)
            kw.update(addend=a_, grp_src=src, imgs_per_group=B)
            ref += a_.double()[idx]
            absref += a_.double()[idx].abs()
        K.conv_gemm(kind, a, b, out, N, H, H, Ck, Cn, **kw)
        assert_within(out, ref, absref, taps * Ck, cdt, name=f"conv kind {kind} {name} out={cdt} addend={adt}",
                      locate=conv_locate(kind, H, s))
        del ref, absref
        for i0, i1 in image_slices(N, HW, unit, s, sms):
            sub = conv_tiles(kind, i1 - i0, H, H, Ck, Cn, 0, sms)
            assert sub.tiles <= sms
            o = torch.empty(out_shape(kind, i1 - i0, H, Cn), device="cuda", dtype=cdt)
            kws = dict(kw)
            if adt is not None:
                kws["grp_src"] = src[i0 // B:]
            K.conv_gemm(kind, a[i0:i1], b, o, i1 - i0, H, H, Ck, Cn, **kws)
            assert torch.equal(o, out[i0:i1]), f"{name} {cdt}/{adt}: images [{i0}, {i1}) differ from a launch of just those images"


# ------------------------------------------------------------------ weight gradients, kinds 1 / 4

WGRAD_CASES = [
    # id, kind, H (small map; kind 4: the map), Cm, Cn, starting N.  The split-K cost model picks the split count.
    ("k1_swap", 1, 4, 64, 2048, 64),        # 64 output channels: swapped operand roles, >= 16 K blocks
    ("k1_noswap", 1, 4, 384, 1024, 64),
    ("k4_bw64_noswap", 4, 128, 256, 512, 2),   # W = 128 > 64: each 64-pixel K block is half a row
    ("k4_bw64_swap", 4, 128, 64, 1024, 2),
]


@pytest.mark.parametrize("case", WGRAD_CASES, ids=[c[0] for c in WGRAD_CASES])
def test_conv_weight_gradient_multi_round(K, sms, case):
    """Weight gradients keep few output tiles, so the cost model decides the rounds: each case spans at least three."""
    name, kind, H, Cm, Cn, N0 = case
    (N,), s = fit(((N0 + j,) for j in range(64)), lambda N: conv_tiles(kind, N, H, H, 0, Cn, Cm, sms), need_n_change=False,
                  min_tiles=2 * sms + 1)
    assert s.swap == ("_swap" in name)
    taps = 9 if kind == 4 else 16
    Hb = 2 * H if kind == 1 else H
    torch.manual_seed(15)
    a = randn(N, H, H, Cm, scale=0.5, dtype=torch.bfloat16)
    b = randn(N, Hb, Hb, Cn, scale=0.5, dtype=torch.bfloat16)
    ref, absref = conv_ref64(kind, a, b, N, H, H, 0, Cn, Cm)
    keff = s.kb_per_split * 64 + 16 * s.splits

    def loc(idx):
        i, j = idx
        return s.where(0, j // 128, i // s.BN) if s.swap else s.where(0, i // 128, j // s.BN)
    out = torch.full((Cm, taps * Cn), NAN, device="cuda")
    K.conv_gemm(kind, a, b, out, N, H, H, 0, Cn, Cm=Cm)
    assert_within(out, ref, absref, keff, torch.float32, name=f"wgrad {name} splits={s.splits}", locate=loc)
    c0 = randn(Cm, taps * Cn)
    out = c0.clone()
    K.conv_gemm(kind, a, b, out, N, H, H, 0, Cn, Cm=Cm, accumulate=True)
    assert_within(out, ref + c0.double(), absref + c0.double().abs(), keff, torch.float32, name=f"wgrad {name} accumulate", locate=loc)


# ------------------------------------------------------------------ fused BatchNorm statistics, every partial row

STAT_CASES = [
    # id, kind, H, Ck, Cn candidates, starting N, image step (= images per BatchNorm group)
    ("k0_hw256_cn1024", 0, 16, 128, (1024, 1280), 28, 4),       # 8 column tiles; bn_fwd_stats needs C / 8 to divide 256
    ("k2_hw256_cn256", 2, 16, 128, (256, 640), 25, 5),
    ("k2_hw16_bn64", 2, 4, 256, (64,), 800, 16),
]


@pytest.mark.parametrize("cdt", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("case", STAT_CASES, ids=[c[0] for c in STAT_CASES])
def test_fused_statistics_every_row_multi_round(K, sms, case, cdt):
    name, kind, H, Ck, Cn_cands, N0, B = case
    (N, Cn), s = conv_fit(kind, H, Ck, Cn_cands, N0, B, sms, stat=True)
    assert s.BM == 128
    torch.manual_seed(16)
    a, b = conv_operands(kind, N, H, Ck, Cn)
    bias = randn(Cn)
    phases = s.phases
    part = torch.full((s.tiles_m * phases, Cn, 2), NAN, device="cuda")
    out = torch.empty(out_shape(kind, N, H, Cn), device="cuda", dtype=cdt)
    K.conv_gemm(kind, a, b, out, N, H, H, Ck, Cn, bias=bias, stat_partial=part)
    plain = torch.empty_like(out)
    K.conv_gemm(kind, a, b, plain, N, H, H, Ck, Cn, bias=bias)
    assert torch.equal(out, plain), "the fused statistics must not change the stored output"
    rows = rows_by_tile(out, kind, N, H, Cn, s.tiles_m)
    # each partial row: a fixed-order fp32 tree over 128 stored values (per-warp butterfly of 32, then four warps), each add
    # off by at most 2^-24 of the magnitude summed so far: 8 levels -> 2^-21; 2^-18 leaves 8x
    a_stat = 2.0 ** -18

    def loc(idx):
        r, c = idx[0], idx[1]
        return s.where(0, r // phases, c // s.BN, r % phases)
    for j, (val, mag) in enumerate(((rows.sum(1), rows.abs().sum(1)), ((rows * rows).sum(1), (rows * rows).sum(1)))):
        assert_within(part[:, :, j], val, mag, 0, torch.float32, alpha=a_stat, locate=loc,
                      name=f"stat rows {name} {cdt} {'sum' if j == 0 else 'sum of squares'}")
    del rows
    # tile-aligned slices: output and statistics rows bit-identical to a launch of just those images
    HW = H * H
    unit = math.lcm(B, max(1, 128 // HW))
    for i0, i1 in image_slices(N, HW, unit, s, sms):
        p = torch.full((cdiv((i1 - i0) * HW, 128) * phases, Cn, 2), NAN, device="cuda")
        o = torch.empty(out_shape(kind, i1 - i0, H, Cn), device="cuda", dtype=cdt)
        K.conv_gemm(kind, a[i0:i1], b, o, i1 - i0, H, H, Ck, Cn, bias=bias, stat_partial=p)
        t0 = i0 * HW // 128
        assert torch.equal(o, out[i0:i1]) and torch.equal(p, part[t0 * phases:t0 * phases + p.shape[0]]), \
            f"{name}: images [{i0}, {i1}) or their statistics rows differ from a launch of just those images"
    # finalize per group of B images, against the statistics of the stored output
    G, Hout = N // B, (2 * H if kind == 2 else H)
    R = B * Hout * Hout
    gamma, beta = torch.rand(Cn, device="cuda") + 0.5, torch.randn(Cn, device="cuda")
    outs = [torch.empty(G * Cn, device="cuda") for _ in range(5)]
    K.bn_fwd_finalize_tiles(part, (B * HW // 128) * phases, Cn, 1, G, R, Cn, gamma, beta, *outs)
    refs = [torch.empty(G * Cn, device="cuda") for _ in range(5)]
    K.bn_fwd_stats(out, G, R, Cn, gamma, beta, *refs)
    for x, y, nm in zip(outs, refs, ("mean", "invstd", "var_unbiased", "scale", "shift")):
        assert torch.allclose(x, y, rtol=2e-5, atol=2e-6), nm


# ------------------------------------------------------------------ eval-BatchNorm epilogue

EVAL_CASES = [
    ("k0_hw256_cn576", 0, 16, 128, (576, 640), 40, 1, 0),
    ("k2_hw256_cn256", 2, 16, 128, (256, 640), 25, 5, 5),
    ("k2_hw16_bn64", 2, 4, 256, (64,), 800, 16, 16),
]


@pytest.mark.parametrize("act", [ACT_LRELU, ACT_TANH], ids=["lrelu", "tanh"])
@pytest.mark.parametrize("case", EVAL_CASES, ids=[c[0] for c in EVAL_CASES])
def test_eval_epilogue_multi_round(K, sms, case, act):
    """act(scale * (conv + bias + addend) + shift) stored by the epilogue, against float64."""
    name, kind, H, Ck, Cn_cands, N0, step, B = case
    (N, Cn), s = conv_fit(kind, H, Ck, Cn_cands, N0, step, sms, eval_epi=True)
    assert s.BM == 128
    torch.manual_seed(17)
    a, b = conv_operands(kind, N, H, Ck, Cn)
    bias = randn(Cn)
    sc, sh = torch.rand(Cn, device="cuda") + 0.5, randn(Cn)
    pre, mag = conv_ref64(kind, a, b, N, H, H, Ck, Cn)
    pre += bias.double()
    mag += bias.double().abs()
    kw = dict(bias=bias)
    if kind == 2:
        G, nsrc = N // B, 2
        src = torch.tensor([(g + 1) % nsrc for g in range(G)], dtype=torch.int32, device="cuda")
        idx = torch.tensor([int(src[n // B]) * B + n % B for n in range(N)], device="cuda")
        add = randn(nsrc * B, 2 * H, 2 * H, Cn, dtype=torch.bfloat16)
        kw.update(addend=add, grp_src=src, imgs_per_group=B)
        pre += add.double()[idx]
        mag += add.double()[idx].abs()
    pre = pre * sc.double() + sh.double()
    # a Lipschitz-1 activation passes the error of its argument on unchanged: the bound is on scale * |conv terms| + |shift|
    mag = mag * sc.double() + sh.double().abs()
    ref = torch.where(pre > 0, pre, 0.2 * pre) if act == ACT_LRELU else torch.tanh(pre)
    del pre
    for cdt in (torch.bfloat16, torch.float32):
        out = torch.full(out_shape(kind, N, H, Cn), NAN, device="cuda", dtype=cdt)
        K.conv_gemm(kind, a, b, out, N, H, H, Ck, Cn, eval_scale=sc, eval_shift=sh, act=act, **kw)
        assert_within(out, ref, mag, 16 * Ck, cdt, name=f"eval epilogue {name} act={act} {cdt}", locate=conv_locate(kind, H, s))
