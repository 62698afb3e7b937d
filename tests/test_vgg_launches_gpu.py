"""The bf16 vgg_64 training step's kernel launches against float64, at the shapes of the C3 benchmark configuration (3-channel
64x64 frames, T = 30, B = 128).

  A. every implicit-GEMM launch of the step at its exact C3 shape (tests/vgg_ref.py derives the list from the engine's layer
     tables and rules): float64 on image slices of the first, middle and last round, bit-identity of those slices against a
     launch of just those images, per-(image, channel) sums of the whole output, every fused statistics row and the
     finalized statistics, the kind-4 weight gradients in full, and the two explicit GEMMs of the 3-channel ends;
  B. kind-3 edges the C3 list does not reach but the ABI allows, on multi-round schedules;
  C. the vgg.cu data-movement kernels at C3 sizes (up to 10^9 elements): exact statements, and the vector paths against the
     scalar ones;
  D. an audit of a real bf16 step at T = 30, B = 32: every launch checked on its own operands as it runs, coverage of every
     path of the launch list, and a step bit-identical to the unaudited one.
"""
import math
import time

import numpy as np
import pytest
import torch

from oracle import p2p_oracle as O
from p2pvg_b200.engine import StepPlan
from tests.tc_schedule import BETA, alpha_for, assert_within, cdiv, conv_tiles, gemm_tc_tiles, sm_count
from tests.test_tc_schedule_gpu import fit, image_slices
from tests.vgg_ref import (assert_exact, backward_launches, binary01, bound_check, check_col2im3, check_conv3_sums,
                           check_finalize_vs_output, check_im2col3, check_maxpool, check_stat_rows, check_upsample_bwd,
                           check_upsample_fwd, conv3_ref64_elem, finalize_ref, forward_launches, gemm_ref64, variant, windows,
                           wgrad_ref64)

pytestmark = pytest.mark.gpu

C3 = dict(T=30, B=128, nc=3)
BENCH_OPT = dict(skip_prob=0.0, n_past=1, last_frame_skip=False)
NAN = float("nan")


@pytest.fixture(scope="module")
def K():
    from p2pvg_b200._lib import CudaKernels
    return CudaKernels("cuda")


@pytest.fixture(autouse=True)
def memory_per_test(request):
    if torch.cuda.is_available():
        torch.cuda.reset_peak_memory_stats()
        t0 = time.time()
    yield
    if torch.cuda.is_available():
        print(f"\n[memory] {request.node.name}: {time.time() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


@pytest.fixture(scope="module")
def sms():
    return sm_count()


def c3_plan():
    probs = np.zeros(C3["T"] - 1)
    opt = O.default_opt(**BENCH_OPT)
    return StepPlan(C3["T"], probs, opt)


def randn(*shape, scale=1.0, dtype=torch.bfloat16):
    return (torch.randn(*shape, device="cuda") * scale).to(dtype)


def _release():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------ one kind-3 / kind-5 launch, every check

def slices_with_boundary(N, HW, s, sms, B):
    """Tile-aligned image ranges of the first, middle and last round, each a launch of <= SMs tiles; the middle one straddles
    the boundary between two image groups of B."""
    unit = max(1, 128 // HW)
    first, _, last = image_slices(N, HW, unit, s, sms)
    ni = first[1]
    if ni < 2:
        return [first, last]
    b = (N // 2) // B * B
    i0 = max(unit, (b - ni // 2) // unit * unit)
    return [first, (i0, min(N, i0 + ni)), last]


def run_conv(K, sms, L, cdt, seed, label=""):
    """Launch kind 3 / 5 as L describes (forward_launches / backward_launches entry, or a part-B case) on seeded operands
    and run checks 1-4 of the launch list.  Returns the variant it exercised."""
    kind, N, H, Ck, Cn, B = L["kind"], L["N"], L["H"], L["Ck"], L["Cn"], L["B"]
    HW = H * H
    name = f"{label}{L['name']} kind {kind} N={N} {H}x{H} {Ck}->{Cn} out={str(cdt)[6:]}"
    torch.manual_seed(seed)
    a = randn(N, H, H, Ck, scale=0.5)
    b = randn(Cn, 9 * Ck, scale=1.0 / math.sqrt(9 * Ck))
    bias = randn(Cn, dtype=torch.float32) if L["bias"] else None
    add = src = idx = None
    ipg = L["ipg"]
    if L["addend"]:
        nsrc = L.get("nsrc", 1)
        G = cdiv(N, ipg)
        src = torch.tensor([(g + 1) % nsrc for g in range(G)], dtype=torch.int32, device="cuda")
        srcl = src.tolist()
        idx = torch.tensor([srcl[n // ipg] * ipg + n % ipg for n in range(N)], device="cuda")
        add = randn(nsrc * ipg, H, H, Cn)
    st = L["stat"]
    s = conv_tiles(kind, N, H, H, Ck, Cn, 0, sms)
    part = torch.full((s.tiles_m, Cn, 2), NAN, device="cuda") if st is not None else None
    out = torch.full((N, H, H, Cn), NAN, device="cuda", dtype=cdt)
    K.conv_gemm(kind, a, b, out, N, H, H, Ck, Cn, bias=bias, addend=add, grp_src=src, imgs_per_group=ipg, stat_partial=part)
    torch.cuda.synchronize()
    assert not torch.isnan(out).any(), f"{name}: unwritten output elements"
    # 1 + 2: float64 and bit-identity on slices of the first, middle and last round
    worst = 0.0
    for i0, i1 in slices_with_boundary(N, HW, s, sms, max(1, ipg or B)):
        arows = add[idx[i0:i1]] if add is not None else None
        ref, absref = conv3_ref64_elem(kind, a[i0:i1], b, H, Ck, Cn, bias, arows)
        worst = max(worst, assert_within(out[i0:i1], ref, absref, 9 * Ck, cdt, quiet=True, name=f"{name} images [{i0}, {i1})",
                                         locate=lambda ix, i0=i0: s.where(0, ((i0 + ix[0]) * HW + ix[1] * H + ix[2]) // 128, ix[3] // s.BN)))
        del ref, absref
        sub = conv_tiles(kind, i1 - i0, H, H, Ck, Cn, 0, sms)
        assert sub.tiles <= sms
        o = torch.empty(i1 - i0, H, H, Cn, device="cuda", dtype=cdt)
        p = torch.full((sub.tiles_m, Cn, 2), NAN, device="cuda") if st is not None else None
        kw = {}
        if add is not None:   # the same addend rows, one group per image
            kw = dict(addend=arows.contiguous(), grp_src=torch.arange(i1 - i0, dtype=torch.int32, device="cuda"), imgs_per_group=1)
        K.conv_gemm(kind, a[i0:i1], b, o, i1 - i0, H, H, Ck, Cn, bias=bias, stat_partial=p, **kw)
        assert torch.equal(o, out[i0:i1]), f"{name}: images [{i0}, {i1}) differ from a launch of just those images"
        if p is not None:
            t0 = i0 * HW // 128
            assert torch.equal(p, part[t0:t0 + p.shape[0]]), f"{name}: statistics rows of images [{i0}, {i1}) differ"
        del o, p, arows
    print(f"[bound] {name} slices: worst error/bound {worst:.3g}")
    # 3: every tile, through the per-(image, channel) sums
    check_conv3_sums(out, kind, a, b, N, H, Ck, Cn, bias, add, idx, name=name)
    # 4: statistics rows and the finalize per BatchNorm group
    if st is not None:
        check_stat_rows(part, out, N, H, Cn, name=name)
        check_finalize_vs_output(K, part, st["parts_per_group"], out, N // B, B * HW, Cn, name=name)
    v = variant(kind, Ck, Cn, st is not None, add.dtype if add is not None else None, cdt)
    del a, b, out, part, add
    _release()
    return v


def _dedup(launches):
    seen, out = set(), []
    for L in launches:
        key = (L["kind"], L["N"], L["H"], L["Ck"], L["Cn"], L["bias"], L["addend"], L["stat"] is not None)
        if key not in seen:
            seen.add(key)
            out.append(L)
    return out


def encoder_first(backward):
    """A backward list with the encoder's launches first, in layer order (the engine runs them last, in reverse): each shape
    is then represented by its longest launch (all T B frames) under the encoder layer's name."""
    enc = [L for L in backward if L["name"].startswith("enc")]
    return enc[::-1] + [L for L in backward if not L["name"].startswith("enc")]


def _c3_conv_launches():
    p = c3_plan()
    T, B = C3["T"], C3["B"]
    return _dedup([L for L in forward_launches(T, B, p.S, p.nskip) + encoder_first(backward_launches(T, B, p.S, p.nskip, has_cpc=p.has_cpc))
                   if L["kind"] != 4])


C3_CONV = _c3_conv_launches()


def test_c3_launch_list_matches_the_engine():
    """The derived list has the rows the C3 table has: bres at 64x64, fused statistics exactly from 16x16 down, a bf16 addend
    on every decoder stage entry, and a data gradient per layer: the decoder's at S B = 3712 images (reconstruction calls)
    and B = 128 (the CPC decode and the skip halves), the encoder's at T B = 3840 but none for the first layer."""
    p = c3_plan()
    fwd = forward_launches(C3["T"], C3["B"], p.S, p.nskip)
    bwd = backward_launches(C3["T"], C3["B"], p.S, p.nskip, has_cpc=p.has_cpc)
    assert p.S == 29 and p.nskip == 1 and p.has_cpc
    assert [(L["H"], L["stat"] is not None) for L in fwd if L["name"].startswith("enc")] == \
        [(64, False), (32, False), (32, False), (16, True), (16, True), (16, True), (8, True), (8, True), (8, True)]
    entries = [L for L in fwd if L["name"].endswith(".D")]
    assert [(L["H"], L["stat"] is not None, L["ipg"]) for L in entries] == [(8, True, 128), (16, True, 128), (32, False, 128), (64, False, 128)]
    assert all(L["N"] == 3840 for L in fwd if not L["name"].endswith(".S"))
    assert all(L["N"] == 128 for L in fwd if L["name"].endswith(".S"))
    dec = [L for L in bwd if "dec" in L["name"]]
    assert {(L["kind"], L["N"]) for L in dec if L["name"].startswith("dec") and ".S " not in L["name"]} == {(5, 3712), (4, 3712)}
    assert {(L["kind"], L["N"]) for L in dec if ".S " in L["name"]} == {(5, 128), (4, 128)}
    assert {(L["kind"], L["N"]) for L in dec if L["name"].startswith("cpc ")} == {(5, 128)}
    assert sum(L["kind"] == 5 for L in dec) == 2 * 9 + 4
    assert {L["N"] for L in bwd if L["name"].startswith("enc")} == {3840}
    assert not any(L["name"].startswith("enc0.0") for L in bwd)


@pytest.mark.parametrize("L", C3_CONV, ids=[L["name"].replace(" ", "_") for L in C3_CONV])
def test_c3_conv_launch(K, sms, L):
    """Checks 1-4 of one kind-3 / kind-5 launch of the C3 step, with the engine's output dtype (bf16)."""
    run_conv(K, sms, L, torch.bfloat16, seed=21)


def wgrad_classes(launches):
    """The first kind-4 launch of each (map size, swapped roles) class of a backward list, encoder launches first."""
    sms_ = sm_count() if torch.cuda.is_available() else 132
    seen, out = set(), []
    for L in encoder_first(launches):
        if L["kind"] != 4:
            continue
        s = conv_tiles(4, L["N"], L["H"], L["H"], 0, L["Cn"], L["Cm"], sms_)
        if (L["H"], s.swap) not in seen:
            seen.add((L["H"], s.swap))
            out.append(L)
    return out


_p = c3_plan()
C3_WGRAD = wgrad_classes(backward_launches(C3["T"], C3["B"], _p.S, _p.nskip, has_cpc=_p.has_cpc))


@pytest.mark.parametrize("L", C3_WGRAD, ids=[f"{L['H']}x{L['H']}_{L['Cm']}x{L['Cn']}" for L in C3_WGRAD])
def test_c3_weight_gradient(K, sms, L):
    """One kind-4 launch per (map size, swapped roles) class at C3 size, against a full float64 reduction over all
    N * H * W pixels (K = 15.7M at 64x64)."""
    run_wgrad(K, sms, L)


def run_wgrad(K, sms, L):
    """A kind-4 launch as L describes.  Zero-mean operands would cancel: over K = N H W the worst-case accumulation bound is
    larger than the result itself.  So (1) 0 / 1 operands, whose fp32 sums are exact integers: the result must equal float64
    bit for bit, and one lost 64-pixel block or split changes it; (2) real operands that do not cancel (one positive, one of
    mean 1/2), so that the bound is a small fraction of the value."""
    N, H, Cm, Cn = L["N"], L["H"], L["Cm"], L["Cn"]
    s = conv_tiles(4, N, H, H, 0, Cn, Cm, sms)
    name = f"wgrad {L['name']} {H}x{H} {Cm}x{Cn} swap={s.swap} splits={s.splits}"
    torch.manual_seed(22)
    a, b = binary01((N, H, H, Cm)), binary01((N, H, H, Cn))
    out = torch.full((Cm, 9 * Cn), NAN, device="cuda")
    K.conv_gemm(4, a, b, out, N, H, H, 0, Cn, Cm=Cm)
    assert_exact(out, wgrad_ref64(a, b, N, H, Cm, Cn)[0], N * H * H, name + " 0/1 operands")
    a = torch.rand(N, H, H, Cm, device="cuda").bfloat16()
    b = randn(N, H, H, Cn, scale=0.5) + 0.5
    K.conv_gemm(4, a, b, out, N, H, H, 0, Cn, Cm=Cm)
    ref, absref = wgrad_ref64(a, b, N, H, Cm, Cn)
    keff = s.kb_per_split * 64 + 16 * s.splits
    assert (ref.abs() >= 0.5 * absref).all()
    assert_within(out, ref, absref, keff, torch.float32, name=f"{name} K={N * H * H} non-cancelling operands")
    del a, b, out, ref, absref
    _release()


def test_c3_end_gemms(K):
    """The explicit GEMMs of the 3-channel ends at C3 size."""
    run_end_gemms(K, C3["T"] * C3["B"] * 64 * 64)


def run_end_gemms(K, M):
    """The explicit GEMMs of the 3-channel ends over M pixels: the first encoder layer ([M, 32] x [64, 32] after im2col3) and
    the last decoder layer ([M, 64] x [64, 32], MN-major weight), and the [64, 32] weight gradient with K = M that both the
    first layer (dy^T col) and the last layer (x^T dcol, row pitch up8(27) = 32) launch."""
    torch.manual_seed(23)
    col = randn(M, 32)
    col[:, 27:] = 0
    w = randn(64, 32, scale=0.3)
    bias = randn(64, dtype=torch.float32)
    out = torch.full((M, 64), NAN, device="cuda", dtype=torch.bfloat16)
    K.gemm(col, w, out, M, 64, 32, bias=bias)
    for r0 in range(0, M, 1 << 21):
        r1 = min(M, r0 + (1 << 21))
        ref, absref = gemm_ref64(col[r0:r1], w, r1 - r0, 64, 32, False, False, 32, 32, bias=bias)
        assert_within(out[r0:r1], ref, absref, 32, torch.bfloat16, quiet=r0 > 0, name=f"enc first layer GEMM rows {r0}")
    a = randn(M, 64)
    wl = randn(64, 32, scale=0.2)
    colT = torch.full((M, 32), NAN, device="cuda", dtype=torch.bfloat16)
    K.gemm(a, wl, colT, M, 32, 64, b_mn=True)
    for r0 in range(0, M, 1 << 21):
        r1 = min(M, r0 + (1 << 21))
        ref, absref = gemm_ref64(a[r0:r1], wl, r1 - r0, 32, 64, False, True, 64, 32)
        assert_within(colT[r0:r1], ref, absref, 64, torch.bfloat16, quiet=r0 > 0, name=f"dec last layer GEMM rows {r0}")
    del col, out, a, colT
    # the first layer's weight gradient, K = M: exact on 0 / 1 operands, and within the bound on operands that do not cancel
    s = gemm_tc_tiles(64, 32, M, sm_count())
    name = f"enc first layer weight gradient K={M} splits={s.splits}"
    dy, col = binary01((M, 64)), binary01((M, 32))
    gw = torch.full((64, 32), NAN, device="cuda")
    K.set_gemm_impl("tc")
    try:
        K.gemm(dy, col, gw, 64, 32, M, a_mn=True, b_mn=True, lda=64, ldb=32)
        assert_exact(gw, gemm_ref64(dy, col, 64, 32, M, True, True, 64, 32)[0], M, name + " 0/1 operands")
        dy = torch.rand(M, 64, device="cuda").bfloat16()
        col = randn(M, 32, scale=0.5) + 0.5
        K.gemm(dy, col, gw, 64, 32, M, a_mn=True, b_mn=True, lda=64, ldb=32)
    finally:
        K.set_gemm_impl("auto")
    ref, absref = gemm_ref64(dy, col, 64, 32, M, True, True, 64, 32)
    assert (ref.abs() >= 0.5 * absref).all()
    assert_within(gw, ref, absref, s.kb_per_split * 64 + 16 * s.splits, torch.float32, name=name)
    del dy, col
    _release()


# ------------------------------------------------------------------ B. kind-3 edges on multi-round schedules

EDGE_CASES = [
    # id, H, Ck, Cn, images per group (0: no addend), nsrc, stats, starting N, image step
    ("add_8x8_ipg1", 8, 256, 640, 1, 3, False, 700, 1),       # 5 column tiles: CTAs change n0 between tiles
    ("add_8x8_ipg3", 8, 256, 256, 3, 3, False, 699, 3),
    ("add_stats_16x16_ipg4", 16, 128, 256, 4, 3, True, 200, 4),
    ("stats_bres_32x32", 32, 64, 64, 0, 0, True, 60, 1),
    ("ragged_8x8", 8, 128, 128, 0, 0, False, 701, 2),
    ("ragged_stats_8x8", 8, 256, 128, 0, 0, True, 701, 2),
    ("rowcoop_add_bn64_32x32", 32, 64, 64, 2, 2, False, 60, 2),
    ("rowcoop_add_bn128_16x16", 16, 128, 128, 2, 3, False, 200, 2),
]


@pytest.mark.parametrize("cdt", [torch.bfloat16, torch.float32], ids=["bf16", "f32"])
@pytest.mark.parametrize("case", EDGE_CASES, ids=[c[0] for c in EDGE_CASES])
def test_kind3_edges_multi_round(K, sms, case, cdt):
    name, H, Ck, Cn, ipg, nsrc, stats, N0, step = case
    ragged = name.startswith("ragged")
    (N,), s = fit(((N0 + step * j,) for j in range(400) if ((N0 + step * j) * H * H % 128 != 0) == ragged),
                  lambda N: conv_tiles(3, N, H, H, Ck, Cn, 0, sms), need_n_change=Cn > 256)
    assert (N * H * H % 128 != 0) == ragged
    if ipg == 1 or ipg == 3:
        assert 128 // (H * H) > 1, "a 128-row tile must hold several images"
    B = ipg if ipg else max(1, 128 // (H * H))
    L = dict(name=name, kind=3, N=N, H=H, Ck=Ck, Cn=Cn, bias=True, addend=ipg > 0, ipg=ipg, B=B, nsrc=nsrc,
             stat=dict(parts_per_group=B * H * H // 128) if stats else None)
    if ragged and stats:
        # rows past the end of the last tile count as zeros of its statistics row; a ragged map has no whole BatchNorm groups
        v = _run_ragged_stats(K, sms, L, cdt)
    else:
        assert not stats or B * H * H % 128 == 0
        v = run_conv(K, sms, L, cdt, seed=24, label="edge ")
    if name.startswith("rowcoop"):
        assert v[-1] == ("rowcoop" if cdt == torch.bfloat16 else "perrow")


def _run_ragged_stats(K, sms, L, cdt):
    N, H, Ck, Cn = L["N"], L["H"], L["Ck"], L["Cn"]
    s = conv_tiles(3, N, H, H, Ck, Cn, 0, sms)
    torch.manual_seed(25)
    a = randn(N, H, H, Ck, scale=0.5)
    b = randn(Cn, 9 * Ck, scale=1.0 / math.sqrt(9 * Ck))
    bias = randn(Cn, dtype=torch.float32)
    part = torch.full((s.tiles_m, Cn, 2), NAN, device="cuda")
    out = torch.full((N, H, H, Cn), NAN, device="cuda", dtype=cdt)
    K.conv_gemm(3, a, b, out, N, H, H, Ck, Cn, bias=bias, stat_partial=part)
    ref, absref = conv3_ref64_elem(3, a, b, H, Ck, Cn, bias)
    assert_within(out, ref, absref, 9 * Ck, cdt, name=f"edge {L['name']} out={cdt}")
    plain = torch.empty_like(out)
    K.conv_gemm(3, a, b, plain, N, H, H, Ck, Cn, bias=bias)
    assert torch.equal(out, plain), "the fused statistics must not change the stored output"
    check_stat_rows(part, out, N, H, Cn, name=f"edge {L['name']} out={cdt}")
    return variant(3, Ck, Cn, True, None, cdt)


# ------------------------------------------------------------------ C. vgg.cu kernels at C3 sizes

DTYPES = [torch.bfloat16, torch.float32]
C3_N = C3["T"] * C3["B"]


def misaligned_like(n, dtype):
    """A flat tensor of n elements whose data pointer is not 16-byte aligned (forces the scalar kernels)."""
    return torch.empty(n + 1, device="cuda", dtype=dtype)[1:]


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "f32"])
def test_maxpool_c3(K, dtype):
    """maxpool2_fwd / maxpool2_bwd on the 64x64x64 encoder map of C3 (N = 3840: 10^9 input elements)."""
    run_maxpool(K, C3_N, 64, 64, dtype, "C3")


def run_maxpool(K, N, H, C, dtype, label):
    """maxpool2_fwd / maxpool2_bwd on an N x H x H x C map with planted ties: equal pairs, four equal values, and -0 / +0.
    The gradient goes to the first maximum in row-major order; the scalar paths equal the vector ones."""
    torch.manual_seed(26)
    x = randn(N, H, H, C, dtype=dtype)
    w = windows(x, N, H, H, C)
    # ties, on every 7th / 11th / 13th window channel
    w[1][..., 0::7].copy_(w[0][..., 0::7])                        # pair (0, 1)
    w[3][..., 3::11].copy_(w[2][..., 3::11])                      # pair (2, 3)
    for k in (1, 2, 3):
        w[k][:, ::5, :, 5::13].copy_(w[0][:, ::5, :, 5::13])      # four equal
    w[0][:, 1::5, :, 6::13] = -0.0                                 # -0 then +0, the others negative
    w[1][:, 1::5, :, 6::13] = 0.0
    w[2][:, 1::5, :, 6::13] = -1.0
    w[3][:, 1::5, :, 6::13] = -2.0
    del w
    y = torch.empty(N, H // 2, H // 2, C, device="cuda", dtype=dtype)
    K.maxpool2_fwd(x, y, N, H, H, C)
    ys = misaligned_like(y.numel(), dtype).view_as(y)
    K.maxpool2_fwd(x, ys, N, H, H, C)
    dy = randn(N, H // 2, H // 2, C, dtype=dtype)
    dx = torch.empty_like(x)
    K.maxpool2_bwd(x, dy, dx, N, H, H, C)
    dxs = misaligned_like(x.numel(), dtype).view_as(x)
    K.maxpool2_bwd(x, dy, dxs, N, H, H, C)
    check_maxpool(x, y, dy, dx, N, H, H, C, f"{label} {dtype}")
    for n0 in range(0, N, 256):
        sl = slice(n0, n0 + 256)
        assert torch.equal(ys[sl], y[sl]) and torch.equal(dxs[sl], dx[sl]), f"scalar and vector paths differ, images [{n0}, ..)"
    print(f"[exact] maxpool2 fwd/bwd {dtype} N={N} {H}x{H}x{C}: exact, scalar == vector")
    del x, y, ys, dy, dx, dxs
    _release()


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "f32"])
def test_upsample_c3(K, dtype):
    """upsample2_fwd / upsample2_bwd at the 64x64 decoder stage entry of C3 (32x32x64 -> 64x64x64 at N = 3840: 10^9 upsampled
    elements)."""
    run_upsample(K, C3_N, 32, 64, dtype, "C3")


def run_upsample(K, N, H, C, dtype, label):
    """upsample2_fwd / upsample2_bwd from an N x H x H x C map: forward exact; backward bit for bit against torch's fp32
    (a + b) + (c + d) and within one rounding of float64; the scalar paths equal the vector ones."""
    torch.manual_seed(27)
    x = randn(N, H, H, C, dtype=dtype)
    u = torch.empty(N, 2 * H, 2 * H, C, device="cuda", dtype=dtype)
    K.upsample2_fwd(x, u, N, H, H, C)
    us = misaligned_like(u.numel(), dtype).view_as(u)
    K.upsample2_fwd(x, us, N, H, H, C)
    check_upsample_fwd(x, u, N, H, H, C, f"{label} {dtype}")
    for n0 in range(0, N, 256):
        assert torch.equal(us[n0:n0 + 256], u[n0:n0 + 256]), f"upsample2_fwd scalar and vector paths differ, images [{n0}, ..)"
    del us
    dy = u.normal_()   # the 64x64 gradient map, reusing the upsampled buffer
    dx = torch.empty(N, H, H, C, device="cuda", dtype=dtype)
    K.upsample2_bwd(dy, dx, N, H, H, C)
    dxs = misaligned_like(dx.numel(), dtype).view_as(dx)
    K.upsample2_bwd(dy, dxs, N, H, H, C)
    worst = check_upsample_bwd(dy, dx, N, H, H, C, f"{label} {dtype}")
    for n0 in range(0, N, 256):
        assert torch.equal(dxs[n0:n0 + 256], dx[n0:n0 + 256]), f"upsample2_bwd scalar and vector paths differ, images [{n0}, ..)"
    print(f"[bound] upsample2 {dtype} N={N} {H}x{H}x{C}: fwd exact, bwd bit-exact, worst error/bound vs float64 {worst:.3g}")
    del x, u, dy, dx, dxs
    _release()


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "f32"])
def test_im2col3_col2im3_c3(K, dtype):
    """The 3-channel ends at C3 size (N = 3840 frames of 64x64x3)."""
    run_im2col3_col2im3(K, C3_N, 64, dtype, "C3")


def run_im2col3_col2im3(K, N, H, dtype, label):
    """The 3-channel ends on N frames of H x H x 3: im2col3's row32 path (ld = 32) against the generic one (ld = 40) and an
    exact statement for both tap signs, pad columns zero; col2im3 within 9 fp32 adds and one rounding."""
    C = 3
    torch.manual_seed(28)
    x = randn(N, H, H, C, dtype=dtype)
    for sgn in (1, -1):
        c32 = torch.full((N * H * H, 32), 7.0, device="cuda", dtype=dtype)
        c40 = torch.full((N * H * H, 40), 7.0, device="cuda", dtype=dtype)
        K.im2col3(x, c32, N, H, H, C, 32, sgn)
        K.im2col3(x, c40, N, H, H, C, 40, sgn)
        check_im2col3(x, c40, N, H, H, C, 40, sgn, f"{label} generic {dtype}")
        check_im2col3(x, c32, N, H, H, C, 32, sgn, f"{label} row32 {dtype}")
        del c32, c40
    ld = 32
    col = randn(N * H * H, ld, dtype=dtype)
    bias = randn(C, dtype=torch.float32)
    y = torch.full((N, H, H, C), NAN, device="cuda", dtype=dtype)
    K.col2im3(col, y, N, H, H, C, ld, bias=bias)
    worst = check_col2im3(col, y, N, H, H, C, ld, bias, f"{label} {dtype}")
    print(f"[bound] im2col3 exact (row32 == generic), col2im3 {dtype}: worst error/bound {worst:.3g}")
    del x, col, y
    _release()


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "f32"])
def test_skip_index_kernels_c3(K, dtype):
    """gather_add, group_sum and add_indexed at the engine's C3 sizes at 64x64x64 (groups of B = 128 images, G = 30 calls):
    n = 33.5M elements per group, 10^9 in all; three distinct skip sources."""
    run_skip_index(K, C3["T"], C3["B"], 64, 64, dtype, gather=True)


def run_skip_index(K, G, B, H, C, dtype, gather):
    """(gather: gather_add,) group_sum and add_indexed over G groups of B images of H x H x C, three distinct skip sources."""
    nsrc = 3
    n = B * H * H * C
    src = torch.tensor([(g + 1) % nsrc for g in range(G)], dtype=torch.int32, device="cuda")
    srcl = src.tolist()
    torch.manual_seed(29)
    big = randn(G * n, dtype=dtype)
    if gather:
        small = randn(nsrc * n, dtype=torch.float32)
        dst0 = big.clone()
        # gather_add: dst[g] += src[grp_src[g]] (fp32 addend); a bf16 destination rounds twice (fp32, then bf16): one bf16 ulp
        K.gather_add(big, small, src, G, n)
        worst = 0.0
        for g in range(G):
            ref = dst0[g * n:(g + 1) * n].double() + small[srcl[g] * n:(srcl[g] + 1) * n].double()
            rel = 2.0 ** -7 if dtype == torch.bfloat16 else 2.0 ** -23
            worst = max(worst, bound_check(big[g * n:(g + 1) * n], ref, rel * ref.abs(), f"gather_add group {g}"))
        print(f"[bound] gather_add {dtype} G={G} n={n}: worst error/bound {worst:.3g}")
        del dst0, small
    # group_sum: out[f] = sum over the groups reading source f (fp32 in group order, one output rounding)
    out = torch.full((nsrc * n,), NAN, device="cuda", dtype=dtype)
    K.group_sum(big, out, src, G, nsrc, n)
    worst = 0.0
    for f in range(nsrc):
        for j0 in range(0, n, 1 << 24):
            j1 = min(n, j0 + (1 << 24))
            gs = [g for g in range(G) if srcl[g] == f]
            ref = sum(big[g * n + j0:g * n + j1].double() for g in gs)
            mag = sum(big[g * n + j0:g * n + j1].double().abs() for g in gs)
            worst = max(worst, bound_check(out[f * n + j0:f * n + j1], ref, len(gs) * 2.0 ** -24 * mag + BETA[dtype] * ref.abs(),
                                            f"group_sum source {f}"))
    print(f"[bound] group_sum {dtype}: worst error/bound {worst:.3g}")
    # add_indexed: dst[dst_idx[f]] += src[f]; the other groups untouched
    dst_idx = torch.tensor([2, 0, 1], dtype=torch.int32, device="cuda")
    dst0 = big.clone()
    K.add_indexed(big, out, dst_idx, nsrc, n)
    worst = 0.0
    for f, d in enumerate(dst_idx.tolist()):
        ref = dst0[d * n:(d + 1) * n].double() + out[f * n:(f + 1) * n].double()
        worst = max(worst, bound_check(big[d * n:(d + 1) * n], ref, BETA[dtype] * ref.abs(), f"add_indexed {f} -> {d}"))
    assert torch.equal(big[nsrc * n:], dst0[nsrc * n:]), "add_indexed wrote outside its destination groups"
    print(f"[bound] add_indexed {dtype}: worst error/bound {worst:.3g}")
    del big, dst0, out
    _release()


# ------------------------------------------------------------------ D. audit of a real step

def _make_audit_class():
    from p2pvg_b200._lib import CudaKernels

    class AuditKernels(CudaKernels):
        """CudaKernels whose data-movement and convolution / GEMM launches are each checked against float64 on their own
        operands right after they run (device synchronised around each call; nothing the step reads is changed)."""

        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            self.log = []          # (method, variant, worst ratio)
            self.seen = set()
            self.skip_reads = []   # grp_src of every launch with a skip addend
            self._sms = sm_count()

        def _rec(self, what, v, worst):
            self.log.append((what, v, worst))
            self.seen.add(v)
            print(f"[audit] {what} {v}: worst error/bound {worst:.3g}")

        # ---- convolutions
        def conv_gemm(self, kind, a, b, c, N, H, W, Ck, Cn, Cm=0, ldb=None, ldc=None, bias=None, addend=None, grp_src=None,
                      imgs_per_group=0, accumulate=False, stat_partial=None, eval_scale=None, eval_shift=None, act=0):
            assert kind in (3, 4, 5) and H == W and eval_scale is None, f"unexpected conv_gemm launch kind {kind} in a vgg step"
            torch.cuda.synchronize()
            c0 = c.clone() if accumulate else None
            super().conv_gemm(kind, a, b, c, N, H, W, Ck, Cn, Cm, ldb, ldc, bias, addend, grp_src, imgs_per_group, accumulate,
                              stat_partial, eval_scale, eval_shift, act)
            torch.cuda.synchronize()
            if kind == 4:
                s = conv_tiles(4, N, H, W, 0, Cn, Cm, self._sms)
                npx = N * H * W
                ref, absref = wgrad_ref64(a.view(-1)[:npx * Cm].view(N, H, W, Cm), b.view(-1)[:npx * Cn].view(N, H, W, Cn), N, H, Cm, Cn)
                if c0 is not None:
                    ref += c0.view(-1)[:Cm * 9 * Cn].view(Cm, 9 * Cn).double()
                    absref += c0.view(-1)[:Cm * 9 * Cn].view(Cm, 9 * Cn).double().abs()
                got = c.view(-1)[:Cm * 9 * Cn].view(Cm, 9 * Cn)
                w = assert_within(got, ref, absref, s.kb_per_split * 64 + 16 * s.splits, torch.float32, quiet=True,
                                  name=f"audit kind 4 N={N} {H}x{W} {Cm}x{Cn}")
                # the step's gradients cancel over these K, so the bound above is loose; the same launch on the 0 / 1 pattern of
                # its operands (x > 0) must be exact
                a01 = (a.view(-1)[:npx * Cm] > 0).bfloat16().view(N, H, W, Cm)
                b01 = (b.view(-1)[:npx * Cn] > 0).bfloat16().view(N, H, W, Cn)
                probe = torch.full((Cm, 9 * Cn), NAN, device=c.device)
                super().conv_gemm(4, a01, b01, probe, N, H, W, 0, Cn, Cm=Cm)
                assert_exact(probe, wgrad_ref64(a01, b01, N, H, Cm, Cn)[0], npx, f"audit kind 4 N={N} {H}x{W} {Cm}x{Cn} 0/1 probe")
                self._rec(f"conv_gemm kind 4 N={N} {H}x{W} {Cm}x{Cn}", variant(4, 0, Cn, False, None, c.dtype, swap=s.swap), w)
                return
            assert not accumulate
            x = a.view(-1)[:N * H * W * Ck].view(N, H, W, Ck)
            wt = b.view(-1)[:Cn * 9 * Ck].view(Cn, 9 * Ck)
            out = c.view(-1)[:N * H * W * Cn].view(N, H, W, Cn)
            add = idx = None
            if addend is not None:
                srcl = grp_src.tolist()
                ipg = max(1, imgs_per_group)
                self.skip_reads.append(srcl[:cdiv(N, ipg)])
                nimg = (max(srcl[:cdiv(N, ipg)]) + 1) * ipg
                add = addend.view(-1)[:nimg * H * W * Cn].view(nimg, H, W, Cn)
                idx = torch.tensor([srcl[n // ipg] * ipg + n % ipg for n in range(N)], device=a.device)
            nm = f"conv_gemm kind {kind} N={N} {H}x{W} {Ck}->{Cn}"
            w = check_conv3_sums(out, kind, x, wt, N, H, Ck, Cn, bias, add, idx, name="audit " + nm)
            for i0 in sorted({0, N // 2, N - 1}):   # three images element-wise
                ref, absref = conv3_ref64_elem(kind, x[i0:i0 + 1], wt, H, Ck, Cn, bias, add[idx[i0:i0 + 1]] if add is not None else None)
                w = max(w, assert_within(out[i0:i0 + 1], ref, absref, 9 * Ck, out.dtype, quiet=True, name=f"audit {nm} image {i0}"))
            if stat_partial is not None:
                tiles = cdiv(N * H * W, 128)
                w = max(w, check_stat_rows(stat_partial.view(-1)[:tiles * Cn * 2].view(tiles, Cn, 2), out, N, H, Cn, name="audit " + nm))
            self._rec(nm, variant(kind, Ck, Cn, stat_partial is not None, addend.dtype if addend is not None else None, c.dtype), w)

        def gemm(self, A, B, C, M, N, K, a_mn=False, b_mn=False, lda=None, ldb=None, ldc=None, accumulate=False, bias=None,
                 addend=None, ldd=None):
            torch.cuda.synchronize()
            lda_ = lda if lda is not None else (M if a_mn else K)
            ldb_ = ldb if ldb is not None else (N if b_mn else K)
            ldc_ = ldc if ldc is not None else N
            ldd_ = ldd if ldd is not None else N
            cv = C.as_strided((M, N), (ldc_, 1))
            c0 = cv.clone() if accumulate else None
            super().gemm(A, B, C, M, N, K, a_mn, b_mn, lda, ldb, ldc, accumulate, bias, addend, ldd)
            torch.cuda.synchronize()
            add = addend.as_strided((M, N), (ldd_, 1)) if addend is not None else None
            # the full K bounds every split-K schedule the launcher may pick
            tf32 = A.dtype == torch.float32 and self.gemm_flags == 1
            w, step = 0.0, max(1, (1 << 22) // N)
            for m0 in range(0, M, step):
                m1 = min(M, m0 + step)
                ref, absref = gemm_ref64(A, B, M, N, K, a_mn, b_mn, lda_, ldb_, bias=bias, rows=(m0, m1),
                                         addend=add[m0:m1] if add is not None else None, c0=c0[m0:m1] if c0 is not None else None)
                w = max(w, assert_within(cv[m0:m1], ref, absref, K, C.dtype, alpha=alpha_for(K, tf32=tf32), quiet=True,
                                         name=f"audit gemm {M}x{N}x{K} a_mn={a_mn} b_mn={b_mn} {A.dtype}->{C.dtype} rows {m0}"))
            if K >= 1 << 16 and C.dtype == torch.float32:
                # long reductions (the weight gradients of the 3-channel ends) cancel and the bound above is loose: the same
                # launch on the 0 / 1 pattern of the operands must be exact
                A01, B01 = (A > 0).to(A.dtype), (B > 0).to(B.dtype)
                probe = torch.full((M, N), NAN, device=C.device)
                super().gemm(A01, B01, probe, M, N, K, a_mn, b_mn, lda, ldb)
                assert_exact(probe, gemm_ref64(A01, B01, M, N, K, a_mn, b_mn, lda_, ldb_)[0], K, f"audit gemm {M}x{N}x{K} 0/1 probe")
            self._rec(f"gemm {M}x{N}x{K}", ("gemm", str(A.dtype)[6:], "tf32" if tf32 else "-"), w)

        # ---- 3-channel ends
        def im2col3(self, x, col, N, H, W, C, ld, sgn=1):
            torch.cuda.synchronize()
            super().im2col3(x, col, N, H, W, C, ld, sgn)
            torch.cuda.synchronize()
            check_im2col3(x, col, N, H, W, C, ld, sgn, "audit")
            self._rec(f"im2col3 N={N} C={C} ld={ld}", ("im2col3", "row32" if ld == 32 and C in (1, 3) else "generic", sgn), 0.0)

        def col2im3(self, col, y, N, H, W, C, ld, bias=None):
            torch.cuda.synchronize()
            super().col2im3(col, y, N, H, W, C, ld, bias)
            torch.cuda.synchronize()
            self._rec(f"col2im3 N={N}", ("col2im3",), check_col2im3(col, y, N, H, W, C, ld, bias, "audit"))

        # ---- pooling / upsampling
        def maxpool2_fwd(self, x, y, N, H, W, C):
            torch.cuda.synchronize()
            super().maxpool2_fwd(x, y, N, H, W, C)
            torch.cuda.synchronize()
            check_maxpool(x, y, None, None, N, H, W, C, "audit")
            self._rec(f"maxpool2_fwd N={N} {H}x{W}x{C}", ("maxpool2_fwd",), 0.0)

        def maxpool2_bwd(self, x, dy, dx, N, H, W, C):
            torch.cuda.synchronize()
            super().maxpool2_bwd(x, dy, dx, N, H, W, C)
            torch.cuda.synchronize()
            check_maxpool(x, None, dy, dx, N, H, W, C, "audit")
            self._rec(f"maxpool2_bwd N={N} {H}x{W}x{C}", ("maxpool2_bwd",), 0.0)

        def upsample2_fwd(self, x, y, N, H, W, C):
            torch.cuda.synchronize()
            super().upsample2_fwd(x, y, N, H, W, C)
            torch.cuda.synchronize()
            check_upsample_fwd(x, y, N, H, W, C, "audit")
            self._rec(f"upsample2_fwd N={N} {H}x{W}x{C}", ("upsample2_fwd",), 0.0)

        def upsample2_bwd(self, dy, dx, N, H, W, C):
            torch.cuda.synchronize()
            super().upsample2_bwd(dy, dx, N, H, W, C)
            torch.cuda.synchronize()
            self._rec(f"upsample2_bwd N={N} {H}x{W}x{C}", ("upsample2_bwd",), check_upsample_bwd(dy, dx, N, H, W, C, "audit"))

        # ---- skip-connection index kernels
        def gather_add(self, dst, src, grp_src, G, n):
            torch.cuda.synchronize()
            d0 = dst.view(-1)[:G * n].clone()
            super().gather_add(dst, src, grp_src, G, n)
            torch.cuda.synchronize()
            srcl = grp_src.tolist()
            ref = d0.double().view(G, n) + src.view(-1).double().view(-1, n)[srcl[:G]]
            rel = 2.0 ** -7 if dst.dtype == torch.bfloat16 else 2.0 ** -23
            self._rec(f"gather_add G={G}", ("gather_add",), bound_check(dst.view(-1)[:G * n].view(G, n), ref, rel * ref.abs(), "audit gather_add"))

        def group_sum(self, inp, out, grp_src, G, F_, n):
            torch.cuda.synchronize()
            super().group_sum(inp, out, grp_src, G, F_, n)
            torch.cuda.synchronize()
            srcl = grp_src.tolist()[:G]
            iv = inp.view(-1)[:G * n].view(G, n)
            w = 0.0
            for f in range(F_):
                gs = [g for g in range(G) if srcl[g] == f]
                ref = iv[gs].double().sum(0) if gs else torch.zeros(n, dtype=torch.float64, device=inp.device)
                mag = iv[gs].double().abs().sum(0) if gs else torch.zeros_like(ref)
                w = max(w, bound_check(out.view(-1)[f * n:(f + 1) * n], ref, len(gs) * 2.0 ** -24 * mag + BETA[out.dtype] * ref.abs(),
                                        "audit group_sum"))
            self._rec(f"group_sum G={G} F={F_}", ("group_sum",), w)

        def add_indexed(self, dst, src, dst_idx, F_, n):
            torch.cuda.synchronize()
            di = dst_idx.tolist()[:F_]
            d0 = [dst.view(-1)[d * n:(d + 1) * n].clone() for d in di]
            super().add_indexed(dst, src, dst_idx, F_, n)
            torch.cuda.synchronize()
            w = 0.0
            for f, d in enumerate(di):
                ref = d0[f].double() + src.view(-1)[f * n:(f + 1) * n].double()
                w = max(w, bound_check(dst.view(-1)[d * n:(d + 1) * n], ref, BETA[dst.dtype] * ref.abs(), "audit add_indexed"))
            self._rec(f"add_indexed F={F_}", ("add_indexed",), w)

        def bn_fwd_finalize_tiles(self, partial, parts_per_group, ldp, fold, G, R, C, gamma, beta, mean, invstd, var_unb, scale,
                                  shift, eps=1e-5):
            torch.cuda.synchronize()
            super().bn_fwd_finalize_tiles(partial, parts_per_group, ldp, fold, G, R, C, gamma, beta, mean, invstd, var_unb, scale,
                                          shift, eps)
            torch.cuda.synchronize()
            assert fold == 1 and ldp == C
            p = partial.view(-1)[:G * parts_per_group * C * 2].view(G, parts_per_group, C, 2).double()
            s1, s2, m1 = p[..., 0].sum(1), p[..., 1].sum(1), p[..., 0].abs().sum(1)
            # the kernel's own operands are exact here: only the float64 combine order and the fp32 outputs differ
            w = 0.0
            for got, (ref, _), nm in zip((mean, invstd, var_unb, scale, shift), finalize_ref(s1, s2, m1, R, gamma, beta, eps, 0.0),
                                         ("mean", "invstd", "var_unbiased", "scale", "shift")):
                g = got.view(-1)[:G * C].view(G, C)
                mag = ref.abs() if nm != "shift" else beta.double().abs() + (s1 / R * scale.view(-1)[:G * C].view(G, C).double()).abs()
                if nm == "mean":
                    mag = mag + 2.0 ** -30 * m1 / R
                w = max(w, bound_check(g, ref, 2.0 ** -20 * mag + 1e-30, f"audit finalize {nm}"))
            self._rec(f"bn_fwd_finalize_tiles G={G} C={C}", ("bn_fwd_finalize_tiles",), w)

    return AuditKernels


def vgg_step(kernels, optkw, T, B, np_seed, W0=64, use_graph=False):
    """One bf16 vgg step (vgg_64 or vgg_128 by W0) from the seeded initial state: (plan, losses, gradients, engine).
    use_graph: the step replayed from a captured CUDA graph, the engine restored in place to its initial state before the
    replay."""
    from p2pvg_b200.engine_vgg import TrainEngineVGG
    cfg = dict(g_dim=128, z_dim=10, rnn_size=256, channels=3, image_width=W0, backbone="vgg", predictor_rnn_layers=2,
               posterior_rnn_layers=1, prior_rnn_layers=1)
    state = O.build_state(cfg, seed=1)
    opt = O.default_opt(**optkw)
    opt["batch_size"] = B
    eng = TrainEngineVGG(state, cfg, opt, kernels, act_dtype=torch.bfloat16)
    x = torch.rand(T, B, 3, W0, W0, generator=torch.Generator().manual_seed(5)).cuda()
    probs = np.random.RandomState(np_seed).uniform(0, 1, T - 1)
    plan = StepPlan(T, probs, opt)
    eps = O.draw_eps(plan.S, B, 10, seed=11).cuda()
    if use_graph:
        from tests.test_measured_gpu import restore, snapshot
        snap = snapshot(eng)
        for _ in range(2):   # eager warm-up, then capture
            eng.step(x, probs=probs, eps=eps, use_graph=True)
        restore(eng, snap)
        del snap
        losses = eng.step(x, probs=probs, eps=eps, use_graph=True)
        assert any(v != "warm" for v in eng._graphs.values()), "the step was not graph-replayed"
    else:
        losses = eng.step(x, probs=probs, eps=eps)
    torch.cuda.synchronize()
    grads = {m: {k: v.detach().clone() for k, v in eng.arena[m].g.items()} for m in eng.arena}
    return plan, np.asarray(losses), grads, eng


def assert_equal_steps(a, b, what):
    """(losses, gradients) of two steps are equal bit for bit."""
    assert np.array_equal(a[0], b[0]), f"{what}: losses {a[0]} vs {b[0]}"
    for m in a[1]:
        for k in a[1][m]:
            assert torch.equal(a[1][m][k], b[1][m][k]), f"{what}: grad {m}.{k} differs"


def _skip_seed(T):
    """The first probability seed whose skip_prob 0.5 / n_past 2 / last-frame-skip plan reads at least three skip sources."""
    opt = O.default_opt(skip_prob=0.5, n_past=2, last_frame_skip=True)
    for seed in range(100):
        p = StepPlan(T, np.random.RandomState(seed).uniform(0, 1, T - 1), opt)
        if len(set(p.skip_src)) >= 3:
            return seed
    raise AssertionError("no seed gives three skip sources")


AUDIT_CASES = [("bench_options", BENCH_OPT, None), ("skip_lfs", dict(skip_prob=0.5, n_past=2, last_frame_skip=True), "search")]


@pytest.mark.parametrize("case", AUDIT_CASES, ids=[c[0] for c in AUDIT_CASES])
def test_audit_vgg_step(K, case):
    """One eager bf16 vgg_64 step at T = 30, B = 32 with every launch checked as it runs."""
    name, optkw, seed = case
    audit_step(name, optkw, 30, 32, seed, W0=64)


def audit_step(name, optkw, T, B, seed, W0):
    """One eager bf16 vgg step with every launch checked as it runs; every path of the launch list must occur, every skip
    addend must be read through the plan's skip sources, and the audited step must equal (torch.equal) the same step on plain
    CudaKernels.  seed "search": _skip_seed.  Returns the plain step's (losses, gradients)."""
    from p2pvg_b200._lib import CudaKernels
    seed = _skip_seed(T) if seed == "search" else 0
    plan, losses, grads, eng = vgg_step(CudaKernels("cuda"), optkw, T, B, seed, W0)
    del eng
    _release()
    if name == "skip_lfs":
        assert len(set(plan.skip_src)) >= 3
    audit = _make_audit_class()("cuda")
    plan_a, losses_a, grads_a, eng = vgg_step(audit, optkw, T, B, seed, W0)
    log, seen, skip_reads = eng.K.log, eng.K.seen, eng.K.skip_reads
    del eng
    _release()
    # coverage: every variant of the derived launch list (and every wrapped data-movement kernel) occurred
    want = set()
    for L in forward_launches(T, B, plan.S, plan.nskip, W0) + backward_launches(T, B, plan.S, plan.nskip, W0, plan.has_cpc):
        if L["kind"] == 4:
            want.add(variant(4, 0, L["Cn"], False, None, torch.float32, swap=conv_tiles(4, L["N"], L["H"], L["H"], 0, L["Cn"], L["Cm"], sm_count()).swap))
        else:
            want.add(variant(L["kind"], L["Ck"], L["Cn"], L["stat"] is not None, torch.bfloat16 if L["addend"] else None, torch.bfloat16))
    want |= {("maxpool2_fwd",), ("maxpool2_bwd",), ("upsample2_fwd",), ("upsample2_bwd",), ("group_sum",), ("add_indexed",),
             ("bn_fwd_finalize_tiles",), ("col2im3",), ("im2col3", "row32", 1)}
    for v in [("k3", "bres", "-", "add_bf16", "rowcoop"), ("k3", "bn128", "stat", "add_bf16", "perrow"), ("k4", "swap"), ("k4", "noswap"),
              ("k3", "bn128", "-", "-", "rowcoop"), ("k5", "bres", "-", "-", "rowcoop")]:
        assert v in want, f"the derived launch list lost {v}"
    missing = want - seen
    assert not missing, f"launch variants that did not occur in the step: {sorted(missing)}"
    assert any(v[0] == "gemm" for v in seen)
    # every decoder stage entry reads, for decoder call s, the skip frame the reference's schedule names (models/p2p_model.py)
    assert len(skip_reads) == sum(1 for L in forward_launches(T, B, plan.S, plan.nskip, W0) if L["addend"])
    for r in skip_reads:
        assert r == plan.skip_src, f"skip addend read through {r}, the schedule says {plan.skip_src}"
    print(f"[audit] {name} {W0}x{W0}: {len(log)} launches checked, worst error/bound {max(w for _, _, w in log):.3g}")
    # the audit does not perturb the step
    assert_equal_steps((losses, grads), (losses_a, grads_a), f"{name}: the audited step")
    return losses, grads
