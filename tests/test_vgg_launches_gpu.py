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

import numpy as np
import pytest
import torch

from oracle import p2p_oracle as O
from p2pvg_b200.engine import StepPlan
from tests.launch_audit import K, memory_per_test, sms  # noqa: F401  (fixtures)
from tests.launch_audit import BENCH_OPT, NAN, randn
from tests.tc_schedule import assert_within, conv_tiles, fit
from tests.vgg_ref import (AUDIT_CASES, audit_vgg_step, backward_launches, check_stat_rows, conv3_ref64_elem, distinct_convs,
                           encoder_first, forward_launches, run_conv, run_end_gemms, run_im2col3_col2im3, run_maxpool,
                           run_skip_index, run_upsample, run_wgrad, variant, wgrad_classes)

pytestmark = pytest.mark.gpu

C3 = dict(T=30, B=128, nc=3)


def c3_plan():
    probs = np.zeros(C3["T"] - 1)
    opt = O.default_opt(**BENCH_OPT)
    return StepPlan(C3["T"], probs, opt)


# ------------------------------------------------------------------ A. every implicit-GEMM launch of the C3 step

def _c3_conv_launches():
    p = c3_plan()
    T, B = C3["T"], C3["B"]
    return distinct_convs(forward_launches(T, B, p.S, p.nskip)
                          + encoder_first(backward_launches(T, B, p.S, p.nskip, has_cpc=p.has_cpc)))


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


_p = c3_plan()
C3_WGRAD = wgrad_classes(backward_launches(C3["T"], C3["B"], _p.S, _p.nskip, has_cpc=_p.has_cpc))


@pytest.mark.parametrize("L", C3_WGRAD, ids=[f"{L['H']}x{L['H']}_{L['Cm']}x{L['Cn']}" for L in C3_WGRAD])
def test_c3_weight_gradient(K, sms, L):
    """One kind-4 launch per (map size, swapped roles) class at C3 size, against a full float64 reduction over all
    N * H * W pixels (K = 15.7M at 64x64)."""
    run_wgrad(K, sms, L)


def test_c3_end_gemms(K):
    """The explicit GEMMs of the 3-channel ends at C3 size."""
    run_end_gemms(K, C3["T"] * C3["B"] * 64 * 64)


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


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "f32"])
def test_maxpool_c3(K, dtype):
    """maxpool2_fwd / maxpool2_bwd on the 64x64x64 encoder map of C3 (N = 3840: 10^9 input elements)."""
    run_maxpool(K, C3_N, 64, 64, dtype, "C3")


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "f32"])
def test_upsample_c3(K, dtype):
    """upsample2_fwd / upsample2_bwd at the 64x64 decoder stage entry of C3 (32x32x64 -> 64x64x64 at N = 3840: 10^9 upsampled
    elements)."""
    run_upsample(K, C3_N, 32, 64, dtype, "C3")


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "f32"])
def test_im2col3_col2im3_c3(K, dtype):
    """The 3-channel ends at C3 size (N = 3840 frames of 64x64x3)."""
    run_im2col3_col2im3(K, C3_N, 64, dtype, "C3")


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "f32"])
def test_skip_index_kernels_c3(K, dtype):
    """gather_add, group_sum and add_indexed at the engine's C3 sizes at 64x64x64 (groups of B = 128 images, G = 30 calls):
    n = 33.5M elements per group, 10^9 in all; three distinct skip sources."""
    run_skip_index(K, C3["T"], C3["B"], 64, 64, dtype, gather=True)


# ------------------------------------------------------------------ D. audit of a real step

@pytest.mark.parametrize("case", AUDIT_CASES, ids=[c[0] for c in AUDIT_CASES])
def test_audit_vgg_step(case):
    """One eager bf16 vgg_64 step at T = 30, B = 32 with every launch checked as it runs."""
    name, optkw = case
    audit_vgg_step(name, optkw, 30, 32, W0=64)
