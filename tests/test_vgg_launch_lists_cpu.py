"""The vgg launch lists tests/vgg_ref.py derives from the engine's layer tables, pinned as literals at the two benchmarked vgg
shapes: C3 (vgg_64, 64x64 frames, T = 30, B = 128) and vgg_128 (128x128 frames, T = 30, B = 32), both with the bench options
(S = 29, one skip frame, a CPC decode).  The GPU launch tests parametrise over these lists and compare them with a recorded
step; this module fails on the CPU when the derivation or the engine's tables or fusion rules change."""
import numpy as np
import pytest
import torch

from oracle import p2p_oracle as O
from p2pvg_b200.engine import StepPlan
from p2pvg_b200.engine_vgg import VGG_DEC, VGG_DEC_128, VGG_ENC, VGG_ENC_128
from tests.vgg_ref import backward_launches, forward_launches, launch_key, vgg_tables

T = 30
SHAPES = {"C3": dict(W0=64, B=128), "vgg128": dict(W0=128, B=32)}


def bench_plan():
    p = StepPlan(T, np.zeros(T - 1), O.default_opt(skip_prob=0.0, n_past=1, last_frame_skip=False))
    assert (p.S, p.nskip, p.has_cpc) == (29, 1, True)
    return p


def lists(name):
    c, p = SHAPES[name], bench_plan()
    return (forward_launches(T, c["B"], p.S, p.nskip, c["W0"]),
            backward_launches(T, c["B"], p.S, p.nskip, c["W0"], has_cpc=p.has_cpc))


def test_tables_follow_the_frame_size():
    assert vgg_tables(64) == (VGG_ENC, VGG_DEC)
    assert vgg_tables(128) == (VGG_ENC_128, VGG_DEC_128)
    with pytest.raises(ValueError):
        vgg_tables(32)


# (map size, fused statistics) of the encoder's implicit layers
ENCODER = {
    "C3": [(64, False), (32, False), (32, False), (16, True), (16, True), (16, True), (8, True), (8, True), (8, True)],
    "vgg128": [(128, False), (64, False), (64, False), (32, True), (32, True), (32, True), (16, True), (16, True), (16, True),
               (8, True), (8, True), (8, True)],
}
# decoder stage entries (upsampled half): map size, fused statistics, images per skip-addend group
ENTRIES = {
    "C3": [(8, True, 128), (16, True, 128), (32, False, 128), (64, False, 128)],
    "vgg128": [(8, True, 32), (16, True, 32), (32, True, 32), (64, False, 32), (128, False, 32)],
}


@pytest.mark.parametrize("name", list(SHAPES))
def test_forward_tables(name):
    fwd, _ = lists(name)
    B = SHAPES[name]["B"]
    assert [(L["H"], L["stat"] is not None) for L in fwd if L["name"].startswith("enc")] == ENCODER[name]
    assert [(L["H"], L["stat"] is not None, L["ipg"]) for L in fwd if L["name"].endswith(".D")] == ENTRIES[name]
    assert all(L["N"] == T * B for L in fwd if not L["name"].endswith(".S"))
    assert all(L["N"] == B and L["stat"] is None and not L["addend"] for L in fwd if L["name"].endswith(".S"))
    assert all(L["addend"] and not L["bias"] for L in fwd if L["name"].endswith(".D"))


# every backward launch: (name, kind, N) in the order the step enqueues them
BACKWARD = {
    "C3": [("dec3.0.D dgrad", 5, 3712), ("dec3.0.D wgrad", 4, 3712), ("dec3.0.S dgrad", 5, 128), ("dec3.0.S wgrad", 4, 128),
           ("dec2.1 dgrad", 5, 3712), ("dec2.1 wgrad", 4, 3712),
           ("dec2.0.D dgrad", 5, 3712), ("dec2.0.D wgrad", 4, 3712), ("dec2.0.S dgrad", 5, 128), ("dec2.0.S wgrad", 4, 128),
           ("dec1.2 dgrad", 5, 3712), ("dec1.2 wgrad", 4, 3712), ("dec1.1 dgrad", 5, 3712), ("dec1.1 wgrad", 4, 3712),
           ("dec1.0.D dgrad", 5, 3712), ("dec1.0.D wgrad", 4, 3712), ("dec1.0.S dgrad", 5, 128), ("dec1.0.S wgrad", 4, 128),
           ("dec0.2 dgrad", 5, 3712), ("dec0.2 wgrad", 4, 3712), ("dec0.1 dgrad", 5, 3712), ("dec0.1 wgrad", 4, 3712),
           ("dec0.0.D dgrad", 5, 3712), ("dec0.0.D wgrad", 4, 3712), ("dec0.0.S dgrad", 5, 128), ("dec0.0.S wgrad", 4, 128),
           ("cpc dec3.0.D dgrad", 5, 128), ("cpc dec2.1 dgrad", 5, 128), ("cpc dec2.0.D dgrad", 5, 128),
           ("cpc dec1.2 dgrad", 5, 128), ("cpc dec1.1 dgrad", 5, 128), ("cpc dec1.0.D dgrad", 5, 128),
           ("cpc dec0.2 dgrad", 5, 128), ("cpc dec0.1 dgrad", 5, 128), ("cpc dec0.0.D dgrad", 5, 128),
           ("enc3.2 wgrad", 4, 3840), ("enc3.2 dgrad", 5, 3840), ("enc3.1 wgrad", 4, 3840), ("enc3.1 dgrad", 5, 3840),
           ("enc3.0 wgrad", 4, 3840), ("enc3.0 dgrad", 5, 3840), ("enc2.2 wgrad", 4, 3840), ("enc2.2 dgrad", 5, 3840),
           ("enc2.1 wgrad", 4, 3840), ("enc2.1 dgrad", 5, 3840), ("enc2.0 wgrad", 4, 3840), ("enc2.0 dgrad", 5, 3840),
           ("enc1.1 wgrad", 4, 3840), ("enc1.1 dgrad", 5, 3840), ("enc1.0 wgrad", 4, 3840), ("enc1.0 dgrad", 5, 3840),
           ("enc0.1 wgrad", 4, 3840), ("enc0.1 dgrad", 5, 3840)],
    "vgg128": [("dec4.0.D dgrad", 5, 928), ("dec4.0.D wgrad", 4, 928), ("dec4.0.S dgrad", 5, 32), ("dec4.0.S wgrad", 4, 32),
               ("dec3.1 dgrad", 5, 928), ("dec3.1 wgrad", 4, 928),
               ("dec3.0.D dgrad", 5, 928), ("dec3.0.D wgrad", 4, 928), ("dec3.0.S dgrad", 5, 32), ("dec3.0.S wgrad", 4, 32),
               ("dec2.2 dgrad", 5, 928), ("dec2.2 wgrad", 4, 928), ("dec2.1 dgrad", 5, 928), ("dec2.1 wgrad", 4, 928),
               ("dec2.0.D dgrad", 5, 928), ("dec2.0.D wgrad", 4, 928), ("dec2.0.S dgrad", 5, 32), ("dec2.0.S wgrad", 4, 32),
               ("dec1.2 dgrad", 5, 928), ("dec1.2 wgrad", 4, 928), ("dec1.1 dgrad", 5, 928), ("dec1.1 wgrad", 4, 928),
               ("dec1.0.D dgrad", 5, 928), ("dec1.0.D wgrad", 4, 928), ("dec1.0.S dgrad", 5, 32), ("dec1.0.S wgrad", 4, 32),
               ("dec0.2 dgrad", 5, 928), ("dec0.2 wgrad", 4, 928), ("dec0.1 dgrad", 5, 928), ("dec0.1 wgrad", 4, 928),
               ("dec0.0.D dgrad", 5, 928), ("dec0.0.D wgrad", 4, 928), ("dec0.0.S dgrad", 5, 32), ("dec0.0.S wgrad", 4, 32),
               ("cpc dec4.0.D dgrad", 5, 32), ("cpc dec3.1 dgrad", 5, 32), ("cpc dec3.0.D dgrad", 5, 32),
               ("cpc dec2.2 dgrad", 5, 32), ("cpc dec2.1 dgrad", 5, 32), ("cpc dec2.0.D dgrad", 5, 32),
               ("cpc dec1.2 dgrad", 5, 32), ("cpc dec1.1 dgrad", 5, 32), ("cpc dec1.0.D dgrad", 5, 32),
               ("cpc dec0.2 dgrad", 5, 32), ("cpc dec0.1 dgrad", 5, 32), ("cpc dec0.0.D dgrad", 5, 32),
               ("enc4.2 wgrad", 4, 960), ("enc4.2 dgrad", 5, 960), ("enc4.1 wgrad", 4, 960), ("enc4.1 dgrad", 5, 960),
               ("enc4.0 wgrad", 4, 960), ("enc4.0 dgrad", 5, 960), ("enc3.2 wgrad", 4, 960), ("enc3.2 dgrad", 5, 960),
               ("enc3.1 wgrad", 4, 960), ("enc3.1 dgrad", 5, 960), ("enc3.0 wgrad", 4, 960), ("enc3.0 dgrad", 5, 960),
               ("enc2.2 wgrad", 4, 960), ("enc2.2 dgrad", 5, 960), ("enc2.1 wgrad", 4, 960), ("enc2.1 dgrad", 5, 960),
               ("enc2.0 wgrad", 4, 960), ("enc2.0 dgrad", 5, 960), ("enc1.1 wgrad", 4, 960), ("enc1.1 dgrad", 5, 960),
               ("enc1.0 wgrad", 4, 960), ("enc1.0 dgrad", 5, 960), ("enc0.1 wgrad", 4, 960), ("enc0.1 dgrad", 5, 960)],
}


@pytest.mark.parametrize("name", list(SHAPES))
def test_backward_row_counts(name):
    """decoder_backward(0, S) runs over S B images with weight gradients, its skip halves over nskip B, the CPC decode over B
    images with data gradients only; the encoder over T B frames, with no data gradient for the 3-channel first layer."""
    _, bwd = lists(name)
    assert [(L["name"], L["kind"], L["N"]) for L in bwd] == BACKWARD[name]
    for L in bwd:
        if L["kind"] == 5:
            assert (L["bias"], L["addend"], L["ipg"], L["stat"]) == (False, False, 0, None)


@pytest.mark.parametrize("name", list(SHAPES))
def test_backward_mirrors_the_forward_channels(name):
    """Every data gradient swaps its forward layer's channel counts, every weight gradient is [cout, 9 cin]; the CPC list is
    the reconstruction list's data gradients without the skip halves."""
    fwd, bwd = lists(name)
    by = {L["name"]: L for L in fwd}
    for L in bwd:
        f = by[L["name"].split()[-2]]
        assert L["H"] == f["H"]
        if L["kind"] == 5:
            assert (L["Ck"], L["Cn"]) == (f["Cn"], f["Ck"])
        else:
            assert (L["Cm"], L["Cn"]) == (f["Cn"], f["Ck"])
    rec = [L["name"] for L in bwd if L["kind"] == 5 and L["name"].startswith("dec") and not L["name"].endswith(".S dgrad")]
    assert [L["name"][4:] for L in bwd if L["name"].startswith("cpc ")] == rec


def test_no_cpc_no_cpc_launches():
    p = bench_plan()
    bwd = backward_launches(T, 32, p.S, p.nskip, 128, has_cpc=False)
    assert not any(L["name"].startswith("cpc") for L in bwd)
    assert len(bwd) == len(BACKWARD["vgg128"]) - 12


def test_launch_keys_are_what_conv_gemm_receives():
    fwd, bwd = lists("vgg128")
    keys = {L["name"]: launch_key(L) for L in fwd + bwd}
    assert keys["dec4.0.D"] == (3, 960, 128, 64, 64, 0, False, torch.bfloat16, 32, False)
    assert keys["dec2.0.D"] == (3, 960, 32, 256, 256, 0, False, torch.bfloat16, 32, True)
    assert keys["enc0.1"] == (3, 960, 128, 64, 64, 0, True, None, 0, False)
    assert keys["enc4.0 wgrad"] == (4, 960, 8, 0, 512, 512, False, None, 0, False)
    assert keys["cpc dec0.0.D dgrad"] == (5, 32, 8, 512, 512, 0, False, None, 0, False)
