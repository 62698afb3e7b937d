"""The fp32 dcgan / vgg launch lists (tests/dcgan_ref.py, tests/vgg_ref.py, precision "fp32") against a step of the engines
on the torch emulation of the kernels (tests/emu_backend.py), and the float64 checkers the fp32 launch tests use, each shown
to reject an fp32 emulation with one deliberate error.

The engines take the same explicit fp32 branches on the emulation as on the GPU (TrainEngine.implicit, bd, fuse_stats,
fuse_last, bn_skip_sums, bn_wgrad_c1 and concurrent are all off in fp32), so a change to those branches that the derivation
does not follow fails here on a machine without a GPU.  Only the backbone methods are compared (encode, decode, losses_fwd,
decoder_backward, encoder_backward): the emulation has no lstm_scan_fwd, so its recurrent phase differs from the CUDA one.
"""
import inspect

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import p2p_oracle as O
from p2pvg_b200.engine import StepPlan, TrainEngine
from p2pvg_b200.engine_vgg import TrainEngineVGG
from tests.dcgan_ref import check_col2im, check_im2col, step_launches
from tests.emu_backend import EmuKernels
from tests.emu_vgg import EmuKernelsVGG
from tests.launch_audit import (BENCH_OPT, FP32_OPS, SKIP_OPT, check_group_sum, check_simt_gemm, fp32_call_key, kernel_for,
                                simt_split, skip_seed, watch_backbone)
from tests.vgg_ref import backward_launches, check_gather_add, forward_launches

def _recording(cls):
    """cls with every FP32_OPS entry point it has logging fp32_call_key while `on` is set."""
    def wrap(op):
        f = getattr(cls, op)
        sig = inspect.signature(f)

        def method(self, *a, **kw):
            if self.on:
                x = sig.bind(self, *a, **kw)
                x.apply_defaults()
                self.calls.append(fp32_call_key(op, x.arguments))
            return f(self, *a, **kw)
        return method
    attrs = {op: wrap(op) for op in FP32_OPS if hasattr(cls, op)}
    attrs.update(on=False)
    return type(f"Recording{cls.__name__}", (cls,), attrs)


def _cfg(backbone, nc, W0):
    c = dict(g_dim=128, z_dim=10, rnn_size=32, channels=nc, image_width=W0, predictor_rnn_layers=2, posterior_rnn_layers=1,
             prior_rnn_layers=1)
    if backbone == "vgg":
        c["backbone"] = "vgg"
    return c


def _recorded_emu_step(backbone, nc, W0, T, B, optkw):
    torch.set_num_threads(8)
    cfg = _cfg(backbone, nc, W0)
    opt = O.default_opt(**optkw)
    opt["batch_size"] = B
    np_seed = skip_seed(T) if optkw.get("skip_prob") else 0
    probs = np.random.RandomState(np_seed).uniform(0, 1, T - 1)
    plan = StepPlan(T, probs, opt)
    K = _recording(EmuKernelsVGG if backbone == "vgg" else EmuKernels)("cpu")
    K.calls = []
    eng = (TrainEngineVGG if backbone == "vgg" else TrainEngine)(O.build_state(cfg, seed=1), cfg, opt, K, act_dtype=torch.float32)
    assert not (eng.implicit or eng.bd or eng.fuse_stats or eng.fuse_last or eng.bn_skip_sums or eng.bn_wgrad_c1 or eng.concurrent)
    watch_backbone(eng)
    x = torch.rand(T, B, nc, W0, W0, generator=torch.Generator().manual_seed(5))
    losses = eng.step(x, probs=probs, eps=O.draw_eps(plan.S, B, cfg["z_dim"], seed=11))
    assert np.all(np.isfinite(np.asarray(losses)))
    return plan, eng.K.calls


CASES = [("dcgan64", "dcgan", 1, 64, 6, 2, BENCH_OPT), ("dcgan64_skip", "dcgan", 1, 64, 8, 2, SKIP_OPT),
         ("dcgan128_rgb", "dcgan", 3, 128, 4, 1, BENCH_OPT), ("vgg64", "vgg", 3, 64, 5, 2, BENCH_OPT),
         ("vgg64_skip", "vgg", 3, 64, 8, 1, SKIP_OPT), ("vgg128", "vgg", 3, 128, 4, 1, BENCH_OPT)]


def derived(backbone, nc, W0, T, B, plan):
    if backbone == "vgg":
        return (forward_launches(T, B, plan.S, plan.nskip, W0, "fp32", nc)
                + backward_launches(T, B, plan.S, plan.nskip, W0, plan.has_cpc, "fp32", nc))
    return step_launches(T, B, plan.S, plan.nskip, nc, W0, plan.has_cpc, "fp32")


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_fp32_list_matches_an_emulated_step(case):
    """The derived fp32 list equals, call for call and in order, what the backbone methods of an fp32 step launch on the
    emulation; the skip cases read three skip sources."""
    name, backbone, nc, W0, T, B, optkw = case
    plan, got = _recorded_emu_step(backbone, nc, W0, T, B, optkw)
    if optkw is SKIP_OPT:
        assert len(set(plan.skip_src)) >= 3 and plan.nskip >= 3
    L = derived(backbone, nc, W0, T, B, plan)
    want = [e["key"] for e in L]
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"{name}: launch {i} is {g}, the derived list says {w} ({L[i]['name']})"
    assert len(got) == len(want), f"{name}: {len(got)} launches recorded, {len(want)} derived"


@pytest.mark.parametrize("backbone,nc,W0", [("dcgan", 1, 64), ("dcgan", 3, 128), ("vgg", 3, 64), ("vgg", 3, 128)])
def test_fp32_lists_have_no_fused_or_implicit_entries(backbone, nc, W0):
    """The fp32 step launches no implicit GEMM, no fused BatchNorm pass and no fused last layer; its weight gradients are
    GEMMs over every pixel, split over K where the output is small."""
    p = StepPlan(30, np.zeros(29), O.default_opt(**BENCH_OPT))
    L = derived(backbone, nc, W0, 30, 4, p)
    ops = {e["op"] for e in L}
    assert not ops & {"conv_gemm", "bn_bwd_group_sum", "bn_bwd_wgrad_c1", "convt_c1_loss", "bn_fwd_finalize_tiles"}, ops
    assert ops <= set(FP32_OPS)
    assert {"gemm", "group_sum", "add_indexed", "bn_fwd_stats", "bn_act", "bn_bwd", "bn_param_grad", "sigmoid_mse", "colsum"} <= ops
    assert ({"im2col", "col2im"} if backbone == "dcgan" else {"im2col3", "col2im3", "gather_add"}) <= ops
    wg = [e for e in L if e["op"] == "gemm" and e["a_mn"]]
    assert any(simt_split(e["M"], e["N"], e["K"])[0] > 1 for e in wg)


def test_fp32_split_schedules_at_the_bench_shapes():
    """The split-K schedules the issue's shapes take: dcgan_64 enc0 64 x 16 x 7.86M (the cap of 296 CTAs), enc1 / dec2
    128 x 1024 x 1.97M (10 splits), vgg_64 64 x 576 x 15.7M (33 splits); all K < 2^24, so 0 / 1 operands stay exact."""
    assert simt_split(64, 16, 7680 * 32 * 32) == (296, 26576)
    assert simt_split(128, 1024, 7680 * 16 * 16)[0] == 10
    assert simt_split(64, 576, 3840 * 64 * 64)[0] == 33
    assert max(7680 * 32 * 32, 3840 * 64 * 64, 960 * 128 * 128) < 1 << 24


# ------------------------------------------------------------------ the float64 checkers reject one deliberate error each

def _gemm32_emulation(A, B, M, N, K, kern, bias=None, drop_last_split=False, bias_twice=False):
    """gemm_simt on fp32 operands (A [M, K], B [N, K], K-major), split-K as `kern` says: fp32 partials per split, summed in
    ascending split order in fp32, then the bias."""
    splits, kps = (1, K) if kern == "simt" else kern[1:]
    parts = [A[:, z * kps:(z + 1) * kps] @ B[:, z * kps:(z + 1) * kps].t() for z in range(splits)]
    if drop_last_split:
        parts = parts[:-1]
    acc = parts[0].clone()
    for p in parts[1:]:
        acc += p
    if bias is not None:
        acc += bias
        if bias_twice:
            acc += bias
    return acc


def _rejects(check, *a, **kw):
    with pytest.raises(AssertionError):
        check(*a, **kw)


def test_simt_gemm_checker_rejects_a_lost_split_and_a_doubled_bias():
    g = torch.Generator().manual_seed(1)
    M, N, K = 16, 24, 8192
    kern = kernel_for(M, N, K, False, False, K, K, 0, 0, False)
    assert kern[0] == "simt-splitK" and kern[1] == 32
    A, B = torch.rand(M, K, generator=g), torch.rand(N, K, generator=g) + 0.25
    bias = torch.randn(N, generator=g)
    ok = _gemm32_emulation(A, B, M, N, K, kern, bias)
    check_simt_gemm(ok, A, B, M, N, K, False, False, K, K, N, kern, bias=bias, name="emulated split-K")
    _rejects(check_simt_gemm, _gemm32_emulation(A, B, M, N, K, kern, bias, drop_last_split=True), A, B, M, N, K, False, False,
             K, K, N, kern, bias=bias, name="split-K without its last split")
    _rejects(check_simt_gemm, _gemm32_emulation(A, B, M, N, K, kern, bias, bias_twice=True), A, B, M, N, K, False, False, K, K, N,
             kern, bias=bias, name="bias added twice")


def test_im2col_checker_rejects_padding_on_the_wrong_side():
    N, H, C = 3, 8, 4
    x = torch.randn(N, H, H, C, generator=torch.Generator().manual_seed(2))
    col = torch.empty(N * (H // 2) ** 2 * 16 * C)
    EmuKernels().im2col(x, col, N, H, H, C)
    check_im2col(x, col, N, H, C, "emulated im2col")
    Ho = H // 2
    xp = F.pad(x, (0, 0, 0, 2, 0, 2))   # both pad rows / columns after the map: tap kh reads 2 oy + kh
    bad = torch.stack([xp[:, kh:kh + 2 * Ho:2, kw:kw + 2 * Ho:2] for kh in range(4) for kw in range(4)], 3).reshape(-1)
    _rejects(check_im2col, x, bad, N, H, C, "im2col padded on the wrong side")


def test_col2im_checker_rejects_the_wrong_skip_image():
    """Three groups of two images; groups 0 and 2 read source 2, group 1 reads source 0, source 1 is read by no group."""
    g = torch.Generator().manual_seed(3)
    G, ipg, Hi, C = 3, 2, 4, 8
    N = G * ipg
    col = torch.randn(N * Hi * Hi * 16 * C, generator=g)
    col2 = torch.randn(3 * ipg * Hi * Hi * 16 * C, generator=g)
    bias = torch.randn(C, generator=g)
    grp = torch.tensor([2, 0, 2], dtype=torch.int32)
    y = torch.empty(N * 4 * Hi * Hi * C)
    EmuKernels().col2im(col, y, N, Hi, Hi, C, bias=bias, col2=col2, grp_src=grp, imgs_per_group=ipg)
    check_col2im(y, col, N, Hi, C, bias, col2, grp, ipg, "emulated col2im")
    bad = torch.empty_like(y)   # image n reads skip image n, not grp_src[n // ipg] * ipg + n % ipg
    EmuKernels().col2im(col, bad, N, Hi, Hi, C, bias=bias, col2=col2, grp_src=torch.arange(G, dtype=torch.int32), imgs_per_group=ipg)
    _rejects(check_col2im, bad, col, N, Hi, C, bias, col2, grp, ipg, "col2im reading skip image n")
    EmuKernels().col2im(col, bad, N, Hi, Hi, C, bias=bias, col2=col2, grp_src=grp, imgs_per_group=ipg)
    bad.view(-1, C).add_(bias)   # the bias added twice
    _rejects(check_col2im, bad, col, N, Hi, C, bias, col2, grp, ipg, "col2im with the bias added twice")


def test_gather_add_and_group_sum_checkers_reject_the_wrong_group():
    g = torch.Generator().manual_seed(4)
    G, n, nsrc = 4, 96, 3
    grp = torch.tensor([1, 1, 0, 2], dtype=torch.int32)
    dst0 = torch.randn(G * n, generator=g)
    src = torch.randn(nsrc * n, generator=g)
    dst = dst0.clone()
    EmuKernelsVGG().gather_add(dst, src, grp, G, n)
    check_gather_add(dst, dst0, src, grp, G, n, "emulated gather_add")
    bad = dst0.clone()
    EmuKernelsVGG().gather_add(bad, src, torch.tensor([1, 0, 0, 2], dtype=torch.int32), G, n)
    _rejects(check_gather_add, bad, dst0, src, grp, G, n, "gather_add of the wrong group")
    out = torch.empty(nsrc * n)
    EmuKernels().group_sum(dst0, out, grp, G, nsrc, n)
    check_group_sum(dst0, out, grp.tolist(), G, nsrc, n, "emulated group_sum")
    EmuKernels().group_sum(dst0, out, torch.tensor([1, 0, 0, 2], dtype=torch.int32), G, nsrc, n)
    _rejects(check_group_sum, dst0, out, grp.tolist(), G, nsrc, n, "group_sum of the wrong group")
