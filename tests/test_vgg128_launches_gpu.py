"""The bf16 vgg_128 training step's kernel launches against float64, at 128x128 (3-channel frames, T = 30, B = 32, the bench
options: S = 29, one skip frame, a CPC decode).

vgg_128 is vgg_64 with a fifth 512-channel stage on both sides (engine_vgg.py VGG_ENC_128 / VGG_DEC_128), so every 3x3 layer
runs at twice the map size of its vgg_64 counterpart: the 64-channel layers at 128x128 (a 128-row tile is one image row, a
256-row bres tile two), the BatchNorm-statistics fusion on other layers than at C3, the 3-channel ends at 128x128.

  A. the launch lists tests/vgg_ref.py derives, against the conv_gemm launches one eager bf16 step records, at this shape and
     at C3 (vgg_64, T = 30, B = 128);
  B. every distinct kind-3 / kind-5 launch at its vgg_128 shape (tests/vgg_ref.py run_conv): no element left
     unwritten, float64 on slices of the first, middle and last round (the middle one straddling a group of B images),
     bit-identity against a launch of just those images, per-(image, channel) sums of the whole output, every fused
     statistics row and the finalized statistics;
  C. weight gradients: one kind-4 launch per (map size, swapped roles) class (K = N H W up to 15.7M), the GEMMs of the
     3-channel ends at 128x128, and the 4x4 GEMMs of the encoder's final layer and of dec-1: exact on 0 / 1 operands and
     within the bound on operands that do not cancel;
  D. BatchNorm at the unfused layers' shapes, every group against float64: bn_fwd_stats + bn_act, bn_bwd with the LeakyReLU
     slope recomputed + bn_param_grad, at vgg_128 and at C3;
  E. the vgg.cu data-movement kernels at 128x128 (up to 10^9 elements);
  F. an audit of real vgg_128 steps at T = 30, B = 8 (bench options, and a skip plan reading three skip sources): every launch
     checked as it runs, coverage of the derived list, skip addends read through plan.skip_src, and a step bit-identical to
     the unaudited step with its concurrent lanes and to a CUDA-graph replay of it.
"""
import math

import numpy as np
import pytest
import torch

from oracle import p2p_oracle as O
from p2pvg_b200._lib import CudaKernels
from p2pvg_b200.engine import ACT_LRELU, StepPlan
from p2pvg_b200.engine_vgg import TrainEngineVGG
from p2pvg_b200.layouts import up8
from tests.launch_audit import K, memory_per_test, sms  # noqa: F401  (fixtures)
from tests.launch_audit import (ALPHA_BN, BENCH_OPT, NAN, RecordingKernels, assert_equal_steps, bn_inputs, bn_stats, randn, run_step,
                                skip_seed)
from tests.ref64 import EPS, assert_exact, binary01, bn_group_ref64, bound_check, finalize_ref, gemm_ref64
from tests.tc_schedule import BETA, assert_within, gemm_tc_tiles
from tests.vgg_ref import (AUDIT_CASES, audit_vgg_step, backward_launches, distinct_convs, forward_launches, launch_key, run_conv,
                           run_end_gemms, run_im2col3_col2im3, run_maxpool, run_skip_index, run_upsample, run_wgrad, vgg_cfg,
                           wgrad_classes)

pytestmark = pytest.mark.gpu

SHAPES = {"vgg128": dict(T=30, B=32, W0=128), "C3": dict(T=30, B=128, W0=64)}
V128 = SHAPES["vgg128"]


def bench_plan(c):
    return StepPlan(c["T"], np.zeros(c["T"] - 1), O.default_opt(**BENCH_OPT))


def launches(name):
    c = SHAPES[name]
    p = bench_plan(c)
    return (forward_launches(c["T"], c["B"], p.S, p.nskip, c["W0"]),
            backward_launches(c["T"], c["B"], p.S, p.nskip, c["W0"], has_cpc=p.has_cpc))


# ------------------------------------------------------------------ A. the launch lists against a recorded step

def _conv_key(k, x):
    assert x["H"] == x["W"]
    return (x["kind"], x["N"], x["H"], x["Ck"], x["Cn"], x["Cm"], x["bias"] is not None,
            x["addend"].dtype if x["addend"] is not None else None, x["imgs_per_group"], x["stat_partial"] is not None)


class VggRecording(RecordingKernels):
    """Logs what every conv_gemm launch is (vgg_ref.launch_key)."""
    RECORD = {"conv_gemm": _conv_key}


@pytest.mark.parametrize("name", list(SHAPES))
def test_launch_list_matches_a_recorded_step(name):
    """The derived forward + backward list equals, launch for launch and in order, the conv_gemm launches of one eager bf16
    step at the shape: kind, N, H, channels, bias, addend, images per group and fused statistics.  The decoder's backward
    launches run over S B images (and B for the CPC decode), not over the forward's (S + 1) B."""
    c = SHAPES[name]
    T, B, W0 = c["T"], c["B"], c["W0"]
    rec = VggRecording("cuda")
    plan, (losses, _, _) = run_step(TrainEngineVGG, vgg_cfg(W0), BENCH_OPT, rec, T, B, 0)
    got = rec.calls
    assert np.all(np.isfinite(losses))
    assert (plan.S, plan.nskip, plan.has_cpc) == (29, 1, True)
    fwd, bwd = launches(name)
    want = [launch_key(L) for L in fwd + bwd]
    names = [L["name"] for L in fwd + bwd]
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"{name}: conv_gemm launch {i} is {g}, the derived list says {w} ({names[i]})"
    assert len(got) == len(want), f"{name}: {len(got)} conv_gemm launches recorded, {len(want)} derived"
    print(f"[list] {name}: {len(got)} conv_gemm launches, in order")


# ------------------------------------------------------------------ B. every distinct kind-3 / kind-5 launch

CONV = distinct_convs(sum(launches("vgg128"), []))


@pytest.mark.parametrize("L", CONV, ids=[f"{L['name'].replace(' ', '_')}-N{L['N']}" for L in CONV])
def test_vgg128_conv_launch(K, sms, L):
    """Checks 1-4 of one kind-3 / kind-5 launch of the vgg_128 step, with the engine's output dtype (bf16)."""
    run_conv(K, sms, L, torch.bfloat16, seed=51)


# ------------------------------------------------------------------ C. weight gradients

WGRAD = wgrad_classes(launches("vgg128")[1])


@pytest.mark.parametrize("L", WGRAD, ids=[f"{L['H']}x{L['H']}_{L['Cm']}x{L['Cn']}" for L in WGRAD])
def test_vgg128_weight_gradient(K, sms, L):
    """One kind-4 launch per (map size, swapped roles) class at its vgg_128 shape (K = N H W = 15.7M at 128x128: 0 / 1
    operands of density 1/4 sum to about K / 16, far below 2^24)."""
    run_wgrad(K, sms, L)


def test_vgg128_end_gemms(K):
    """The explicit GEMMs of the 3-channel ends at 128x128 (M = T B 128^2 = 15.7M pixels), including the last layer's
    [64 x ldl] weight gradient with K = M (ldl = up8(9 nc) = 32, the same launch as the first layer's)."""
    assert up8(9 * 3) == 32
    run_end_gemms(K, V128["T"] * V128["B"] * 128 * 128)


def _top_gemms():
    """The 4x4 GEMMs of vgg_128 (engine_vgg.py encode / decode / encoder_backward / decoder_backward): name, M, N, K, a_mn,
    b_mn, bias, output dtype."""
    T, B, g = V128["T"], V128["B"], 128
    S = bench_plan(V128).S
    bf, f32 = torch.bfloat16, torch.float32
    return [("enc_c6_fwd", T * B, g, 16 * 512, False, False, True, bf),
            ("enc_c6_wgrad", g, 16 * 512, T * B, True, True, False, f32),
            ("enc_c6_dgrad", T * B, 16 * 512, g, False, True, False, bf),
            ("dec-1_fwd", (S + 1) * B, 16 * 512, g, False, True, True, bf),
            ("dec-1_wgrad", g, 16 * 512, S * B, True, True, False, f32),
            ("dec-1_dgrad", S * B, g, 16 * 512, False, False, False, bf)]


TOP = _top_gemms()


@pytest.mark.parametrize("case", TOP, ids=[c[0] for c in TOP])
def test_vgg128_top_gemms(K, sms, case):
    """The encoder's final 4x4 layer and dec-1 at the vgg_128 shape.  Forward / data gradient: random operands against
    float64 within the K-long accumulation bound and one output rounding.  Weight gradients (fp32, both operands MN-major):
    exact on 0 / 1 operands, and within the split-K bound on operands that do not cancel."""
    name, M, N, Kd, a_mn, b_mn, has_bias, cdt = case
    torch.manual_seed(52)
    lda, ldb = (M if a_mn else Kd), (N if b_mn else Kd)
    if cdt == torch.float32:
        s = gemm_tc_tiles(M, N, Kd, sms)
        K.set_gemm_impl("tc")
        try:
            A, Bm = binary01((Kd, M)), binary01((Kd, N))
            C = torch.full((M, N), NAN, device="cuda")
            K.gemm(A, Bm, C, M, N, Kd, a_mn=True, b_mn=True)
            assert_exact(C, gemm_ref64(A, Bm, M, N, Kd, True, True, M, N)[0], Kd, f"{name} 0/1 operands")
            A = torch.rand(Kd, M, device="cuda").bfloat16()
            Bm = randn(Kd, N, scale=0.5) + 0.5
            K.gemm(A, Bm, C, M, N, Kd, a_mn=True, b_mn=True)
        finally:
            K.set_gemm_impl("auto")
        ref, absref = gemm_ref64(A, Bm, M, N, Kd, True, True, M, N)
        assert (ref.abs() >= 0.5 * absref).all()
        assert_within(C, ref, absref, s.kb_per_split * 64 + 16 * s.splits, torch.float32, name=f"{name} {M}x{N} K={Kd} splits={s.splits}")
        return
    A = randn(*((Kd, M) if a_mn else (M, Kd)), scale=0.5)
    Bm = randn(*((Kd, N) if b_mn else (N, Kd)), scale=1.0 / math.sqrt(Kd))
    bias = randn(N, dtype=torch.float32) if has_bias else None
    C = torch.full((M, N), NAN, device="cuda", dtype=cdt)
    K.gemm(A, Bm, C, M, N, Kd, a_mn=a_mn, b_mn=b_mn, bias=bias)
    ref, absref = gemm_ref64(A, Bm, M, N, Kd, a_mn, b_mn, lda, ldb, bias=bias)
    assert_within(C, ref, absref, Kd, cdt, name=f"{name} {M}x{N} K={Kd}")


# ------------------------------------------------------------------ D. BatchNorm at the unfused layers' shapes

def _unfused_shapes():
    """(config, G, R, C, layer) of every distinct BatchNorm shape whose statistics come from a separate pass: the implicit
    layers stat_buf does not fuse, and the 3-channel first layer."""
    out = []
    for n, c in SHAPES.items():
        T, B, W0 = c["T"], c["B"], c["W0"]
        shapes = [(T, B * W0 * W0, 64, "enc0.0")]
        shapes += [(T if L["name"].startswith("enc") else bench_plan(c).S + 1, B * L["H"] ** 2, L["Cn"], L["name"])
                   for L in launches(n)[0] if L["stat"] is None and not L["name"].endswith(".S")]
        for G, R, C, nm in shapes:
            if (n, G, R, C) not in [o[:4] for o in out]:
                out.append((n, G, R, C, nm))
    return out


BN = _unfused_shapes()


def _side(x, st, g, C):
    """The LeakyReLU side the kernel takes: the sign of its fp32 fmaf(x, scale, shift)."""
    return x.double() * st["scale"].view(-1, C)[g].double() + st["shift"].view(-1, C)[g].double() > 0


@pytest.mark.parametrize("case", BN, ids=[f"{c[0]}-{c[4]}-G{c[1]}_R{c[2]}_C{c[3]}" for c in BN])
def test_bn_forward_at_launch_shape(K, case):
    """bn_fwd_stats and bn_act (LeakyReLU) over G groups of R rows, every group against float64: the statistics within
    finalize_ref's bound on sums known within ALPHA_BN, y within one fp32 and one bf16 rounding."""
    cfg, G, R, C, nm = case
    name = f"{cfg} {nm} G={G} R={R} C={C}"
    raw, gamma, beta, _ = bn_inputs(G, R, C, seed=G * 7 + C + R)
    st = bn_stats(K, raw, G, R, C, gamma, beta)
    y = torch.full_like(raw, NAN)
    K.bn_act(raw, y, st["scale"], st["shift"], G, R, C, ACT_LRELU)
    x, yv = raw.view(G, R, C), y.view(G, R, C)
    ws = wa = 0.0
    for g in range(G):
        xg = x[g].double()
        refs = finalize_ref(xg.sum(0), (xg * xg).sum(0), xg.abs().sum(0), R, gamma, beta, EPS, ALPHA_BN)
        for k, (ref, bnd), what in zip(("mean", "invstd", "varu", "scale", "shift"), refs, ("mean", "invstd", "varu", "scale", "shift")):
            ws = max(ws, bound_check(st[k].view(G, C)[g], ref, bnd, f"bn_fwd_stats {name} group {g} {what}"))
        sc, sh = st["scale"].view(G, C)[g].double(), st["shift"].view(G, C)[g].double()
        pre = xg * sc + sh
        ref = torch.where(pre > 0, pre, 0.2 * pre)
        wa = max(wa, bound_check(yv[g], ref, BETA[torch.bfloat16] * ref.abs() + 2.0 ** -23 * ((xg * sc).abs() + sh.abs()),
                                 f"bn_act {name} group {g}"))
        del xg, pre, ref
    print(f"[bound] BatchNorm forward {name}: stats {ws:.3g}, bn_act {wa:.3g}")


@pytest.mark.parametrize("case", BN, ids=[f"{c[0]}-{c[4]}-G{c[1]}_R{c[2]}_C{c[3]}" for c in BN])
def test_bn_bwd_at_launch_shape(K, case):
    """bn_bwd as the step calls it (in place, LeakyReLU slope recomputed from scale / shift) and bn_param_grad, every group
    against float64 (ref64.bn_group_ref64): dx within one bf16 rounding, the per-group sums and dgamma / dbeta within
    ALPHA_BN of their magnitudes."""
    cfg, G, R, C, nm = case
    name = f"bn_bwd {cfg} {nm} G={G} R={R} C={C}"
    raw, gamma, beta, gen = bn_inputs(G, R, C, seed=G * 11 + C + R)
    st = bn_stats(K, raw, G, R, C, gamma, beta)
    x = raw.view(G, R, C)
    # dy correlated with xhat, so that the xhat term of dx carries weight
    dy = torch.empty_like(raw)
    for g in range(G):
        xg = x[g].double()
        xh = (xg - xg.mean(0)) / torch.sqrt(xg.var(0, unbiased=False) + EPS)
        dy.view(G, R, C)[g] = (0.5 * xh + torch.randn(R, C, device="cuda", dtype=torch.float64, generator=gen)).to(dy.dtype)
        del xg, xh
    d = dy.clone()
    K.bn_bwd(d, raw, None, st["mean"], st["invstd"], gamma, G, R, C, ACT_LRELU, d, st["sdz"], st["sdzx"], scale=st["scale"],
             shift=st["shift"])
    dg, db = torch.full((C,), NAN, device="cuda"), torch.full((C,), NAN, device="cuda")
    K.bn_param_grad(st["sdz"], st["sdzx"], G, C, dg, db)
    torch.cuda.synchronize()
    w = 0.0
    tot = dict(sdz=0.0, sdzx=0.0, sdz_mag=0.0, sdzx_mag=0.0)
    for g in range(G):
        r = bn_group_ref64(x[g], dy.view(G, R, C)[g], gamma, beta, ACT_LRELU, side=_side(x[g], st, g, C))
        w = max(w, assert_within(d.view(G, R, C)[g], r["dx"], r["dx_mag"], 0, torch.bfloat16, alpha=ALPHA_BN, quiet=True,
                                 name=f"{name} dx group {g}"))
        for k in ("sdz", "sdzx"):
            w = max(w, assert_within(st[k].view(G, C)[g], r[k], r[k + "_mag"], 0, torch.float32, alpha=ALPHA_BN, quiet=True,
                                     name=f"{name} {k} group {g}"))
        for k in tot:
            tot[k] = tot[k] + r[k]
        del r
    w = max(w, assert_within(dg, tot["sdzx"], tot["sdzx_mag"], 0, torch.float32, alpha=ALPHA_BN, name=f"{name} dgamma"))
    w = max(w, assert_within(db, tot["sdz"], tot["sdz_mag"], 0, torch.float32, alpha=ALPHA_BN, name=f"{name} dbeta"))
    print(f"[bound] {name}: worst error/bound {w:.3g}")


# ------------------------------------------------------------------ E. vgg.cu data movement at 128x128

V128_N = V128["T"] * V128["B"]


def test_maxpool_vgg128(K):
    """maxpool2_fwd / maxpool2_bwd from the 128x128x64 encoder map (N = 960: 10^9 input elements) to 64x64."""
    run_maxpool(K, V128_N, 128, 64, torch.bfloat16, "vgg128")


def test_upsample_vgg128(K):
    """upsample2_fwd / upsample2_bwd at the 128x128 decoder stage entry (64x64x64 -> 128x128x64 at N = 960)."""
    run_upsample(K, V128_N, 64, 64, torch.bfloat16, "vgg128")


def test_im2col3_col2im3_vgg128(K):
    """im2col3 (row32 against generic, both tap signs) and col2im3 on N = 960 frames of 128x128x3."""
    run_im2col3_col2im3(K, V128_N, 128, torch.bfloat16, "vgg128")


def test_skip_index_kernels_vgg128(K):
    """group_sum and add_indexed at the 128-stage skip: decoder_backward(0, S) sums S = 29 groups of B = 32 images of
    128x128x64 (n = 33.5M elements per group, 10^9 in all), here onto three skip sources."""
    run_skip_index(K, bench_plan(V128).S, V128["B"], 128, 64, torch.bfloat16, gather=False)


# ------------------------------------------------------------------ F. audit of real vgg_128 steps

@pytest.mark.parametrize("case", AUDIT_CASES, ids=[c[0] for c in AUDIT_CASES])
def test_audit_vgg128_step(case):
    """One eager bf16 vgg_128 step at T = 30, B = 8 with every launch checked as it runs (vgg_ref.audit_vgg_step: coverage of
    the derived list, skip addends through plan.skip_src, equal to the plain step), and the plain step equal to a CUDA-graph
    replay."""
    name, optkw = case
    T, B = 30, 8
    eager = audit_vgg_step(name, optkw, T, B, W0=128)
    np_seed = skip_seed(T) if optkw.get("skip_prob") else 0
    _, graph = run_step(TrainEngineVGG, vgg_cfg(128), optkw, CudaKernels("cuda"), T, B, np_seed, use_graph=True)
    assert_equal_steps(eager, graph, f"vgg128 {name}: graph replay vs eager")
    print(f"[audit] vgg128 {name}: graph replay equals the eager step")
