"""The bf16 dcgan training steps' kernel launches against float64, at the shapes of the C2 benchmark configuration (dcgan_64,
1 channel, T = 30, B = 256) and of C4 (dcgan_128, 3 channels, 128x128, T = 30, B = 64 per GPU).

  A. the launch lists tests/dcgan_ref.py derives from the engine's rules, against what one eager bf16 step records at exactly
     the C2 and C4 shapes, and the rows of the C2 launch table (DESIGN.md §5);
  B. every distinct kind-0 / kind-2 implicit-GEMM launch at its C2 or C4 shape: no element left unwritten, float64 on image
     slices of the first, middle and last round (the middle one straddling a group of B images), bit-identity of those slices
     against a launch of just those images, per-(image, channel) sums of the whole output, every fused statistics row and
     the finalized statistics;
  C. weight gradients: one kind-1 launch per (map size, swapped roles) class and the long-K GEMMs (the encoder's final 4x4
     layer, dec-1, the 3-channel ends of C4 with K = 7.86M), exact on 0 / 1 operands and within the bound on operands that do
     not cancel;
  D. BatchNorm at the launch shapes, group by group against float64: forward statistics and the activation on the unfused
     layers, bn_bwd (LeakyReLU recomputed from scale / shift, and the tanh encoder output) with bn_param_grad, bn_bwd_group_sum
     at dec0..dec2 (one skip source, and four sources of which one is read by no group), its `dout` reduce at C2 dec2 (the
     last layer's weight gradient over 7.6M rows), and bn_bwd_wgrad_c1 at C2 enc0 (capped BatchNorm chunks of 4096 rows);
     the two weight gradients on operands that do not cancel, within the bound of one chunk's fp32 accumulation;
  E. an audit of real steps (dcgan_64 at T = 30, B = 64 with the bench options and with a skip plan; dcgan_128 at T = 30,
     B = 16): every conv_gemm, bf16 GEMM, skip-frame sum and add_indexed checked against float64 as it runs, coverage of
     every conv_gemm variant of the derived list, the skip addends read through plan.skip_src, and a step bit-identical to
     the same step on plain CudaKernels with its concurrent lanes.
"""
import math

import numpy as np
import pytest
import torch

from oracle import p2p_oracle as O
from p2pvg_b200.engine import StepPlan, TrainEngine
from tests.dcgan_ref import (ACT_LRELU, ACT_TANH, check_conv4_sums, check_stat_rows, check_wgrad_c1, conv4_ref64_elem, conv_variant,
                             forward_launches, key, step_launches, wgrad4_ref64, wgrad_c1_ref64)
from tests.launch_audit import K, memory_per_test, sms  # noqa: F401  (fixtures)
from tests.launch_audit import (BENCH_OPT, NAN, SKIP_OPT, AuditKernels, RecordingKernels, addend_index, audit_step, bn_inputs,
                                bn_stats, randn, slices_with_boundary)
from tests.launch_audit import bn_bwd_refs as _refs, check_bn_bwd as _check_bwd, check_bn_stats as _check_stats
from tests.ref64 import EPS, assert_exact, binary01, bound_check, check_finalize_vs_output, gemm_ref64
from tests.tc_schedule import BETA, assert_within, cdiv, conv_tiles, gemm_tc_tiles, sm_count

pytestmark = pytest.mark.gpu

CONFIGS = {"C2": dict(T=30, B=256, nc=1, W0=64), "C4": dict(T=30, B=64, nc=3, W0=128)}


def plan_for(cfg):
    return StepPlan(cfg["T"], np.zeros(cfg["T"] - 1), O.default_opt(**BENCH_OPT))


def launches(name):
    c = CONFIGS[name]
    p = plan_for(c)
    return step_launches(c["T"], c["B"], p.S, p.nskip, c["nc"], c["W0"], p.has_cpc)


# ------------------------------------------------------------------ A. the launch lists

def _bn_key(op, C=None, act=None):
    """What dcgan_ref.key gives a BatchNorm entry point; C / act: the value listed where the entry point takes no such
    argument (None: the entry has none)."""
    def f(k, x):
        return (op, x["G"], x["R"] if "R" in x else None, x["C"] if "C" in x else C, x["act"] if "act" in x else act, x.get("F"),
                x["dout"] is not None if op == "bn_bwd_group_sum" else False)
    return f


class DcganRecording(RecordingKernels):
    """Logs the shapes and flags of every conv_gemm, bf16 gemm and BatchNorm launch."""
    muted = False   # set while the engine runs the LSTM weight gradients (bf16 copies of fp32 operands)
    RECORD = {
        "conv_gemm": lambda k, x: ("conv_gemm", x["kind"], x["N"], x["H"], x["Ck"], x["Cn"], x["Cm"], x["bias"] is not None,
                                   x["addend"].dtype if x["addend"] is not None else None, x["imgs_per_group"],
                                   x["stat_partial"] is not None),
        # the LSTM / latent GEMMs take fp32 operands
        "gemm": lambda k, x: ("gemm", x["M"], x["N"], x["K"], x["a_mn"], x["b_mn"], x["bias"] is not None)
        if x["A"].dtype == torch.bfloat16 and not k.muted else None,
        "bn_fwd_stats": _bn_key("bn_fwd_stats"),
        "bn_fwd_finalize_tiles": _bn_key("bn_fwd_finalize_tiles"),
        "bn_act": _bn_key("bn_act"),
        "bn_bwd": _bn_key("bn_bwd"),
        "bn_bwd_group_sum": _bn_key("bn_bwd_group_sum", act=ACT_LRELU),
        "bn_bwd_wgrad_c1": _bn_key("bn_bwd_wgrad_c1", C=64, act=ACT_LRELU),
        "bn_param_grad": _bn_key("bn_param_grad"),
    }


def _cfg(c):
    return dict(g_dim=128, z_dim=10, rnn_size=256, channels=c["nc"], image_width=c["W0"], predictor_rnn_layers=2,
                posterior_rnn_layers=1, prior_rnn_layers=1)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_launch_list_matches_an_eager_step(name):
    """The derived list equals, call for call and in order, what one eager bf16 step at the configuration's exact shape
    enqueues (conv_gemm, the bf16 GEMMs of the convolution stacks, and the BatchNorm entry points)."""
    from p2pvg_b200.engine import TrainEngine
    c = CONFIGS[name]
    T, B = c["T"], c["B"]
    opt = O.default_opt(**BENCH_OPT)
    opt["batch_size"] = B
    eng = TrainEngine(O.build_state(_cfg(c), seed=1), _cfg(c), opt, DcganRecording("cuda"), act_dtype=torch.bfloat16)
    lin_wgrad = eng.lin_wgrad

    def muted_lin_wgrad(*a, **kw):   # TrainEngine.lin_wgrad: the LSTM / head weight gradients, not part of the lists
        eng.K.muted = True
        try:
            lin_wgrad(*a, **kw)
        finally:
            eng.K.muted = False
    eng.lin_wgrad = muted_lin_wgrad
    x = torch.rand(T, B, c["nc"], c["W0"], c["W0"], generator=torch.Generator().manual_seed(5))
    probs = np.zeros(T - 1)
    plan = StepPlan(T, probs, opt)
    eps = O.draw_eps(plan.S, B, 10, seed=11)
    losses = eng.step(x.cuda(), probs=probs, eps=eps.cuda())
    torch.cuda.synchronize()
    assert np.all(np.isfinite(np.asarray(losses)))
    got = eng.K.calls
    want = [key(L) for L in launches(name)]
    del eng
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"{name}: launch {i} is {g}, the derived list says {w} ({launches(name)[i]['name']})"
    assert len(got) == len(want), f"{name}: {len(got)} launches recorded, {len(want)} derived"
    print(f"[list] {name}: {len(got)} launches, in order")


def test_c2_launch_table():
    """The rows of the C2 launch table (DESIGN.md §5): 21 kind-0 / kind-2 launches, N = 7680 (T B), 7424 (the frames after
    the first) or 256 (skip frames and the CPC step), statistics on enc2, enc3 and dec0, the bf16 skip addend on the three
    decoder stages, and 256 x 64 tiles exactly on dec2 and the enc1 data gradient (and the 256-image dec2 skip half)."""
    L = [x for x in launches("C2") if x["op"] == "conv_gemm" and x["kind"] in (0, 2)]
    assert len(L) == 21
    rows = [(x["name"], x["kind"], x["N"], x["H"], x["Ck"], x["Cn"], x["stat"] is not None, x["addend"] is not None, x["variant"][1])
            for x in L]
    assert rows == [
        ("enc1", 0, 7680, 16, 64, 128, False, False, "128x128"),
        ("enc2", 0, 7680, 8, 128, 256, True, False, "128x128"),
        ("enc3", 0, 7680, 4, 256, 512, True, False, "128x128"),
        ("dec0.S", 2, 256, 4, 512, 256, False, False, "128x128"),
        ("dec0.D", 2, 7680, 4, 512, 256, True, True, "128x128"),
        ("dec1.S", 2, 256, 8, 256, 128, False, False, "128x128"),
        ("dec1.D", 2, 7680, 8, 256, 128, False, True, "128x128"),
        ("dec2.S", 2, 256, 16, 128, 64, False, False, "256x64"),
        ("dec2.D", 2, 7680, 16, 128, 64, False, True, "256x64"),
        ("dec2 dgrad S", 0, 256, 16, 64, 128, False, False, "128x128"),
        ("dec2 dgrad D", 0, 7424, 16, 64, 128, False, False, "128x128"),
        ("dec1 dgrad S", 0, 256, 8, 128, 256, False, False, "128x128"),
        ("dec1 dgrad D", 0, 7424, 8, 128, 256, False, False, "128x128"),
        ("dec0 dgrad S", 0, 256, 4, 256, 512, False, False, "128x128"),
        ("dec0 dgrad D", 0, 7424, 4, 256, 512, False, False, "128x128"),
        ("cpc dec2 dgrad D", 0, 256, 16, 64, 128, False, False, "128x128"),
        ("cpc dec1 dgrad D", 0, 256, 8, 128, 256, False, False, "128x128"),
        ("cpc dec0 dgrad D", 0, 256, 4, 256, 512, False, False, "128x128"),
        ("enc3 dgrad", 2, 7680, 4, 512, 256, False, False, "128x128"),
        ("enc2 dgrad", 2, 7680, 8, 256, 128, False, False, "128x128"),
        ("enc1 dgrad", 2, 7680, 16, 128, 64, False, False, "256x64"),
    ]
    # the statistics layers keep the per-row store; the plain bf16 and bf16-addend launches store rows cooperatively
    assert [x["variant"][-1] for x in L].count("perrow") == 3
    # tile counts of the table's launches on this device
    s = sm_count()
    for x in L:
        sc = conv_tiles(x["kind"], x["N"], x["H"], x["H"], x["Ck"], x["Cn"], 0, s, stat=x["stat"] is not None)
        assert sc.BM == int(x["variant"][1].split("x")[0])
        print(f"[table] {x['name']}: {sc.tiles} tiles of {sc.BM}x{sc.BN}, {sc.rounds} rounds")


# ------------------------------------------------------------------ B. every distinct kind-0 / kind-2 launch

def _dedup(Ls):
    seen, out = set(), []
    for L in Ls:
        if L["op"] == "conv_gemm" and L["kind"] in (0, 2) and key(L) not in seen:
            seen.add(key(L))
            out.append(L)
    return out


CONV = [(n, L) for n in CONFIGS for L in _dedup(launches(n))]


@pytest.mark.parametrize("cfg,L", CONV, ids=[f"{n}-{L['name'].replace(' ', '_')}-N{L['N']}" for n, L in CONV])
def test_conv_launch(K, sms, cfg, L):
    kind, N, H, Ck, Cn, B = L["kind"], L["N"], L["H"], L["Ck"], L["Cn"], CONFIGS[cfg]["B"]
    HW = H * H
    name = f"{cfg} {L['name']} kind {kind} N={N} {H}x{H} {Ck}->{Cn}"
    torch.manual_seed(31)
    Ha = 2 * H if kind == 0 else H
    a = randn(N, Ha, Ha, Ck, scale=0.5)
    b = randn(*((Cn, 16 * Ck) if kind == 0 else (Ck, 16 * Cn)), scale=1.0 / math.sqrt(16 * Ck))
    bias = randn(Cn, dtype=torch.float32) if L["bias"] else None
    Ho = 2 * H if kind == 2 else H
    add = src = idx = None
    ipg = L["ipg"]
    if L["addend"] is not None:
        nsrc = 3   # more sources than the bench plan's one: every group reads another source than its neighbours
        G = cdiv(N, ipg)
        src = torch.tensor([(g + 1) % nsrc for g in range(G)], dtype=torch.int32, device="cuda")
        idx = addend_index(src.tolist(), ipg, N)
        add = randn(nsrc * ipg, Ho, Ho, Cn)
    st = L["stat"]
    s = conv_tiles(kind, N, H, H, Ck, Cn, 0, sms, stat=st is not None)
    assert s.BM == int(L["variant"][1].split("x")[0])
    part = torch.full((s.tiles_m * s.phases, Cn, 2), NAN, device="cuda") if st is not None else None
    out = torch.full((N, Ho, Ho, Cn), NAN, device="cuda", dtype=torch.bfloat16)
    K.conv_gemm(kind, a, b, out, N, H, H, Ck, Cn, bias=bias, addend=add, grp_src=src, imgs_per_group=ipg, stat_partial=part)
    torch.cuda.synchronize()
    assert not torch.isnan(out).any(), f"{name}: unwritten output elements"
    if part is not None:
        assert not torch.isnan(part).any(), f"{name}: unwritten statistics rows"

    def locate(ix, i0):
        n, y, x, c = ix
        if kind == 2:
            row, ph = ((i0 + n) * H + y // 2) * H + x // 2, (y & 1) * 2 + (x & 1)
        else:
            row, ph = ((i0 + n) * H + y) * H + x, 0
        return s.where(0, row // s.BM, c // s.BN, ph)
    worst = 0.0
    for i0, i1 in slices_with_boundary(N, HW, s, sms, B):
        arows = add[idx[i0:i1]] if add is not None else None
        ref, absref = conv4_ref64_elem(kind, a[i0:i1], b, H, Ck, Cn, bias, arows)
        worst = max(worst, assert_within(out[i0:i1], ref, absref, 16 * Ck, torch.bfloat16, quiet=True,
                                         name=f"{name} images [{i0}, {i1})", locate=lambda ix, i0=i0: locate(ix, i0)))
        del ref, absref
        sub = conv_tiles(kind, i1 - i0, H, H, Ck, Cn, 0, sms, stat=st is not None)
        assert sub.tiles <= sms
        o = torch.empty(i1 - i0, Ho, Ho, Cn, device="cuda", dtype=torch.bfloat16)
        p = torch.full((sub.tiles_m * s.phases, Cn, 2), NAN, device="cuda") if st is not None else None
        kw = {}
        if add is not None:   # the same addend rows, one group per image
            kw = dict(addend=arows.contiguous(), grp_src=torch.arange(i1 - i0, dtype=torch.int32, device="cuda"), imgs_per_group=1)
        K.conv_gemm(kind, a[i0:i1], b, o, i1 - i0, H, H, Ck, Cn, bias=bias, stat_partial=p, **kw)
        assert torch.equal(o, out[i0:i1]), f"{name}: images [{i0}, {i1}) differ from a launch of just those images"
        if p is not None:
            t0 = i0 * HW // 128 * s.phases
            assert torch.equal(p, part[t0:t0 + p.shape[0]]), f"{name}: statistics rows of images [{i0}, {i1}) differ"
        del o, p, arows
    print(f"[bound] {name} slices: worst error/bound {worst:.3g}")
    check_conv4_sums(out, kind, a, b, N, H, Ck, Cn, bias, add, idx, name=name)
    if st is not None:
        check_stat_rows(part, out, kind, N, H, Cn, name=name)
        check_finalize_vs_output(K, part, st["parts_per_group"], out, N // B, B * Ho * Ho, Cn, name=name)


# ------------------------------------------------------------------ C. weight gradients

def _wgrad_classes():
    sms_ = sm_count() if torch.cuda.is_available() else 132
    seen, out = set(), []
    for n in CONFIGS:
        for L in launches(n):
            if L["op"] == "conv_gemm" and L["kind"] == 1:
                s = conv_tiles(1, L["N"], L["H"], L["H"], 0, L["Cn"], L["Cm"], sms_)
                if (L["H"], s.swap) not in seen:
                    seen.add((L["H"], s.swap))
                    out.append((n, L))
    return out


WGRAD = _wgrad_classes()


@pytest.mark.parametrize("cfg,L", WGRAD, ids=[f"{n}-{L['name'].replace(' ', '_')}-{L['H']}x{L['H']}" for n, L in WGRAD])
def test_kind1_weight_gradient(K, sms, cfg, L):
    """A kind-1 launch (a: small map [N, H, H, Cm], b: big map [N, 2H, 2H, Cn]) against a float64 reduction over all N H W
    pixels: (1) 0 / 1 operands, exact; (2) operands that do not cancel (one positive, one of mean 1/2), within the bound."""
    N, H, Cm, Cn = L["N"], L["H"], L["Cm"], L["Cn"]
    s = conv_tiles(1, N, H, H, 0, Cn, Cm, sms)
    name = f"{cfg} wgrad {L['name']} N={N} {H}x{H} {Cm}x{Cn} swap={s.swap} splits={s.splits}"
    torch.manual_seed(32)
    a, b = binary01((N, H, H, Cm)), binary01((N, 2 * H, 2 * H, Cn))
    out = torch.full((Cm, 16 * Cn), NAN, device="cuda")
    K.conv_gemm(1, a, b, out, N, H, H, 0, Cn, Cm=Cm)
    assert_exact(out, wgrad4_ref64(a, b, N, H, Cm, Cn)[0], N * H * H, name + " 0/1 operands")
    a = torch.rand(N, H, H, Cm, device="cuda").bfloat16()
    b = randn(N, 2 * H, 2 * H, Cn, scale=0.5) + 0.5
    K.conv_gemm(1, a, b, out, N, H, H, 0, Cn, Cm=Cm)
    ref, absref = wgrad4_ref64(a, b, N, H, Cm, Cn)
    assert (ref.abs() >= 0.25 * absref).all()
    assert_within(out, ref, absref, s.kb_per_split * 64 + 16 * s.splits, torch.float32, name=f"{name} non-cancelling operands")


def _long_gemms():
    out = []
    for n in CONFIGS:
        for L in launches(n):
            if L["op"] == "gemm" and L["a_mn"] and L["b_mn"]:
                out.append((n, L))
    return out


LONG = _long_gemms()


@pytest.mark.parametrize("cfg,L", LONG, ids=[f"{n}-{L['name'].replace(' ', '_')}-K{L['K']}" for n, L in LONG])
def test_weight_gradient_gemm(K, sms, cfg, L):
    """The weight-gradient GEMMs C[M, N] = A[K, M]^T B[K, N] (both MN-major) of the stacks at their shapes, the encoder's final
    4x4 layer, dec-1 and the 1- / 3-channel ends (K up to 7.86M): exact on 0 / 1 operands, and within the bound of the split-K
    schedule gemm_tc picks (each split accumulates kb_per_split K blocks, the reduce adds `splits` partials) on operands that
    do not cancel.  bf16 operands take gemm_tc in the engine's "auto" mode; "tc" makes a fallback an error instead."""
    M, N, Kd = L["M"], L["N"], L["K"]
    s = gemm_tc_tiles(M, N, Kd, sms)
    name = f"{cfg} {L['name']} {M}x{N} K={Kd} splits={s.splits}"
    torch.manual_seed(33)
    K.set_gemm_impl("tc")
    try:
        A, Bm = binary01((Kd, M)), binary01((Kd, N))
        C = torch.full((M, N), NAN, device="cuda")
        K.gemm(A, Bm, C, M, N, Kd, a_mn=True, b_mn=True)
        assert_exact(C, gemm_ref64(A, Bm, M, N, Kd, True, True, M, N)[0], Kd, name + " 0/1 operands")
        A = torch.rand(Kd, M, device="cuda").bfloat16()
        Bm = randn(Kd, N, scale=0.5) + 0.5
        K.gemm(A, Bm, C, M, N, Kd, a_mn=True, b_mn=True)
    finally:
        K.set_gemm_impl("auto")
    ref, absref = gemm_ref64(A, Bm, M, N, Kd, True, True, M, N)
    assert (ref.abs() >= 0.5 * absref).all()
    assert_within(C, ref, absref, s.kb_per_split * 64 + 16 * s.splits, torch.float32, name=f"{name} non-cancelling operands")


# ------------------------------------------------------------------ D. BatchNorm at the launch shapes

def _unfused_fwd_shapes():
    out = []
    for n in CONFIGS:
        for L in launches(n):
            if L["op"] == "bn_act" and (n, L["G"], L["R"], L["C"], L["act"]) not in [o[:5] for o in out]:
                out.append((n, L["G"], L["R"], L["C"], L["act"], L["name"]))
    return out


FWD = _unfused_fwd_shapes()


@pytest.mark.parametrize("case", FWD, ids=[f"{c[0]}-{c[5]}-G{c[1]}_R{c[2]}_C{c[3]}" for c in FWD])
def test_bn_forward_at_launch_shape(K, case):
    """bn_fwd_stats (the layers without fused statistics; run on every BatchNorm shape of the step) and bn_act: statistics
    within the float64 bound, y = act(fmaf(x, scale, shift)) within one fp32 and one bf16 rounding."""
    cfg, G, R, C, act, nm = case
    name = f"{cfg} {nm} G={G} R={R} C={C}"
    raw, gamma, beta, _ = bn_inputs(G, R, C, seed=G * 7 + C)
    st = bn_stats(K, raw, G, R, C, gamma, beta)
    w = _check_stats(st, raw, G, R, C, gamma, beta, f"bn_fwd_stats {name}")
    y = torch.full_like(raw, NAN)
    K.bn_act(raw, y, st["scale"], st["shift"], G, R, C, act)
    x, yv = raw.view(G, R, C), y.view(G, R, C)
    sc, sh = st["scale"].view(G, 1, C).double(), st["shift"].view(G, 1, C).double()
    wa = 0.0
    for g in range(G):
        pre = x[g].double() * sc[g] + sh[g]
        mag = (x[g].double() * sc[g]).abs() + sh[g].abs()
        if act == ACT_LRELU:
            ref = torch.where(pre > 0, pre, 0.2 * pre)
            bnd = BETA[torch.bfloat16] * ref.abs() + 2.0 ** -23 * mag
        else:
            ref = torch.tanh(pre)
            bnd = BETA[torch.bfloat16] * ref.abs() + 2.0 ** -23 * mag + 2.0 ** -21
        wa = max(wa, bound_check(yv[g], ref, bnd, f"bn_act {name} group {g}"))
    print(f"[bound] {name}: stats {w:.3g}, bn_act {wa:.3g}")


def _bwd_shapes():
    out = []
    for n in CONFIGS:
        for L in launches(n):
            if L["op"] == "bn_bwd" and (n, L["G"], L["R"], L["C"], L["act"]) not in [o[:5] for o in out]:
                out.append((n, L["G"], L["R"], L["C"], L["act"], L["name"]))
    return out


BWD = _bwd_shapes()


@pytest.mark.parametrize("case", BWD, ids=[f"{c[0]}-{c[5]}-G{c[1]}_R{c[2]}_C{c[3]}" for c in BWD])
def test_bn_bwd_at_launch_shape(K, case):
    """bn_bwd as the step calls it (in place; LeakyReLU: y = None, slope from scale / shift; tanh: y given) and bn_param_grad."""
    cfg, G, R, C, act, nm = case
    name = f"bn_bwd {cfg} {nm} G={G} R={R} C={C}"
    raw, gamma, beta, gen = bn_inputs(G, R, C, seed=G * 11 + C)
    st = bn_stats(K, raw, G, R, C, gamma, beta)
    x64 = raw.view(G, R, C)
    # dy correlated with xhat, so that the xhat term of dx carries weight
    dy = torch.empty_like(raw)
    for g in range(G):
        xg = x64[g].double()
        xh = (xg - xg.mean(0)) / torch.sqrt(xg.var(0, unbiased=False) + EPS)
        dy.view(G, R, C)[g] = (0.5 * xh + torch.randn(R, C, device="cuda", dtype=torch.float64, generator=gen)).to(dy.dtype)
    y = None
    if act == ACT_TANH:
        y = torch.empty_like(raw)
        K.bn_act(raw, y, st["scale"], st["shift"], G, R, C, ACT_TANH)
    refs = _refs(raw, dy, st, gamma, beta, G, R, C, act, y)
    d = dy.clone()
    if act == ACT_LRELU:
        K.bn_bwd(d, raw, None, st["mean"], st["invstd"], gamma, G, R, C, act, d, st["sdz"], st["sdzx"], scale=st["scale"], shift=st["shift"])
    else:
        K.bn_bwd(d, raw, y, st["mean"], st["invstd"], gamma, G, R, C, act, d, st["sdz"], st["sdzx"])
    dg, db = torch.full((C,), NAN, device="cuda"), torch.full((C,), NAN, device="cuda")
    K.bn_param_grad(st["sdz"], st["sdzx"], G, C, dg, db)
    w = _check_bwd(dict(dx=d.view(G, R, C), sdz=st["sdz"], sdzx=st["sdzx"], dgamma=dg, dbeta=db), refs, G, C, name)
    print(f"[bound] {name}: worst error/bound {w:.3g}")


def _group_sum_cases():
    out = []
    for L in launches("C2"):
        if L["op"] == "bn_bwd_group_sum":
            Ho = int(round(math.sqrt(L["R"] // CONFIGS["C2"]["B"])))
            out.append(("C2", L["name"], L["G"], L["R"], L["C"], Ho, L["dout"]))
    return out


GS = _group_sum_cases()
PLANS = {"one_source": lambda G: ([0] * G, 1),
         # four sources, the third read by no group, in runs and out of order
         "four_sources": lambda G: ([(0, 1, 3)[(g * 5 // G + g % 2) % 3] for g in range(G)], 4)}


@pytest.mark.parametrize("plan", list(PLANS))
@pytest.mark.parametrize("case", GS, ids=[f"{c[0]}-{c[1]}-G{c[2]}_R{c[3]}_C{c[4]}{'_dout' if c[6] else ''}" for c in GS])
def test_bn_bwd_group_sum_at_launch_shape(K, case, plan):
    """bn_bwd_group_sum at dec0, dec1 and dec2 of C2 (G = 29, R = B Ho^2): dx and the BatchNorm sums against float64, the skip
    sums against the float64 sums of the stored dx over the groups that read each source (zeros for a source no group reads),
    and at dec2 with `dout`: the weight gradient of the 64 -> 1 last layer over all G R rows against float64."""
    cfg, nm, G, R, C, Ho, with_dout = case
    srcl, Fs = PLANS[plan](G)
    assert G == 29 and R == CONFIGS[cfg]["B"] * Ho * Ho
    if plan == "four_sources":
        assert len(set(srcl)) == 3 and 2 not in srcl
    name = f"bn_bwd_group_sum {cfg} {nm} G={G} R={R} C={C} {plan}"
    raw, gamma, beta, gen = bn_inputs(G, R, C, seed=G * 13 + C)
    if with_dout:   # beta >= 0.5: y = lrelu(gamma xhat + beta) has a positive mean in every channel, so y * dout does not cancel
        beta = beta.abs() + 0.5
    st = bn_stats(K, raw, G, R, C, gamma, beta)
    dy = (torch.randn(G * R * C, device="cuda", generator=gen) * 1e-2).to(torch.bfloat16)
    refs = _refs(raw, dy, st, gamma, beta, G, R, C, ACT_LRELU)
    grp = torch.tensor(srcl, dtype=torch.int32, device="cuda")
    n = R * C
    d = dy.clone()
    dsum = torch.full((Fs * n,), NAN, device="cuda").to(torch.bfloat16)
    wg = {}
    if with_dout:
        B = CONFIGS[cfg]["B"]
        # a positive output-map gradient: y (LeakyReLU of the normalised rows, mean about 0.3) times it does not cancel, so
        # one chunk's or one group's share of the sum is well above the bound
        dout = (torch.rand(G * B * 4 * Ho * Ho, device="cuda", generator=gen) * 1e-2).to(torch.bfloat16)
        dw = torch.full((C * 16,), NAN, device="cuda")
        wg = dict(dout=dout, Ho=Ho, wpart=torch.empty(K.bn_wgrad_c1_partial_numel(G), device="cuda"), dw=dw)
    K.bn_bwd_group_sum(d, raw, st["mean"], st["invstd"], gamma, G, R, C, d, st["sdz"], st["sdzx"], st["scale"], st["shift"], grp, Fs,
                       dsum, **wg)
    torch.cuda.synchronize()
    w = _check_bwd(dict(dx=d.view(G, R, C), sdz=st["sdz"], sdzx=st["sdzx"]), refs, G, C, name)
    del refs
    dv = d.view(G, n)
    ws = 0.0
    for f in range(Fs):
        gs = [g for g in range(G) if srcl[g] == f]
        if not gs:
            assert torch.count_nonzero(dsum[f * n:(f + 1) * n].float()) == 0, f"{name}: source {f} has no group and must be zeros"
            continue
        ref = torch.zeros(n, dtype=torch.float64, device="cuda")
        mag = torch.zeros_like(ref)
        for g in gs:
            ref += dv[g].double()
            mag += dv[g].double().abs()
        ws = max(ws, bound_check(dsum[f * n:(f + 1) * n], ref, len(gs) * 2.0 ** -24 * mag + BETA[torch.bfloat16] * ref.abs(),
                                 f"{name} skip sum of source {f}"))
        del ref, mag
    msg = f"[bound] {name}: dx / sums {w:.3g}, skip sums {ws:.3g}"
    if with_dout:
        # y as bn_act stores it, then sum over rows of y[row, c] * tap(dout)[row, t]
        y = torch.empty_like(raw)
        K.bn_act(raw, y, st["scale"], st["shift"], G, R, C, ACT_LRELU)
        exact, absum = wgrad_c1_ref64(y, dout, Ho)
        assert (exact >= 0.3 * absum).all(), "the operands cancel: the check would not see a lost chunk"
        ratio = check_wgrad_c1(wg["dw"], exact, absum, R, C, f"{name} last-layer weight gradient")
        msg += f", dout weight gradient over {G * R} rows {ratio:.3g}"
    print(msg)


def test_bn_bwd_wgrad_c1_c2_enc0(K):
    """bn_bwd_wgrad_c1 at C2 enc0 (G = 30, R = 256 * 32 * 32 = 262144 rows per group: the chunk cap of 64 applies, 4096 rows per
    chunk; G R = 7.86M rows): the BatchNorm sums against float64, dx not written, and the first layer's weight gradient against
    a float64 sum over the stored dx (bn_bwd out of place) and the 1-channel input map."""
    c = CONFIGS["C2"]
    G, Ho, C = c["T"], c["W0"] // 2, 64
    R = c["B"] * Ho * Ho
    name = f"bn_bwd_wgrad_c1 C2 enc0 G={G} R={R}"
    raw, gamma, beta, gen = bn_inputs(G, R, C, seed=41)
    st = bn_stats(K, raw, G, R, C, gamma, beta)
    # dx is orthogonal to 1 (and to xhat) per group and channel, so against an arbitrary input map its weight gradient cancels.
    # Here dy has the sign s = +1 on even images and -1 on odd ones: dx then has about that sign (its mean terms are small),
    # and the input map is zero on the odd images, so the weight gradient sums |dx| * taps without cancelling
    nimg = G * c["B"]
    sgn = torch.where(torch.arange(nimg, device="cuda") % 2 == 0, 1.0, -1.0).view(nimg, 1)
    dy = (torch.rand(nimg, Ho * Ho * C, device="cuda", generator=gen) * sgn * 1e-3).to(torch.bfloat16).view(-1)
    cin = (torch.rand(nimg, 4 * Ho * Ho, device="cuda", generator=gen) * (sgn > 0)).to(torch.bfloat16).view(-1)
    refs = _refs(raw, dy, st, gamma, beta, G, R, C, ACT_LRELU)
    dx = torch.empty_like(dy)
    sdz0, sdzx0 = torch.empty(G * C, device="cuda"), torch.empty(G * C, device="cuda")
    K.bn_bwd(dy, raw, None, st["mean"], st["invstd"], gamma, G, R, C, ACT_LRELU, dx, sdz0, sdzx0, scale=st["scale"], shift=st["shift"])
    w = _check_bwd(dict(dx=dx.view(G, R, C), sdz=sdz0, sdzx=sdzx0), refs, G, C, "bn_bwd " + name)
    del refs
    d = dy.clone()
    wpart = torch.empty(K.bn_wgrad_c1_partial_numel(G), device="cuda")
    dw = torch.full((C * 16,), NAN, device="cuda")
    K.bn_bwd_wgrad_c1(d, raw, st["mean"], st["invstd"], gamma, G, R, st["sdz"], st["sdzx"], st["scale"], st["shift"], cin, Ho, wpart, dw)
    torch.cuda.synchronize()
    assert torch.equal(d, dy), "the weight-gradient pass must not write dx"
    assert torch.equal(st["sdz"], sdz0) and torch.equal(st["sdzx"], sdzx0)
    exact, absum = wgrad_c1_ref64(dx, cin, Ho)
    assert (exact.abs() >= 0.5 * absum).all(), "the operands cancel: the check would not see a lost chunk"
    ratio = check_wgrad_c1(dw, exact, absum, R, C, f"{name} weight gradient")
    print(f"[bound] {name}: dx / sums {w:.3g}, weight gradient over {G * R} rows {ratio:.3g}")


# ------------------------------------------------------------------ E. audit of real steps

class DcganAudit(AuditKernels):
    """AuditKernels for a dcgan step: its conv_gemm launches (kinds 0, 1, 2), the bf16 GEMMs only, and the skip sums of
    bn_bwd_group_sum.  The data-movement kernels of the 1- / 3-channel ends (im2col, col2im, convt_c1_loss, nchw_to_nhwc_dual)
    and the other BatchNorm entry points are not audited here: parts B-D and tests/test_bn_*_gpu.py check them at the step's
    shapes.  The fp32 LSTM / latent GEMMs: tests/test_lstm_scan_gpu.py, test_tc_schedule_gpu.py."""
    GEMM_FP32 = False
    GEMM_ACCUMULATE = False
    GEMM_PROBE_K = 1 << 12

    def conv_gemm(self, kind, a, b, c, N, H, W, Ck, Cn, Cm=0, ldb=None, ldc=None, bias=None, addend=None, grp_src=None,
                  imgs_per_group=0, accumulate=False, stat_partial=None, eval_scale=None, eval_shift=None, act=0):
        assert kind in (0, 1, 2) and H == W and eval_scale is None and not accumulate, f"unexpected conv_gemm launch kind {kind}"
        self._sync("conv_gemm", kind, a, b, c, N, H, W, Ck, Cn, Cm, ldb, ldc, bias, addend, grp_src, imgs_per_group, accumulate,
                   stat_partial, eval_scale, eval_shift, act)
        if kind == 1:
            s = conv_tiles(1, N, H, W, 0, Cn, Cm, self._sms)
            x = a.view(-1)[:N * H * H * Cm].view(N, H, H, Cm)
            g = b.view(-1)[:N * 4 * H * H * Cn].view(N, 2 * H, 2 * H, Cn)
            ref, absref = wgrad4_ref64(x, g, N, H, Cm, Cn)
            w = assert_within(c.view(-1)[:Cm * 16 * Cn].view(Cm, 16 * Cn), ref, absref, s.kb_per_split * 64 + 16 * s.splits,
                              torch.float32, quiet=True, name=f"audit kind 1 N={N} {H}x{H} {Cm}x{Cn}")
            # the step's gradients cancel over these K, so the bound above is loose: the same launch on the 0 / 1 pattern
            # of its operands must be exact
            x01, g01 = (x > 0).bfloat16(), (g > 0).bfloat16()
            probe = torch.full((Cm, 16 * Cn), NAN, device=c.device)
            super().conv_gemm(1, x01, g01, probe, N, H, H, 0, Cn, Cm=Cm)
            assert_exact(probe, wgrad4_ref64(x01, g01, N, H, Cm, Cn)[0], N * H * H, f"audit kind 1 N={N} {H}x{H} 0/1 probe")
            self._rec(f"conv_gemm kind 1 N={N} {H}x{H} {Cm}x{Cn}", ("k1",), w)
            return
        Ha, Ho = (2 * H, H) if kind == 0 else (H, 2 * H)
        x = a.view(-1)[:N * Ha * Ha * Ck].view(N, Ha, Ha, Ck)
        wt = b.view(-1)[:16 * Ck * Cn].view(*((Cn, 16 * Ck) if kind == 0 else (Ck, 16 * Cn)))
        out = c.view(-1)[:N * Ho * Ho * Cn].view(N, Ho, Ho, Cn)
        add, idx = self._addend(addend, grp_src, imgs_per_group, N, Ho, Cn) if addend is not None else (None, None)
        nm = f"conv_gemm kind {kind} N={N} {H}x{H} {Ck}->{Cn}"
        w = check_conv4_sums(out, kind, x, wt, N, H, Ck, Cn, bias, add, idx, name="audit " + nm)
        for i0 in sorted({0, N // 2, N - 1}):   # three images element-wise
            ref, absref = conv4_ref64_elem(kind, x[i0:i0 + 1], wt, H, Ck, Cn, bias, add[idx[i0:i0 + 1]] if add is not None else None)
            w = max(w, assert_within(out[i0:i0 + 1], ref, absref, 16 * Ck, out.dtype, quiet=True, name=f"audit {nm} image {i0}"))
        if stat_partial is not None:
            rows = cdiv(N * H * H, 128) * (4 if kind == 2 else 1)
            w = max(w, check_stat_rows(stat_partial.view(-1)[:rows * Cn * 2].view(rows, Cn, 2), out, kind, N, H, Cn, name="audit " + nm))
        self._rec(nm, conv_variant(kind, Cn, stat_partial is not None, addend.dtype if addend is not None else None, H, c.dtype), w)

    def bn_bwd_group_sum(self, dy, x, mean, invstd, gamma, G, R, C, dx, sum_dz, sum_dzx, scale, shift, grp_src, F, dx_sum,
                         dout=None, Ho=0, wpart=None, dw=None):
        self._sync("bn_bwd_group_sum", dy, x, mean, invstd, gamma, G, R, C, dx, sum_dz, sum_dzx, scale, shift, grp_src, F, dx_sum,
                   dout, Ho, wpart, dw)
        w = self._skip_sums(dx, dx_sum, grp_src.tolist()[:G], G, F, R * C, "bn_bwd_group_sum skip sums")
        self._rec(f"bn_bwd_group_sum G={G} R={R} C={C}", ("bn_bwd_group_sum", dout is not None), w)


AUDIT_CASES = [("dcgan64_bench_options", "C2", BENCH_OPT, 64), ("dcgan64_skip_lfs", "C2", SKIP_OPT, 64),
               ("dcgan128_bench_options", "C4", BENCH_OPT, 16)]


@pytest.mark.parametrize("case", AUDIT_CASES, ids=[c[0] for c in AUDIT_CASES])
def test_audit_dcgan_step(case):
    """One eager bf16 step at T = 30 with the audited launches checked as they run.  Every conv_gemm variant of the derived
    launch list must occur, every skip addend must be read through plan.skip_src, and losses, gradients and parameters must
    equal (torch.equal) the same step on plain CudaKernels with its concurrent lanes (so the side lanes share no scratch)."""
    name, cfg, optkw, B = case
    c, T = CONFIGS[cfg], 30

    def expect(plan):
        want = {L["variant"] for L in step_launches(T, B, plan.S, plan.nskip, c["nc"], c["W0"], plan.has_cpc) if L["op"] == "conv_gemm"}
        # the explicit last layer sums its skip columns with group_sum; a 1-channel one defers its weight gradient to `dout`
        want |= {("gemm", "bfloat16", "-"), ("bn_bwd_group_sum", False), ("add_indexed",), ("group_sum",)}
        if c["nc"] == 1:
            want.add(("bn_bwd_group_sum", True))
        assert conv_variant(2, 64, False, torch.bfloat16, 16) in want, "the derived list lost the 256-row addend launch"
        fwd = forward_launches(T, B, plan.S, plan.nskip, c["nc"], c["W0"])
        return want, [plan.skip_src] * sum(1 for L in fwd if L["op"] == "conv_gemm" and L["addend"] is not None)
    audit_step(TrainEngine, _cfg(c), optkw, T, B, DcganAudit("cuda"), expect, name)
