"""The fp32 dcgan training steps' kernel launches against float64 (P2PVG_PRECISION=fp32, the parity mode), at the shapes of
the C2 benchmark configuration (dcgan_64, 1 channel, T = 30, B = 256) and of C4 (dcgan_128, 3 channels, T = 30, B = 64).

In fp32 the step takes none of the bf16 fusions: every 4x4 convolution is im2col -> gemm_simt, every transposed one
gemm_simt -> col2im, the weight gradients are CUDA-core GEMMs over every pixel (split-K), BatchNorm runs as separate passes
and the decoder's skip gradient is a group_sum of the full dcol buffer.  At C2 the im2col / dcol buffers hold 2.01e9 elements
(93.75 % of 2^31), so the 64-bit index paths are exercised here and nowhere else.

  A. the fp32 launch list tests/dcgan_ref.py derives (precision "fp32") against what one eager fp32 step records, at exactly
     C2 and C4; the step's peak device memory is printed (DESIGN.md §1 lists it);
  B. every distinct GEMM of the C2 / C4 lists at its shape and pitches on gemm_simt, against float64 (launch_audit
     gemm32_at_shape), the weight gradients exact on 0 / 1 operands;
  C. im2col bit-exact over its full buffers, col2im with the skip half (several groups sharing a source, one source read by
     no group) and the bias at every decoder stage and on the encoder's data-gradient path, and group_sum of C2 dec2's dcol;
  D. BatchNorm on fp32 rows at every BatchNorm launch shape of the C2 / C4 lists: bn_fwd_stats, bn_act, bn_bwd (in place,
     LeakyReLU slope from scale / shift, and the tanh encoder output) and bn_param_grad against float64;
  E. audited fp32 steps at T = 30 (dcgan_64 B = 128 with the bench options and with a skip plan, dcgan_128 B = 32): every
     GEMM, im2col, col2im, group_sum, add_indexed and BatchNorm entry point checked against float64 as it runs, serially,
     bit-identical to the plain step and to its graph replay;
  F. the whole fp32 step at the audit batches (T = 30) against the float64 oracle on the device (the oracle's step took
     3.7 s at dcgan_64 B = 128 and 3.3 s at dcgan_128 B = 32 on an H100 80GB HBM3 at 700 W; the time is printed).
"""
import time

import numpy as np
import pytest
import torch

from oracle import p2p_oracle as O
from p2pvg_b200._lib import CudaKernels
from p2pvg_b200.engine import StepPlan, TrainEngine
from tests.dcgan_ref import ACT_LRELU, ACT_TANH, check_col2im, check_im2col, step_launches
from tests.launch_audit import K, memory_per_test  # noqa: F401  (fixtures)
from tests.launch_audit import (BENCH_OPT, NAN, SENTINEL, SKIP_OPT, SimtAudit, assert_equal_steps, assert_serial, audit_step,
                                bn_bwd_refs, bn_inputs, bn_stats, check_bn_bwd, check_bn_stats, check_group_sum, gemm32_at_shape,
                                gemm_ws_bytes, kernel_for, recorded_fp32_step, release, run_step, skip_seed, step_inputs)
from tests.ref64 import bound_check

pytestmark = pytest.mark.gpu

CONFIGS = {"C2": dict(T=30, B=256, nc=1, W0=64), "C4": dict(T=30, B=64, nc=3, W0=128)}


def _cfg(c):
    return dict(g_dim=128, z_dim=10, rnn_size=256, channels=c["nc"], image_width=c["W0"], predictor_rnn_layers=2,
                posterior_rnn_layers=1, prior_rnn_layers=1)


def launches(name, B=None):
    c = CONFIGS[name]
    p = StepPlan(c["T"], np.zeros(c["T"] - 1), O.default_opt(**BENCH_OPT))
    return step_launches(c["T"], B or c["B"], p.S, p.nskip, c["nc"], c["W0"], p.has_cpc, "fp32")


# ------------------------------------------------------------------ A. the launch lists

@pytest.mark.parametrize("name", list(CONFIGS))
def test_fp32_launch_list_matches_an_eager_step(name):
    """The derived fp32 list equals, call for call and in order, the backbone launches of one eager fp32 step at the
    configuration's exact shape; the step runs serially and has no implicit-GEMM or fused BatchNorm launch."""
    c = CONFIGS[name]
    plan, got, peak = recorded_fp32_step(TrainEngine, _cfg(c), BENCH_OPT, c["T"], c["B"])
    L = launches(name)
    want = [e["key"] for e in L]
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"{name}: launch {i} is {g}, the derived list says {w} ({L[i]['name']})"
    assert len(got) == len(want), f"{name}: {len(got)} launches recorded, {len(want)} derived"
    print(f"[list] {name} fp32: {len(got)} launches, in order; peak device memory of the step {peak:.2f} GiB")


# ------------------------------------------------------------------ B. every distinct GEMM at its shape

def _distinct_gemms():
    seen, out = set(), []
    for n in CONFIGS:
        for e in launches(n):
            if e["op"] == "gemm" and e["key"] not in seen:
                seen.add(e["key"])
                out.append((n, e))
    return out


GEMMS = _distinct_gemms()


@pytest.mark.parametrize("cfg,e", GEMMS, ids=[f"{n}-{e['name'].replace(' ', '_')}-{e['M']}x{e['N']}x{e['K']}" for n, e in GEMMS])
def test_fp32_gemm_at_launch_shape(K, cfg, e):
    kern, _ = gemm32_at_shape(K, e, e["M"] * 7 + e["N"] * 3 + e["K"], cfg)
    if e["a_mn"] and e["K"] >= 1 << 20:
        assert not isinstance(kern, str), "a weight gradient over every pixel runs unsplit"


def test_fp32_gemm_coverage():
    """The distinct GEMMs include the split schedules of the issue's table: C2 enc0 64 x 16 over 7.86M pixels (296 splits),
    enc1 / dec2 128 x 1024 over 1.97M (10 splits), and the 2.01e9-element col operands of C2 enc1 and dec2."""
    geo = {(n, e["M"], e["N"], e["K"]) for n, e in GEMMS}
    assert ("C2", 64, 16, 7680 * 1024) in geo and ("C2", 128, 1024, 7680 * 256) in geo
    assert ("C2", 7680 * 256, 128, 1024) in geo                    # enc1: col [1.97M, 1024]
    assert ("C2", 7680 * 256, 1024, 128) in geo                    # dec2.D: colD [1.97M, 1024]


# ------------------------------------------------------------------ C. the lowering kernels at their shapes

def _im2col_shapes():
    seen = []
    for n in CONFIGS:
        for e in launches(n):
            if e["op"] == "im2col" and (n,) + e["args"] not in seen:
                seen.append((n,) + e["args"])
    return seen


IM2COL = _im2col_shapes()


@pytest.mark.parametrize("case", IM2COL, ids=[f"{c[0]}-N{c[1]}_{c[2]}x{c[2]}x{c[3]}" for c in IM2COL])
def test_im2col_full_buffer(K, case):
    """im2col over the whole launch (C2: 2.01e9 output elements), bit-exact against the gather, nothing written past the end."""
    cfg, N, H, C = case
    x = torch.randn(N * H * H * C, device="cuda")
    n = N * (H // 2) ** 2 * 16 * C
    col = torch.full((n + 64,), SENTINEL, device="cuda")
    K.im2col(x, col, N, H, H, C)
    torch.cuda.synchronize()
    assert (col[n:] == SENTINEL).all(), "im2col wrote past its output"
    check_im2col(x, col, N, H, C, f"{cfg} im2col")
    print(f"[exact] {cfg} im2col N={N} {H}x{H}x{C}: {n} elements ({n / 2 ** 31:.4f} x 2^31), bit-exact")


def _col2im_shapes():
    seen = []
    for n in CONFIGS:
        for e in launches(n):
            if e["op"] == "col2im" and (n,) + e["args"] not in seen:
                seen.append((n,) + e["args"])
    return seen


COL2IM = _col2im_shapes()


@pytest.mark.parametrize("case", COL2IM, ids=[f"{c[0]}-N{c[1]}_{c[2]}x{c[2]}x{c[3]}{'_skip' if c[5] else ''}" for c in COL2IM])
def test_col2im_at_launch_shape(K, case):
    """col2im at every decoder stage (col2 + grp_src + bias: four sources, two groups sharing one, one source read by no
    group) and on the encoder's data-gradient path, over every output element, against float64."""
    cfg, N, Hi, C, bias_, skip, ipg = case
    gen = torch.Generator(device="cuda").manual_seed(N + Hi + C)
    col = torch.randn(N * Hi * Hi * 16 * C, device="cuda", generator=gen)
    bias = torch.randn(C, device="cuda", generator=gen) if bias_ else None
    col2 = grp = None
    if skip:
        G = N // ipg
        srcl = [(0, 1, 3)[(g * 5 // G + g % 2) % 3] for g in range(G)]   # source 2 is read by no group
        assert 2 not in srcl and len(set(srcl)) == 3
        grp = torch.tensor(srcl, dtype=torch.int32, device="cuda")
        col2 = torch.randn(4 * ipg * Hi * Hi * 16 * C, device="cuda", generator=gen)
    n = N * 4 * Hi * Hi * C
    y = torch.full((n + 64,), SENTINEL, device="cuda")
    y[:n] = NAN
    K.col2im(col, y, N, Hi, Hi, C, bias=bias, col2=col2, grp_src=grp, imgs_per_group=ipg)
    torch.cuda.synchronize()
    assert (y[n:] == SENTINEL).all(), "col2im wrote past its output"
    w = check_col2im(y, col, N, Hi, C, bias, col2, grp, ipg, f"{cfg} col2im")
    print(f"[bound] {cfg} col2im N={N} {Hi}x{Hi}->{2 * Hi}x{2 * Hi}x{C} skip={skip}: worst error/bound {w:.3g}")


def test_group_sum_c2_dec2_dcol(K):
    """group_sum of C2 dec2's dcol (G = 29 groups of 256 x 16 x 16 x 16 x 64 = 67M floats) into four sources, one read by no
    group, against float64."""
    L = [e for e in launches("C2") if e["op"] == "group_sum" and e["name"] == "dec2 dcol skip sum"]
    G, _, n = L[0]["args"]
    assert G == 29 and n == 256 * 16 * 16 * 16 * 64
    srcl = [(0, 1, 3)[(g * 5 // G + g % 2) % 3] for g in range(G)]
    inp = torch.randn(G * n, device="cuda")
    out = torch.full((4 * n + 64,), SENTINEL, device="cuda")
    K.group_sum(inp, out, torch.tensor(srcl, dtype=torch.int32, device="cuda"), G, 4, n)
    torch.cuda.synchronize()
    assert (out[4 * n:] == SENTINEL).all()
    w = check_group_sum(inp, out, srcl, G, 4, n, "C2 dec2 group_sum")
    print(f"[bound] C2 dec2 group_sum G={G} n={n}: worst error/bound {w:.3g}")


# ------------------------------------------------------------------ D. BatchNorm in fp32 at the launch shapes

def _bn_shapes(op):
    out = []
    for n in CONFIGS:
        for e in launches(n):
            if e["op"] == op and (n,) + e["args"] not in [o[:5] for o in out]:
                out.append((n,) + e["args"] + (e["name"],))
    return out


BN_FWD, BN_BWD = _bn_shapes("bn_act"), _bn_shapes("bn_bwd")


@pytest.mark.parametrize("case", BN_FWD, ids=[f"{c[0]}-{c[5]}-G{c[1]}_R{c[2]}_C{c[3]}" for c in BN_FWD])
def test_fp32_bn_forward_at_launch_shape(K, case):
    """bn_fwd_stats on fp32 rows (every BatchNorm layer of the fp32 step: none has fused statistics) within the float64 bound,
    and bn_act: y = act(fmaf(x, scale, shift)) within one fp32 rounding of each (tanh: a few ulp more)."""
    cfg, G, R, C, act, nm = case
    name = f"{cfg} {nm} fp32 G={G} R={R} C={C}"
    raw, gamma_, beta, _ = bn_inputs(G, R, C, seed=G * 7 + C + 1, dt=torch.float32)
    st = bn_stats(K, raw, G, R, C, gamma_, beta)
    w = check_bn_stats(st, raw, G, R, C, gamma_, beta, f"bn_fwd_stats {name}")
    y = torch.full((G * R * C + 64,), SENTINEL, device="cuda")
    y[:G * R * C] = NAN
    K.bn_act(raw, y, st["scale"], st["shift"], G, R, C, act)
    torch.cuda.synchronize()
    assert (y[G * R * C:] == SENTINEL).all(), f"bn_act {name} wrote past its output"
    x, yv = raw.view(G, R, C), y[:G * R * C].view(G, R, C)
    sc, sh = st["scale"].view(G, 1, C).double(), st["shift"].view(G, 1, C).double()
    wa = 0.0
    for g in range(G):
        pre = x[g].double() * sc[g] + sh[g]
        mag = (x[g].double() * sc[g]).abs() + sh[g].abs()
        ref = torch.where(pre > 0, pre, 0.2 * pre) if act == ACT_LRELU else torch.tanh(pre)
        bnd = 2.0 ** -23 * mag + (2.0 ** -23 * ref.abs() if act == ACT_LRELU else 2.0 ** -21)
        wa = max(wa, bound_check(yv[g], ref, bnd, f"bn_act {name} group {g}"))
    print(f"[bound] {name}: stats {w:.3g}, bn_act {wa:.3g}")


@pytest.mark.parametrize("case", BN_BWD, ids=[f"{c[0]}-{c[5]}-G{c[1]}_R{c[2]}_C{c[3]}" for c in BN_BWD])
def test_fp32_bn_bwd_at_launch_shape(K, case):
    """bn_bwd on fp32 rows as the fp32 step calls it (in place; LeakyReLU: y = None and the slope from scale / shift; tanh: y
    given) and bn_param_grad, against float64 per group: the sums within ALPHA_BN of their magnitudes, dx within that and one
    fp32 rounding."""
    cfg, G, R, C, act, nm = case
    name = f"bn_bwd {cfg} {nm} fp32 G={G} R={R} C={C}"
    raw, gamma_, beta, gen = bn_inputs(G, R, C, seed=G * 11 + C + 1, dt=torch.float32)
    st = bn_stats(K, raw, G, R, C, gamma_, beta)
    x = raw.view(G, R, C)
    dy = torch.empty_like(raw)
    for g in range(G):   # dy correlated with xhat, so that the xhat term of dx carries weight
        xg = x[g].double()
        xh = (xg - xg.mean(0)) / torch.sqrt(xg.var(0, unbiased=False) + 1e-5)
        dy.view(G, R, C)[g] = (0.5 * xh + torch.randn(R, C, device="cuda", dtype=torch.float64, generator=gen)).float()
    y = None
    if act == ACT_TANH:
        y = torch.empty_like(raw)
        K.bn_act(raw, y, st["scale"], st["shift"], G, R, C, ACT_TANH)
    refs = bn_bwd_refs(raw, dy, st, gamma_, beta, G, R, C, act, y)
    d = dy.clone()
    if act == ACT_LRELU:
        K.bn_bwd(d, raw, None, st["mean"], st["invstd"], gamma_, G, R, C, act, d, st["sdz"], st["sdzx"], scale=st["scale"], shift=st["shift"])
    else:
        K.bn_bwd(d, raw, y, st["mean"], st["invstd"], gamma_, G, R, C, act, d, st["sdz"], st["sdzx"])
    dg, db = torch.full((C,), NAN, device="cuda"), torch.full((C,), NAN, device="cuda")
    K.bn_param_grad(st["sdz"], st["sdzx"], G, C, dg, db)
    torch.cuda.synchronize()
    w = check_bn_bwd(dict(dx=d.view(G, R, C), sdz=st["sdz"], sdzx=st["sdzx"], dgamma=dg, dbeta=db), refs, G, C, name,
                     dx_dtype=torch.float32)
    print(f"[bound] {name}: worst error/bound {w:.3g}")


# ------------------------------------------------------------------ E. audited steps

class DcganFp32Audit(SimtAudit):
    """The fp32 dcgan step: GEMMs on the SIMT bound, im2col / col2im, group_sum / add_indexed and the BatchNorm forward."""
    REPORT_GEMMS_ONLY = True

    def im2col(self, x, col, N, H, W, C):
        self._sync("im2col", x, col, N, H, W, C)
        check_im2col(x, col, N, H, C, "audit")
        self._rec(f"im2col N={N} {H}x{W}x{C}", ("im2col",), 0.0)

    def col2im(self, col, y, N, Hi, Wi, C, bias=None, col2=None, grp_src=None, imgs_per_group=0, accumulate=False):
        assert not accumulate
        self._sync("col2im", col, y, N, Hi, Wi, C, bias, col2, grp_src, imgs_per_group, accumulate)
        if col2 is not None:
            self.skip_reads.append(grp_src.tolist()[:N // imgs_per_group])
        w = check_col2im(y, col, N, Hi, C, bias, col2, grp_src, imgs_per_group, "audit")
        self._rec(f"col2im N={N} {Hi}x{Wi}x{C}", ("col2im", bias is not None, col2 is not None), w)


# The audited step runs at half the recorded step's batch: beside the step's own buffers (58.9 GiB at C2 B 256, 62.0 GiB at
# C4 B 64) it holds the plain step's results, fp32 0 / 1 copies of both operands of every long GEMM it probes (at C2 B 256
# the enc1 weight gradient's col operand alone is 7.5 GiB) and float64 reference chunks: at B 128 / 32 the audit peaks at
# 31.8 - 37.7 GiB (H100 80GB), about twice the 15.8 - 18.2 GiB it took at B 64 / 16.
AUDIT = [("dcgan64_bench_options", "C2", BENCH_OPT, 128), ("dcgan64_skip_lfs", "C2", SKIP_OPT, 128),
         ("dcgan128_bench_options", "C4", BENCH_OPT, 32)]


@pytest.mark.parametrize("case", AUDIT, ids=[c[0] for c in AUDIT])
def test_audit_fp32_dcgan_step(case):
    """One eager fp32 step at T = 30 with the audited launches checked as they run: every GEMM and lowering variant of the
    derived list occurs, every skip half is read through plan.skip_src, and losses, gradients and parameters equal the plain
    serial step and its graph replay bit for bit."""
    name, cfg, optkw, B = case
    c, T = CONFIGS[cfg], 30
    audit = DcganFp32Audit("cuda")

    def expect(plan):
        L = step_launches(T, B, plan.S, plan.nskip, c["nc"], c["W0"], plan.has_cpc, "fp32")
        want = {("im2col",), ("group_sum",), ("add_indexed",), ("bn_fwd_stats",), ("bn_act", 1), ("bn_act", 2), ("bn_bwd", 1),
                ("bn_bwd", 2), ("bn_param_grad",)}
        for e in L:
            if e["op"] == "gemm":
                kern = kernel_for(e["M"], e["N"], e["K"], e["a_mn"], e["b_mn"], e["lda"], e["ldb"], 0, 0, False, gemm_ws_bytes(audit))
                want.add(("gemm", kern if isinstance(kern, str) else kern[0], e["a_mn"], e["b_mn"], e["bias"]))
            elif e["op"] == "col2im":
                want.add(("col2im", e["args"][3], e["args"][4]))
        assert ("gemm", "simt-splitK", True, True, False) in want and ("col2im", True, True) in want
        return want, [plan.skip_src] * sum(1 for e in L if e["op"] == "col2im" and e["args"][4])

    plan, plain = audit_step(TrainEngine, _cfg(c), optkw, T, B, audit, expect, f"{name} fp32", act_dtype=torch.float32)
    np_seed = skip_seed(T) if optkw.get("skip_prob") else 0
    _, graph = run_step(TrainEngine, _cfg(c), optkw, CudaKernels("cuda"), T, B, np_seed, use_graph=True, act_dtype=torch.float32,
                        prepare=assert_serial)
    assert_equal_steps(plain, graph, f"{name}: graph replay vs eager")


# ------------------------------------------------------------------ F. against the float64 oracle

ORACLE = [(a[0].split("_")[0], a[1], 30, a[3]) for a in AUDIT if a[2] is BENCH_OPT]   # the audit batches


def _bn_cancelled(m, k):
    """Conv / ConvT biases feeding a training-mode BatchNorm: exactly-zero true gradient (test_step_gpu.py)."""
    if m == "encoder":
        return k.endswith(".0.bias")
    if m == "decoder":
        return (k.endswith(".0.bias") and not k.startswith(("upc5.0", "upc6.0"))) or k == "upc1.0.bias"
    return False


@pytest.mark.parametrize("case", ORACLE, ids=[c[0] for c in ORACLE])
def test_fp32_step_vs_float64_oracle(case):
    """Losses to rtol 1e-4 and every gradient to cosine >= 1 - 1e-5 against the float64 oracle (DESIGN.md's fp32 thresholds),
    the BatchNorm-cancelled biases exempt."""
    name, cfg, T, B = case
    c = CONFIGS[cfg]
    opt, probs, plan, x, eps = step_inputs(_cfg(c), BENCH_OPT, T, B, 0)
    state = {m: {k: v.cuda() for k, v in sd.items()} for m, sd in O.build_state(_cfg(c), seed=1, dtype=torch.float64).items()}
    adam = {m: O.new_adam_state(state[m]) for m in O.MODULES}
    t0 = time.time()
    ref = O.train_step(state, adam, x.double().cuda(), opt, c["W0"], eps.double().cuda(), probs, mode="A")
    torch.cuda.synchronize()
    print(f"[oracle] float64 {name} T={T} B={B} step on the device: {time.time() - t0:.1f} s")
    del state, adam
    release()
    eng = TrainEngine(O.build_state(_cfg(c), seed=1), _cfg(c), opt, CudaKernels("cuda"), act_dtype=torch.float32)
    got = eng.step(x.cuda(), probs=probs, eps=eps.cuda())
    torch.cuda.synchronize()
    np.testing.assert_allclose(got, np.array(ref["losses"]), rtol=1e-4, atol=1e-7, err_msg=name)
    worst = []
    for m in O.MODULES:
        for k, gref in ref["grads"][m].items():
            if _bn_cancelled(m, k):
                continue
            g = eng.arena[m].g[k].detach().double()
            cos = torch.nn.functional.cosine_similarity(g.flatten(), gref.flatten().to(g.device), dim=0).item()
            worst.append((cos, f"{m}.{k}"))
    worst.sort()
    print(f"[oracle] {name}: losses {got} vs {np.array(ref['losses'])}; worst cosines "
          + ", ".join(f"{n} {1 - cs:.2e}" for cs, n in worst[:5]))
    bad = [f"{n}: cosine {cs:.8f}" for cs, n in worst if cs < 1 - 1e-5]
    assert not bad, "\n".join(bad)
