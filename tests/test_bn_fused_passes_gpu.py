"""The bf16 BatchNorm-backward passes that also do the next launch's work on the tensors they stream:

- p2pvg_bn_bwd_group_sum writes the decoder's skip-frame sums of dx (what p2pvg_group_sum would read back), and with
  `dout` its reduce pass also sums the weight gradient of a following 64 -> 1 transposed convolution;
- p2pvg_bn_bwd_wgrad_c1 writes the weight gradient of a 1-channel first encoder layer instead of its dx.

Each is checked at the kernel level (against p2pvg_bn_bwd + p2pvg_group_sum, and against a float64 sum over the same bf16
operands), and through whole eager dcgan_64 steps against the engine's launch sequence without them: a kernel backend that
hides the two entry points makes TrainEngine take the unfused sequence.  Everything but the first encoder layer's weight
gradient and the half of the last decoder layer's that reads the previous stage (fp32 sums in another order) must be
bit-identical, and the steps deterministic, eager or replayed from a graph."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import p2p_oracle as O
from p2pvg_b200.engine import StepPlan

pytestmark = pytest.mark.gpu

ACT_LRELU = 1
FUSED = ("bn_bwd_group_sum", "bn_bwd_wgrad_c1")


@pytest.fixture(scope="module")
def K():
    from p2pvg_b200._lib import CudaKernels
    return CudaKernels("cuda")


def _unfused_kernels():
    from p2pvg_b200._lib import CudaKernels

    class UnfusedKernels(CudaKernels):
        """CudaKernels without the fused BatchNorm passes: the engine then launches bn_bwd, group_sum and the GEMMs."""

        def __getattribute__(self, name):
            if name in FUSED:
                raise AttributeError(name)
            return super().__getattribute__(name)

    return UnfusedKernels("cuda")


def _bn_state(G, R, C, seed):
    """Forward statistics of a random pre-activation, the bf16 tensors and a seeded upstream gradient."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    raw = (torch.randn(G * R * C, device="cuda", generator=gen) * 1.5 + 0.3).to(torch.bfloat16)
    dy = (torch.randn(G * R * C, device="cuda", generator=gen) * 1e-3).to(torch.bfloat16)
    gamma = torch.rand(C, device="cuda", generator=gen) + 0.5
    beta = torch.randn(C, device="cuda", generator=gen) * 0.1
    st = {k: torch.empty(G * C, device="cuda") for k in ("mean", "invstd", "varu", "scale", "shift", "sdz", "sdzx")}
    return raw, dy, gamma, beta, st


def _fwd(K, raw, G, R, C, gamma, beta, st):
    K.bn_fwd_stats(raw, G, R, C, gamma, beta, st["mean"], st["invstd"], st["varu"], st["scale"], st["shift"])


GS_CASES = [
    # (G, R, C, grp_src, F): one source; several sources in runs; sources out of order; a source no group maps to (F = 4,
    # source 2 unused); ragged row counts that end mid-visit and mid-chunk
    (29, 4096, 64, [0] * 29, 1),
    (7, 1000, 64, [0, 0, 1, 1, 1, 2, 2], 3),
    (6, 777, 128, [1, 0, 1, 3, 0, 3], 4),
    (5, 64 * 4 + 3, 256, [0, 1, 2, 3, 4], 5),
    (3, 50, 512, [0, 0, 0], 2),
]


@pytest.mark.parametrize("case", GS_CASES, ids=[f"G{c[0]}_R{c[1]}_C{c[2]}_F{c[4]}" for c in GS_CASES])
def test_group_sum_pass_equals_bn_bwd_then_group_sum(K, case):
    G, R, C, src, Fs = case
    raw, dy, gamma, beta, st = _bn_state(G, R, C, seed=G * 131 + C)
    _fwd(K, raw, G, R, C, gamma, beta, st)
    grp = torch.tensor(src, dtype=torch.int32, device="cuda")
    n = R * C
    dx_ref, sdz_ref, sdzx_ref = torch.empty_like(dy), torch.empty(G * C, device="cuda"), torch.empty(G * C, device="cuda")
    K.bn_bwd(dy, raw, None, st["mean"], st["invstd"], gamma, G, R, C, ACT_LRELU, dx_ref, sdz_ref, sdzx_ref, scale=st["scale"],
             shift=st["shift"])
    sum_ref = torch.full((Fs * n,), float("nan"), device="cuda").to(torch.bfloat16)
    K.group_sum(dx_ref, sum_ref, grp, G, Fs, n)
    d = dy.clone()   # in place, as the engine calls it
    sdz, sdzx = torch.empty(G * C, device="cuda"), torch.empty(G * C, device="cuda")
    dsum = torch.full((Fs * n,), float("nan"), device="cuda").to(torch.bfloat16)
    K.bn_bwd_group_sum(d, raw, st["mean"], st["invstd"], gamma, G, R, C, d, sdz, sdzx, st["scale"], st["shift"], grp, Fs, dsum)
    torch.cuda.synchronize()
    assert torch.equal(sdz, sdz_ref) and torch.equal(sdzx, sdzx_ref)
    assert torch.equal(d, dx_ref), "dx differs from bn_bwd"
    assert torch.equal(dsum, sum_ref), "skip sums differ from group_sum of the stored dx"
    for f in set(range(Fs)) - set(src):
        assert torch.count_nonzero(dsum[f * n:(f + 1) * n].float()) == 0, f"source {f} has no group and must be zeros"


RW_CASES = [(29, 8, 32, [0] * 29, 1), (3, 3, 16, [1, 0, 1], 2), (2, 1, 4, [0, 0], 1)]   # (G, images per group, Ho, grp_src, F)


@pytest.mark.parametrize("case", RW_CASES, ids=[f"G{c[0]}_B{c[1]}_Ho{c[2]}_F{c[4]}" for c in RW_CASES])
def test_group_sum_pass_with_transposed_conv_wgrad(K, case):
    """The reduce pass that also sums the weight gradient of a ConvTranspose2d(64, 1, 4, 2, 1) reading y: every other output
    bit-identical to the pass without it, dw against a float64 sum over y (as bn_act stores it) and the output-map gradient."""
    G, B, Ho, src, Fs = case
    C, R = 64, B * Ho * Ho
    raw, dy, gamma, beta, st = _bn_state(G, R, C, seed=11 * G + Ho)
    _fwd(K, raw, G, R, C, gamma, beta, st)
    y = torch.empty_like(raw)
    K.bn_act(raw, y, st["scale"], st["shift"], G, R, C, ACT_LRELU)
    gen = torch.Generator(device="cuda").manual_seed(4)
    dout = (torch.randn(G * B * 4 * Ho * Ho, device="cuda", generator=gen) * 1e-2).to(torch.bfloat16)
    grp = torch.tensor(src, dtype=torch.int32, device="cuda")
    outs = []
    for with_w in (False, True):
        d = dy.clone()
        sdz, sdzx = torch.empty(G * C, device="cuda"), torch.empty(G * C, device="cuda")
        dsum = torch.empty(Fs * R * C, device="cuda", dtype=torch.bfloat16)
        dw = torch.full((C * 16,), float("nan"), device="cuda")
        wg = dict(dout=dout, Ho=Ho, wpart=torch.empty(K.bn_wgrad_c1_partial_numel(G), device="cuda"), dw=dw) if with_w else {}
        K.bn_bwd_group_sum(d, raw, st["mean"], st["invstd"], gamma, G, R, C, d, sdz, sdzx, st["scale"], st["shift"], grp, Fs, dsum, **wg)
        outs.append((d, sdz, sdzx, dsum, dw))
    torch.cuda.synchronize()
    for a, b in zip(outs[0][:4], outs[1][:4]):
        assert torch.equal(a, b), "the weight-gradient reduce changed dx, the BatchNorm sums or the skip sums"
    exact, absum = _wgrad64(y, dout, Ho)
    err = (outs[1][4].view(C, 16).double() - exact).abs()
    ratio = (err / _fp32_bound(absum, R)).max().item()
    print(f"[reduce wgrad] G={G} B={B} Ho={Ho}: worst error / fp32 bound {ratio:.3g}")
    assert ratio <= 1.0


def _taps64(cin, Ho):
    """float64 [N, 16, Ho*Ho] 4x4 / stride-2 / pad-1 patches of the 1-channel map cin [N, 2Ho, 2Ho], tap = kh*4 + kw."""
    N = cin.numel() // (4 * Ho * Ho)
    return F.unfold(cin.view(N, 1, 2 * Ho, 2 * Ho).double(), kernel_size=4, stride=2, padding=1)


def _wgrad64(dx, cin, Ho, C=64):
    """float64 sum over rows of bf16 dx[row, c] * tap[row, t], and the same sum of absolute products (the error scale)."""
    N = cin.numel() // (4 * Ho * Ho)
    d = dx.view(N, Ho * Ho, C).double()
    t = _taps64(cin, Ho)
    return torch.einsum("npc,ntp->ct", d, t), torch.einsum("npc,ntp->ct", d.abs(), t.abs())


def _fp32_bound(absum, rows):
    """|fp32 sum - exact| <= rows * 2^-24 * sum |products| (any order of at most `rows` fp32 additions per partial)."""
    return rows * 2.0 ** -24 * absum + 1e-30


WG_CASES = [(30, 8, 32), (3, 5, 32), (2, 3, 64), (1, 1, 4)]   # (G, images per group, Ho)


@pytest.mark.parametrize("case", WG_CASES, ids=[f"G{c[0]}_B{c[1]}_Ho{c[2]}" for c in WG_CASES])
def test_wgrad_c1_pass_against_float64(K, case):
    G, B, Ho = case
    C, R = 64, B * Ho * Ho
    raw, dy, gamma, beta, st = _bn_state(G, R, C, seed=7 * G + Ho)
    _fwd(K, raw, G, R, C, gamma, beta, st)
    gen = torch.Generator(device="cuda").manual_seed(3)
    cin = torch.rand(G * B * 4 * Ho * Ho, device="cuda", generator=gen).to(torch.bfloat16)
    dx_ref, sdz_ref, sdzx_ref = torch.empty_like(dy), torch.empty(G * C, device="cuda"), torch.empty(G * C, device="cuda")
    K.bn_bwd(dy, raw, None, st["mean"], st["invstd"], gamma, G, R, C, ACT_LRELU, dx_ref, sdz_ref, sdzx_ref, scale=st["scale"],
             shift=st["shift"])
    d = dy.clone()
    sdz, sdzx = torch.empty(G * C, device="cuda"), torch.empty(G * C, device="cuda")
    wpart = torch.empty(K.bn_wgrad_c1_partial_numel(G), device="cuda")
    dw = torch.full((C * 16,), float("nan"), device="cuda")
    K.bn_bwd_wgrad_c1(d, raw, st["mean"], st["invstd"], gamma, G, R, sdz, sdzx, st["scale"], st["shift"], cin, Ho, wpart, dw)
    dw2 = torch.full_like(dw, float("nan"))
    K.bn_bwd_wgrad_c1(d, raw, st["mean"], st["invstd"], gamma, G, R, sdz, sdzx, st["scale"], st["shift"], cin, Ho, wpart, dw2)
    torch.cuda.synchronize()
    assert torch.equal(d, dy), "the weight-gradient pass must not write dx"
    assert torch.equal(sdz, sdz_ref) and torch.equal(sdzx, sdzx_ref)
    assert torch.equal(dw, dw2), "not deterministic"
    exact, absum = _wgrad64(dx_ref, cin, Ho)
    err = (dw.view(C, 16).double() - exact).abs()
    ratio = (err / _fp32_bound(absum, R)).max().item()
    print(f"[wgrad_c1] G={G} B={B} Ho={Ho}: worst error / fp32 bound {ratio:.3g}, worst relative {(err.max() / exact.abs().max()).item():.3g}")
    assert ratio <= 1.0


def test_wgrad_c1_rejects_bad_arguments(K):
    from p2pvg_b200._lib import KernelError
    G, B, Ho = 2, 1, 4
    R = B * Ho * Ho
    raw, dy, gamma, beta, st = _bn_state(G, R, 64, seed=1)
    cin = torch.zeros(G * B * 4 * Ho * Ho, device="cuda", dtype=torch.bfloat16)
    dw = torch.empty(64 * 16, device="cuda")
    args = (dy, raw, st["mean"], st["invstd"], gamma, G, R, st["sdz"], st["sdzx"], st["scale"], st["shift"], cin)
    with pytest.raises(KernelError, match="partial buffer too small"):
        K.bn_bwd_wgrad_c1(*args, Ho, torch.empty(16, device="cuda"), dw)
    with pytest.raises(KernelError, match="whole number"):
        K.bn_bwd_wgrad_c1(*args, 3, torch.empty(K.bn_wgrad_c1_partial_numel(G), device="cuda"), dw)


# ------------------------------------------------------------------ whole steps
CFG = dict(g_dim=128, z_dim=10, rnn_size=256, channels=1, image_width=64, predictor_rnn_layers=2, posterior_rnn_layers=1,
           prior_rnn_layers=1)
BENCH_OPT = dict(skip_prob=0.0, n_past=1, last_frame_skip=False)
SKIP_OPT = dict(skip_prob=0.5, n_past=2, last_frame_skip=True)
T, B = 30, 32
ENC0_W = ("encoder", "c1.main.0.weight")
DEC_LAST_W = ("decoder", "upc5.0.weight")   # [128, 1, 4, 4]: input channels 0..63 read the previous stage, 64..127 the skip


def _skip_seed():
    """The first probability seed whose skip_prob 0.5 / n_past 2 / last-frame-skip plan has at least three skip sources and a
    source frame that no executed step reads (the frame a skipped step would have used)."""
    opt = O.default_opt(**SKIP_OPT)
    for seed in range(200):
        p = StepPlan(T, np.random.RandomState(seed).uniform(0, 1, T - 1), opt)
        if len(set(p.skip_src[:p.S])) >= 3 and set(range(p.nskip)) - set(p.skip_src[:p.S]):
            return seed
    raise AssertionError("no seed gives such a plan")


def _engine(kernels, optkw):
    from p2pvg_b200.engine import TrainEngine
    state = O.build_state(CFG, seed=1)
    opt = O.default_opt(**optkw)
    opt["batch_size"] = B
    return TrainEngine(state, CFG, opt, kernels, act_dtype=torch.bfloat16)


def _inputs(optkw, seed):
    opt = O.default_opt(**optkw)
    x = torch.rand(T, B, 1, 64, 64, generator=torch.Generator().manual_seed(5)).cuda()
    probs = np.random.RandomState(seed).uniform(0, 1, T - 1)
    plan = StepPlan(T, probs, opt)
    eps = O.draw_eps(plan.S, B, 10, seed=11).cuda()
    return x, probs, eps, plan


def _snapshot(eng, losses):
    torch.cuda.synchronize()
    return dict(losses=np.asarray(losses), grads={(m, k): v.detach().clone() for m in eng.arena for k, v in eng.arena[m].g.items()},
                params={(m, k): v.detach().clone() for m in eng.arena for k, v in eng.arena[m].p.items()})


STEP_CASES = [("bench_options", BENCH_OPT), ("skip_lfs", SKIP_OPT)]


@pytest.mark.parametrize("case", STEP_CASES, ids=[c[0] for c in STEP_CASES])
def test_step_matches_the_unfused_sequence(K, case):
    name, optkw = case
    seed = _skip_seed() if name == "skip_lfs" else 0
    x, probs, eps, plan = _inputs(optkw, seed)
    if name == "skip_lfs":
        assert plan.nskip > len(set(plan.skip_src[:plan.S])) >= 3
    eng = _engine(_unfused_kernels(), optkw)
    assert not eng.bn_skip_sums and not eng.bn_wgrad_c1
    old = _snapshot(eng, eng.step(x, probs=probs, eps=eps))
    gy0 = eng._bufs["enc_gy0"][:T * B * 32 * 32 * 64].clone()   # enc0's dx, stored by the unfused sequence only
    cin = eng.enc_in[:T * B * 64 * 64].clone()
    S = plan.S
    y2 = eng.dec[2]["d"][:S * B * 32 * 32 * 64].clone()            # dec2's output, the input of the last layer's first half
    dout = eng.d_rawout[:S * B * 64 * 64].clone()
    del eng
    eng = _engine(K, optkw)
    assert eng.bn_skip_sums and eng.bn_wgrad_c1
    new = _snapshot(eng, eng.step(x, probs=probs, eps=eps))
    del eng
    assert np.array_equal(old["losses"], new["losses"]), (old["losses"], new["losses"])
    for key in old["grads"]:
        if key in (ENC0_W, DEC_LAST_W):
            continue
        assert torch.equal(old["grads"][key], new["grads"][key]), f"gradient {key} differs"
    d_old, d_new = old["grads"][DEC_LAST_W].view(128, 16), new["grads"][DEC_LAST_W].view(128, 16)
    assert torch.equal(d_old[64:], d_new[64:]), "the skip half of the last layer's weight gradient differs"
    rel = ((d_new[:64] - d_old[:64]).abs().max() / d_old[:64].abs().max()).item()
    exact, absum = _wgrad64(y2, dout, 32)
    ratio = ((d_new[:64].double() - exact).abs() / _fp32_bound(absum, B * 32 * 32)).max().item()
    print(f"[step] {name}: last decoder layer weight gradient vs unfused {rel:.3g} relative, worst error / fp32 bound {ratio:.3g}")
    assert rel <= 1e-5
    assert ratio <= 1.0
    # the first encoder layer's weight gradient: the same bf16 products, summed in another order
    g_old, g_new = old["grads"][ENC0_W].double().view(64, 16), new["grads"][ENC0_W].double().view(64, 16)
    rel = ((g_new - g_old).abs().max() / g_old.abs().max()).item()
    exact, absum = _wgrad64(gy0, cin, 32)
    ratio = ((g_new - exact).abs() / _fp32_bound(absum, B * 32 * 32)).max().item()
    print(f"[step] {name}: enc0 weight gradient vs unfused {rel:.3g} relative, worst error / fp32 bound {ratio:.3g}")
    assert rel <= 1e-5
    assert ratio <= 1.0
    # the parameters moved by Adam only differ through those two gradients
    for key in old["params"]:
        if key not in (ENC0_W, DEC_LAST_W):
            assert torch.equal(old["params"][key], new["params"][key]), f"parameter {key} differs"


def test_step_is_deterministic_eager_and_graphed(K):
    """Two eager steps twice over, and the same two steps with the second one captured and replayed from a CUDA graph."""
    seed = _skip_seed()
    x, probs, eps, _ = _inputs(SKIP_OPT, seed)
    runs = []
    for graphed in (False, False, True):
        eng = _engine(K, SKIP_OPT)
        eng.step(x, probs=probs, eps=eps, use_graph=graphed)
        runs.append(_snapshot(eng, eng.step(x, probs=probs, eps=eps, use_graph=graphed)))
        if graphed:
            assert eng._graphs and all(v != "warm" for v in eng._graphs.values()), "the second step did not replay a graph"
        del eng
    for other in runs[1:]:
        assert np.array_equal(runs[0]["losses"], other["losses"])
        for key in runs[0]["grads"]:
            assert torch.equal(runs[0]["grads"][key], other["grads"][key]), f"gradient {key} differs between runs"
            assert torch.equal(runs[0]["params"][key], other["params"][key]), f"parameter {key} differs between runs"
