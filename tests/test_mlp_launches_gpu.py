"""The h36m_mlp training step's fp32 and TF32 launches against float64, at the shapes of the C5 benchmark configuration
(T = 60, B = 256 per GPU, rnn_size 512).

  A. the launch list tests/mlp_ref.py derives from engine_mlp.py (every GEMM with its operands' buffers, offsets and pitches,
     and the element-wise kernels), against what one eager step records: at exactly C5 in the bf16 (TF32) mode and in the fp32
     mode, and at C5 with a skip plan;
  B. dispatch: every GEMM of the C5 step rerun on its real operands through a view that makes a SIMT fallback an error; the
     derived list's "tf32" launches must run there bit-identically, its "simt" ones must be refused and rerun bit-identically
     on the exact kernel;
  C. every distinct GEMM of the list at its C5 shape against float64, on the engine's pitches and offsets with NaN-poisoned
     neighbours and a sentinel around the output segment, on the kernel the list names; the weight gradients (K = 15 360 and
     15 104, split-K) exact on 0 / 1 operands and within the split-K bound on operands that do not cancel; a TF32 launch with
     bias followed by a SIMT accumulate into the same output, as d2 / d3 do;
  D. the element-wise kernels at C5 sizes: ReLU forward / backward (in place, exact zeros), tanh, permute4 (copy and the
     residual / dx1 sums), gather_add_cols on the skip-gradient matrix and build_concat of the skip matrix;
  E. an audit of real steps (C5 with the bench options, and a skip plan at B = 32): every GEMM of any dtype, the ReLU / tanh,
     permute4, gather / concat and LayerNorm launches checked against float64 as they run, coverage of the derived variants,
     the skip tables, and steps bit-identical to plain CudaKernels with concurrent lanes and to a graph replay;
  F. the whole C5 step against the float64 oracle on the device, in the fp32 and in the bf16 mode.
"""
import copy
import math
import time

import numpy as np
import pytest
import torch

from oracle import p2p_oracle as O
from p2pvg_b200._lib import CudaKernels, KernelError
from p2pvg_b200.engine import StepPlan
from p2pvg_b200.engine_mlp import TrainEngineMLP
from tests.launch_audit import K, memory_per_test  # noqa: F401  (fixtures)
from tests.launch_audit import (BENCH_OPT, NAN, SKIP_OPT, TF32_FLAG, TF32_REQUIRE, AuditKernels, RecordingKernels, assert_concurrent,
                                assert_equal_steps, audit_step, entry_kernel, gemm_alpha, kernel_for, release, run_step, simt_alpha,
                                skip_seed, step_inputs, watch_backbone)
from tests.loss_ref import (ACT_RELU, ACT_TANH, TINY, act_bwd_ref, act_fwd_ref, build_concat_ref, check_gather_add_cols,
                            check_layernorm_bwd, check_layernorm_fwd)
from tests.lstm_schedule import U
from tests.mlp_ref import POSE, backbone_launches, gemm_variant, key
from tests.ref64 import assert_exact, bound_check, gemm_ref64
from tests.tc_schedule import alpha_for, assert_within, gemm_tc_tiles

pytestmark = pytest.mark.gpu

C5 = dict(T=60, B=256, R=512)
CFG = dict(g_dim=128, z_dim=10, rnn_size=512, backbone="mlp", predictor_rnn_layers=2, posterior_rnn_layers=1, prior_rnn_layers=1)
H = 128                      # h_dim = g_dim (engine_mlp.py:130)
LD = 2 * H + 2               # pitch of the skip matrix (engine_mlp.py:167)
SENTINEL = -777.0
def _np_seed(T, optkw):
    return skip_seed(T) if optkw.get("skip_prob") else 0


# ------------------------------------------------------------------ A. the launch lists

class _Locator:
    """Names the buffer a pointer lies in, as tests/mlp_ref.py does: the input frames, arena parameters / gradients, engine
    scratch buffers (fbuf names)."""

    def __init__(self, eng, x):
        self.eng, self.x, self.regions = eng, x, []

    def _scan(self):
        R = [("x", self.x)] + list(self.eng._bufs.items())
        for m, A in self.eng.arena.items():
            R += [(f"p:{m}.{k}", v) for k, v in A.p.items()] + [(f"g:{m}.{k}", v) for k, v in A.g.items()]
        self.regions = [(n, t.data_ptr(), t.numel() * t.element_size(), t.element_size()) for n, t in R]

    def __call__(self, t):
        p = t.data_ptr()
        for attempt in range(2):
            for n, base, nb, es in self.regions:
                if base <= p < base + nb:
                    return (n, (p - base) // es)
            self._scan()
        return ("?", p)


def _on(f):
    return lambda k, x: f(k.loc, x) if k.on else None


class MlpRecording(RecordingKernels):
    """Logs every launch of the backbone (while `on`), with its operands located by buffer and offset.  rerun=True: each
    fp32 GEMM is also rerun on copies of its output through a view with P2PVG_GEMM_TF32 | P2PVG_GEMM_TF32_REQUIRE and through
    one with flags 0, logging (ran on TF32, TF32 rerun identical, flags-0 rerun identical) in `reruns`."""
    RECORD = {
        "gemm": _on(lambda L, x: ("gemm", x["M"], x["N"], x["K"], x["a_mn"], x["b_mn"],
                                  x["lda"] if x["lda"] is not None else (x["M"] if x["a_mn"] else x["K"]),
                                  x["ldb"] if x["ldb"] is not None else (x["N"] if x["b_mn"] else x["K"]),
                                  x["ldc"] if x["ldc"] is not None else x["N"], bool(x["accumulate"]), x["bias"] is not None,
                                  L(x["A"]), L(x["B"]), L(x["C"]))),
        "act_fwd": _on(lambda L, x: ("act_fwd", L(x["x"]), x["n"], x["act"])),
        "act_bwd": _on(lambda L, x: ("act_bwd", L(x["dy"]), L(x["y"]), L(x["dx"]), x["n"], x["act"])),
        "permute4": _on(lambda L, x: ("permute4", L(x["src"]), L(x["dst"]), tuple(x["dims"]), tuple(x["strides"]),
                                      bool(x["accumulate"]))),
        "layernorm_fwd": _on(lambda L, x: ("layernorm_fwd", L(x["x"]), L(x["y"]), x["rows"], x["C"])),
        "layernorm_bwd": _on(lambda L, x: ("layernorm_bwd", L(x["dy"]), L(x["x"]), L(x["dx"]), x["dgamma"] is not None, x["rows"],
                                           x["C"])),
        "build_concat": _on(lambda L, x: ("build_concat", L(x["dst"]), L(x["A"]), L(x["ia"]), x["ga"], L(x["Bm"]), L(x["ib"]),
                                          x["gb"], x["S"], x["B"], x["ld"])),
        "gather_add_cols": _on(lambda L, x: ("gather_add_cols", L(x["dst"]), L(x["src"]), L(x["idx"]), x["S"], x["T"], x["B"],
                                             x["g"], x["W"], x["col0"])),
        "colsum": _on(lambda L, x: ("colsum", L(x["x"]), x["rows"], x["cols"], x["ld"], L(x["out"]))),
        "mse_plain": _on(lambda L, x: ("mse_plain", L(x["pred"]), L(x["x"]), L(x["tgt"]), x["G"], x["E"])),
    }

    def __init__(self, *a, rerun=False, **kw):
        super().__init__(*a, **kw)
        self.reruns = []
        self.on, self.rerun, self.loc = False, rerun, None

    def launch(self, op, args):
        if op != "gemm" or not (self.on and self.rerun):
            return super().launch(op, args)
        C = args["C"]
        torch.cuda.synchronize()
        C0 = C.clone()
        super().launch(op, args)
        torch.cuda.synchronize()
        req, plain = copy.copy(self), copy.copy(self)
        req.gemm_flags, plain.gemm_flags = TF32_FLAG | TF32_REQUIRE, 0
        C1, C2 = C0.clone(), C0.clone()
        try:
            CudaKernels.gemm(**{**args, "self": req, "C": C1})
            ran = True
        except KernelError:
            ran = False
        CudaKernels.gemm(**{**args, "self": plain, "C": C2})
        torch.cuda.synchronize()
        self.reruns.append((ran, ran and torch.equal(C1, C), torch.equal(C2, C)))


def _recorded_step(T, B, optkw, adt, rerun=False):
    rec = MlpRecording("cuda", rerun=rerun)

    def prepare(eng, x):   # eng.K is the engine's view of rec (CudaKernels.with_mode): same logs, its own flags
        watch_backbone(eng)
        eng.K.loc = _Locator(eng, x)
    plan, (losses, _, _) = run_step(TrainEngineMLP, CFG, optkw, rec, T, B, _np_seed(T, optkw), act_dtype=adt, prepare=prepare)
    assert np.all(np.isfinite(losses))
    return plan, rec


LIST_CASES = [("C5-bf16", BENCH_OPT, torch.bfloat16, C5["B"]), ("C5-fp32", BENCH_OPT, torch.float32, C5["B"]),
              ("C5-skip-bf16", SKIP_OPT, torch.bfloat16, C5["B"])]


@pytest.mark.parametrize("case", LIST_CASES, ids=[c[0] for c in LIST_CASES])
def test_launch_list_matches_an_eager_step(case):
    """The derived list equals, call for call and in order, the backbone launches of one eager step (the recurrent phase
    muted): shapes, flags, pitches, and the buffer and offset of every operand."""
    name, optkw, adt, B = case
    plan, rec = _recorded_step(C5["T"], B, optkw, adt)
    if optkw is SKIP_OPT:
        assert len(set(plan.skip_src)) >= 3 and plan.has_cpc
    got = rec.calls
    derived = backbone_launches(plan, B)
    want = [key(e) for e in derived]
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"{name}: launch {i} is {g}, the derived list says {w} ({derived[i]['name']})"
    assert len(got) == len(want), f"{name}: {len(got)} launches recorded, {len(want)} derived"
    print(f"[list] {name}: {len(got)} launches, {sum(1 for e in derived if e['op'] == 'gemm')} GEMMs, in order")


# ------------------------------------------------------------------ B. dispatch

def test_dispatch_of_every_c5_gemm():
    """Each fp32 GEMM of the bf16-mode C5 step, rerun on its real operands: where the list says tf32 it must run on the TF32
    kernel when a fallback is an error, bit-identically to the step; where it says simt it must be refused there, and a rerun
    with flags 0 (the exact kernel) must be bit-identical."""
    plan, rec = _recorded_step(C5["T"], C5["B"], BENCH_OPT, torch.bfloat16, rerun=True)
    derived = [e for e in backbone_launches(plan, C5["B"]) if e["op"] == "gemm"]
    reruns = rec.reruns
    assert len(reruns) == len(derived)
    n_tf32 = 0
    for e, (ran, same_req, same_plain) in zip(derived, reruns):
        kern = entry_kernel(e, True)
        what = f"{e['name']} {e['M']}x{e['N']}x{e['K']} lda={e['lda']} ldb={e['ldb']} (list: {kern})"
        if kern == "tf32":
            n_tf32 += 1
            assert ran, f"{what}: refused by the TF32 kernel"
            assert same_req, f"{what}: the TF32 rerun differs from the step's launch"
        else:
            assert not ran, f"{what}: ran on the TF32 kernel"
            assert same_plain, f"{what}: the exact-kernel rerun differs from the step's launch"
    # the forward GEMMs of e2, e3, d1 and the first segments of d2 / d3
    assert n_tf32 == 14, n_tf32
    print(f"[dispatch] {len(derived)} GEMMs: {n_tf32} on TF32, {len(derived) - n_tf32} on the CUDA cores")


# ------------------------------------------------------------------ C. every distinct GEMM against float64

def _c5_plan():
    return StepPlan(C5["T"], np.zeros(C5["T"] - 1), O.default_opt(**BENCH_OPT))


def _distinct_gemms():
    seen, out = set(), []
    for e in backbone_launches(_c5_plan(), C5["B"]):
        if e["op"] != "gemm":
            continue
        geo = (e["M"], e["N"], e["K"], e["a_mn"], e["b_mn"], e["lda"], e["ldb"], e["ldc"], e["accumulate"], e["bias"],
               e["A"][1] % e["lda"], e["B"][1] % e["ldb"], e["C"][1] % e["ldc"], e["A"][1] >= e["lda"])
        for tf32 in (True, False):
            kern = entry_kernel(e, tf32)
            if (geo, kern) not in seen:
                seen.add((geo, kern))
                out.append((e, tf32))
    return out


DISTINCT = _distinct_gemms()


def _operand(off, rows, cols, ld, fill, gen, pad=64):
    """A buffer holding a [rows, cols] matrix of pitch ld at element offset off; everything else is `fill`."""
    buf = torch.full((off + (rows - 1) * ld + cols + pad,), fill, device="cuda")
    view = buf[off:].as_strided((rows, cols), (ld, 1))
    return buf, view


def _run_gemm(K, e, gen, tf32, values="randn"):
    """Operands of entry e at its pitches and offsets (NaN around the operands, SENTINEL around the output), one launch on the
    view of the given mode.  Returns (C view, C buffer, mask of the output elements, float64 reference, magnitude)."""
    M, N, Kd = e["M"], e["N"], e["K"]
    ar, ac = (Kd, M) if e["a_mn"] else (M, Kd)
    br, bc = (Kd, N) if e["b_mn"] else (N, Kd)
    Abuf, Av = _operand(e["A"][1], ar, ac, e["lda"], NAN, gen)
    Bbuf, Bv = _operand(e["B"][1], br, bc, e["ldb"], NAN, gen)
    if values == "randn":
        Av.copy_(torch.randn(ar, ac, device="cuda", generator=gen))
        Bv.copy_(torch.randn(br, bc, device="cuda", generator=gen))
    elif values == "binary":
        Av.copy_((torch.rand(ar, ac, device="cuda", generator=gen) < 0.25).float())
        Bv.copy_((torch.rand(br, bc, device="cuda", generator=gen) < 0.25).float())
    else:   # non-cancelling: one positive operand, one of mean 1/2
        Av.copy_(torch.rand(ar, ac, device="cuda", generator=gen))
        Bv.copy_(torch.randn(br, bc, device="cuda", generator=gen) * 0.5 + 0.5)
    Cbuf, Cv = _operand(e["C"][1], M, N, e["ldc"], SENTINEL, gen)
    mask = torch.zeros_like(Cbuf, dtype=torch.bool)
    mask[e["C"][1]:].as_strided((M, N), (e["ldc"], 1)).fill_(True)
    c0 = None
    if e["accumulate"]:
        c0 = torch.randn(M, N, device="cuda", generator=gen)
        Cv.copy_(c0)
    else:
        Cv.fill_(NAN)   # must be overwritten, never read
    bias = torch.randn(N, device="cuda", generator=gen) if e["bias"] else None
    K.with_mode(tf32).gemm(Abuf[e["A"][1]:], Bbuf[e["B"][1]:], Cbuf[e["C"][1]:], M, N, Kd, e["a_mn"], e["b_mn"], e["lda"], e["ldb"],
                           e["ldc"], e["accumulate"], bias)
    torch.cuda.synchronize()
    assert (Cbuf[~mask] == SENTINEL).all(), f"{e['name']}: elements outside the output segment were written"
    ref, absref = gemm_ref64(Abuf[e["A"][1]:], Bbuf[e["B"][1]:], M, N, Kd, e["a_mn"], e["b_mn"], e["lda"], e["ldb"], bias=bias, c0=c0)
    return Cv, ref, absref, bias, c0


@pytest.mark.parametrize("e,tf32", DISTINCT, ids=[f"{e['name'].replace(' ', '_')}-{e['M']}x{e['N']}x{e['K']}-"
                                                  f"{'tf32mode' if t else 'fp32mode'}" for e, t in DISTINCT])
def test_gemm_at_c5_shape(K, e, tf32):
    """One launch of the GEMM at its C5 shape, pitches and offsets, on the kernel the list names, against float64."""
    kern = entry_kernel(e, tf32)
    name = f"{e['name']} {e['M']}x{e['N']}x{e['K']} lda={e['lda']} ldb={e['ldb']} ldc={e['ldc']} on {kern}"
    gen = torch.Generator(device="cuda").manual_seed(e["M"] * 7 + e["N"] * 3 + e["K"])
    extra = int(e["bias"]) + int(e["accumulate"])
    Cv, ref, absref, _, _ = _run_gemm(K, e, gen, tf32)
    assert_within(Cv, ref, absref, e["K"], torch.float32, alpha=gemm_alpha(e["K"], kern, extra), name=name)
    if e["K"] >= 2048:
        # the weight gradients: sums of 0 / 1 products stay below 2^24, exact in any order; then operands that do not
        # cancel, where a lost or doubled split is far outside the bound
        assert not isinstance(kern, str), f"{name}: the list says this long reduction is not split"
        Cv, ref, _, _, _ = _run_gemm(K, e, gen, tf32, values="binary")
        assert_exact(Cv, ref, e["K"], name + " 0/1 operands")
        Cv, ref, absref, _, _ = _run_gemm(K, e, gen, tf32, values="positive")
        assert (ref.abs() >= 0.25 * absref).all()
        assert_within(Cv, ref, absref, e["K"], torch.float32, alpha=simt_alpha(e["K"], kern, extra),
                      name=name + " non-cancelling operands")


def test_c5_gemm_coverage():
    """The distinct GEMMs include the edges the kernels treat specially."""
    geo = {(e["name"].split(" ")[0], e["M"], e["N"], e["K"], entry_kernel(e, True)) for e, _ in DISTINCT}
    assert ("d3.fc3", 15360, POSE, H, "tf32") in geo                   # ragged N = 51 TF32 output (204-byte rows)
    assert ("e1.fc1.long_path.2", 15360, 25, 25, "simt") in geo        # N = K = 25
    assert ("e1.fc1.shortcut.0", 15360, H, POSE, "simt") in geo        # x at pitch 51
    ks = {(e["K"], entry_kernel(e, True)) for e, _ in DISTINCT if e["a_mn"]}
    assert (15360, ("simt-splitK", 60, 256)) in ks and (15104, ("simt-splitK", 59, 256)) in ks
    cpc = [e for e, _ in DISTINCT if e["A"][0] == "d_pred" and e["A"][1] > 0]
    assert cpc, "no CPC-call GEMM at a row offset"
    skip_cols = {e["A"][1] % LD for e, _ in DISTINCT if e["lda"] == LD} | {e["B"][1] % LD for e, _ in DISTINCT if e["ldb"] == LD} | \
        {e["C"][1] % LD for e, _ in DISTINCT if e["ldc"] == LD}
    assert skip_cols == {0, H}, skip_cols


PAIRS = [("d2.fc2.shortcut.0 fwd", H), ("d2.fc2.long_path.0 fwd", H), ("d3.fc3 fwd", 0)]


@pytest.mark.parametrize("lin,col0", PAIRS, ids=[p[0].split(" ")[0] for p in PAIRS])
def test_tf32_bias_then_simt_accumulate(K, lin, col0):
    """[x0 | skip] . W^T + b as d2 / d3 evaluate it at C5: a TF32 launch with bias over the dense segment, then a SIMT launch
    accumulating the skip columns (pitch 258, neighbours NaN) into the same output; the result against float64 of the whole
    product, within the TF32 bound of the first part plus the SIMT bound of the second."""
    segs = [e for e in backbone_launches(_c5_plan(), C5["B"]) if e["op"] == "gemm" and e["name"].startswith(lin)]
    assert [entry_kernel(e, True) for e in segs] == ["tf32", "simt"] and segs[1]["A"][1] == col0 and segs[1]["lda"] == LD
    e0, e1 = segs
    M, N = e0["M"], e0["N"]
    gen = torch.Generator(device="cuda").manual_seed(77)
    X0 = torch.randn(M, H, device="cuda", generator=gen)
    Sbuf, Sv = _operand(0, M, LD, LD, NAN, gen)
    Sv[:, col0:col0 + H].copy_(torch.randn(M, H, device="cuda", generator=gen))
    W = torch.randn(N, 2 * H, device="cuda", generator=gen) / math.sqrt(2 * H)
    b = torch.randn(N, device="cuda", generator=gen)
    C = torch.full((M * N + 64,), SENTINEL, device="cuda")
    Kt = K.with_mode(True)
    Kt.gemm(X0, W.view(-1), C, M, N, H, lda=H, ldb=2 * H, bias=b)
    Kt.gemm(Sbuf[col0:], W.view(-1)[H:], C, M, N, H, lda=LD, ldb=2 * H, accumulate=True)
    torch.cuda.synchronize()
    assert (C[M * N:] == SENTINEL).all()
    r0, a0 = gemm_ref64(X0, W, M, N, H, False, False, H, 2 * H, bias=b)
    r1, a1 = gemm_ref64(Sbuf[col0:], W.view(-1)[H:], M, N, H, False, False, LD, 2 * H)
    ref = r0 + r1
    bound = (alpha_for(H, tf32=True) + U) * a0 + simt_alpha(H, "simt", 1) * (a1 + a0 * (1 + alpha_for(H, tf32=True))) + 2.0 ** -22 * ref.abs()
    w = bound_check(C[:M * N].view(M, N), ref, bound, f"{lin} TF32 + bias then SIMT accumulate")
    print(f"[bound] {lin}: worst error/bound {w:.3g}")


# ------------------------------------------------------------------ D. element-wise kernels at C5 sizes

def test_relu_forward_backward_exact(K):
    """act_fwd / act_bwd with ReLU on the e2 / d2 long-path sizes (N rows x 128), with exact zeros in x and in y, and the
    backward in place (dy == dx) as the engine runs it on g2 / g1: both bit-exact."""
    n = C5["T"] * C5["B"] * H
    gen = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(n, device="cuda", generator=gen)
    x[::7] = 0.0
    x[1::11] = -0.0
    y = x.clone()
    K.act_fwd(y, n, ACT_RELU)
    torch.cuda.synchronize()
    assert torch.equal(y, x.clamp_min(0)), "ReLU forward"
    assert (y == 0).sum() > n // 3
    dy = torch.randn(n, device="cuda", generator=gen)
    ref = torch.where(y > 0, dy, torch.zeros_like(dy))
    K.act_bwd(dy, y, dy, n, ACT_RELU)
    torch.cuda.synchronize()
    assert torch.equal(dy, ref), "ReLU backward in place: gradient passed where y == 0, or dropped where y > 0"


def test_tanh_latent(K):
    """act_fwd / act_bwd with tanh on the latent (T B x g) and the encoder's dpre, within act_fwd_ref / act_bwd_ref."""
    n = C5["T"] * C5["B"] * H
    gen = torch.Generator(device="cuda").manual_seed(4)
    x = torch.randn(n, device="cuda", generator=gen) * 2
    y = x.clone()
    K.act_fwd(y, n, ACT_TANH)
    ref, err = act_fwd_ref(x, ACT_TANH)
    w = bound_check(y, ref, err + TINY, "tanh forward")
    dy = torch.randn(n, device="cuda", generator=gen)
    dx = torch.full_like(dy, NAN)
    K.act_bwd(dy, y, dx, n, ACT_TANH)
    ref, err = act_bwd_ref(dy, y, ACT_TANH)
    w = max(w, bound_check(dx, ref, err + TINY, "tanh backward"))
    print(f"[bound] tanh: worst error/bound {w:.3g}")


def test_permute4_copy_and_sum(K):
    """permute4 as the residual sum (copy, then accumulate) and the dx1 fold use it: the copy exact, the sum one rounding."""
    n = C5["T"] * C5["B"] * H
    gen = torch.Generator(device="cuda").manual_seed(5)
    a, b = torch.randn(n, device="cuda", generator=gen), torch.randn(n, device="cuda", generator=gen) * 3
    s = torch.full((n + 64,), SENTINEL, device="cuda")
    K.permute4(a, s, (n, 1, 1, 1), (1, 0, 0, 0))
    torch.cuda.synchronize()
    assert torch.equal(s[:n], a) and (s[n:] == SENTINEL).all()
    K.permute4(b, s, (n, 1, 1, 1), (1, 0, 0, 0), accumulate=True)
    ref = a.double() + b.double()
    w = bound_check(s[:n], ref, U * ref.abs(), "permute4 accumulate")
    assert (s[n:] == SENTINEL).all()
    print(f"[bound] permute4 accumulate: worst error/bound {w:.3g}")


def _skip_plan():
    T = C5["T"]
    opt = O.default_opt(**SKIP_OPT)
    p = StepPlan(T, np.random.RandomState(skip_seed(T)).uniform(0, 1, T - 1), opt)
    assert len(set(p.skip_src)) >= 3
    return p


@pytest.mark.parametrize("col0", [0, H])
def test_gather_add_cols_skip_gradients(K, col0):
    """gather_add_cols from the skip-gradient matrix (pitch 258, the columns of h1 or h2) into dh1 / dh2 [T, B, h], over the
    skip plan's skip_src (several calls per source frame), the tuc / dt columns NaN."""
    p = _skip_plan()
    T, B, S = C5["T"], C5["B"], p.S
    gen = torch.Generator(device="cuda").manual_seed(6 + col0)
    src = torch.full(((S + 1) * B * LD,), NAN, device="cuda")
    sv = src.view(S + 1, B, LD)
    sv[:, :, :2 * H] = torch.randn(S + 1, B, 2 * H, device="cuda", generator=gen)
    idx = torch.tensor(p.skip_src, dtype=torch.int32, device="cuda")
    dst0 = torch.randn(T * B * H, device="cuda", generator=gen)
    dst = dst0.clone()
    K.gather_add_cols(dst, src, idx, S, T, B, H, LD, col0)
    torch.cuda.synchronize()
    check_gather_add_cols(dst, dst0, src, idx, S, T, B, H, LD, col0, False)


def test_build_concat_skipsel(K):
    """build_concat of the decoder's skip matrix [h1 | h2 | tuc | dt] (pitch 258) for the S + 1 calls of the skip plan: a copy,
    bit-exact."""
    p = _skip_plan()
    T, B, S = C5["T"], C5["B"], p.S
    G = S + 1
    gen = torch.Generator(device="cuda").manual_seed(7)
    h1, h2 = torch.randn(T * B * H, device="cuda", generator=gen), torch.randn(T * B * H, device="cuda", generator=gen)
    idx = torch.tensor(p.skip_src, dtype=torch.int32, device="cuda")
    tuc = torch.tensor(p.tuc + [p.tuc[-1]], device="cuda")
    dt = torch.tensor(p.dt + [p.dt[-1]], device="cuda")
    dst = torch.full((G * B * LD + 64,), NAN, device="cuda")
    K.build_concat(dst, h1, idx, H, h2, idx, H, tuc, dt, G, B, ld=LD)
    torch.cuda.synchronize()
    assert torch.equal(dst[:G * B * LD], build_concat_ref(h1, idx, H, h2, idx, H, tuc, dt, G, B, LD))
    assert torch.isnan(dst[G * B * LD:]).all()


# ------------------------------------------------------------------ E. audit of real steps

class MlpAudit(AuditKernels):
    """AuditKernels for an mlp step: GEMMs of every dtype on the kernel mlp_ref names, act_fwd / act_bwd, permute4,
    gather_add_cols, build_concat and LayerNorm.  GEMMs outside the backbone methods (`on` unset) are the recurrent ones."""
    REPORT_GEMMS_ONLY = True
    GEMM_PROBE_K = 4096
    GEMM_PROBE_ACCUMULATING = False

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.on, self.eng = False, None

    def _is(self, t, name):
        b = self.eng._bufs.get(name) if self.eng is not None else None
        return b is not None and b.data_ptr() == t.data_ptr()

    def gemm_bound(self, A, B, M, N, K, a_mn, b_mn, lda, ldb, extra):
        if A.dtype == torch.bfloat16:
            s = gemm_tc_tiles(M, N, K, self._sms)
            return alpha_for(s.kb_per_split * 64 + 16 * s.splits), "tc"
        kern = kernel_for(M, N, K, a_mn, b_mn, lda, ldb, A.data_ptr() % 16 // 4, B.data_ptr() % 16 // 4, bool(self.gemm_flags & TF32_FLAG))
        return gemm_alpha(K, kern, extra), kern

    def gemm_variant(self, A, kern, a_mn, b_mn, accumulate, bias, strided):
        v = ("gemm", kern if isinstance(kern, str) else kern[0], a_mn, b_mn, bool(accumulate), bias is not None, strided)
        return v if self.on else ("gemm-recurrent", A.dtype, v[1])

    def act_fwd(self, x, n, act):
        torch.cuda.synchronize()
        x0 = x[:n].clone()
        self._sync("act_fwd", x, n, act)
        ref, err = act_fwd_ref(x0, act)
        self._rec(f"act_fwd {act} n={n}", ("act_fwd", act), bound_check(x[:n], ref, err + (TINY if act != ACT_RELU else 0), f"audit act_fwd {act}"))

    def act_bwd(self, dy, y, dx, n, act):
        torch.cuda.synchronize()
        d0, y0 = dy[:n].clone(), y[:n].clone()
        self._sync("act_bwd", dy, y, dx, n, act)
        ref, err = act_bwd_ref(d0, y0, act)
        aliased = dy.data_ptr() == dx.data_ptr()
        self._rec(f"act_bwd {act} n={n}", ("act_bwd", act, aliased),
                  bound_check(dx[:n], ref, err + (TINY if act != ACT_RELU else 0), f"audit act_bwd {act}"))

    def permute4(self, src, dst, dims, strides, accumulate=False):
        torch.cuda.synchronize()
        n = dims[0] * dims[1] * dims[2] * dims[3]
        d0 = dst.reshape(-1)[:n].clone() if accumulate else None
        self._sync("permute4", src, dst, dims, strides, accumulate)
        s = src.as_strided(tuple(dims), tuple(strides)).reshape(-1).double()
        got = dst.reshape(-1)[:n]
        if accumulate:
            ref = d0.double() + s
            w = bound_check(got, ref, U * ref.abs() if dst.dtype == torch.float32 else 2.0 ** -8 * ref.abs(), "audit permute4 sum")
        else:
            ref = s.to(dst.dtype).double()
            w = bound_check(got, ref, torch.zeros_like(ref), "audit permute4 copy")
        self._rec(f"permute4 {tuple(dims)}", ("permute4", bool(accumulate)), w)

    def gather_add_cols(self, dst, src, idx, S, T, B, g, W, col0, init=False):
        torch.cuda.synchronize()
        d0 = dst.reshape(-1)[:T * B * g].clone()
        self._sync("gather_add_cols", dst, src, idx, S, T, B, g, W, col0, init)
        if self._is(src, "dskipsel"):
            self.skip_reads.append(("gather_add_cols", col0, idx.tolist()[:S]))
        check_gather_add_cols(dst, d0, src, idx, S, T, B, g, W, col0, init)
        self._rec(f"gather_add_cols W={W} col0={col0}", ("gather_add_cols", self._is(src, "dskipsel")), 0.0)

    def build_concat(self, dst, A, ia, ga, Bm, ib, gb, tuc, dt, S, B, ld=None):
        self._sync("build_concat", dst, A, ia, ga, Bm, ib, gb, tuc, dt, S, B, ld)
        ld_ = ld if ld is not None else ga + gb + 2
        if self._is(dst, "skipsel"):
            self.skip_reads.append(("build_concat", 0, ia.tolist()[:S]))
            self.skip_reads.append(("build_concat", ga, ib.tolist()[:S]))
        ref = build_concat_ref(A, ia, ga, Bm, ib, gb, tuc, dt, S, B, ld_)
        assert torch.equal(dst.reshape(-1)[:S * B * ld_], ref), f"audit build_concat S={S} ld={ld_}"
        self._rec(f"build_concat ld={ld_}", ("build_concat", self._is(dst, "skipsel")), 0.0)

    def layernorm_fwd(self, x, gamma_, beta, y, mean, rstd, rows, C, eps=1e-5):
        self._sync("layernorm_fwd", x, gamma_, beta, y, mean, rstd, rows, C, eps)
        check_layernorm_fwd(x, gamma_, beta, y, mean, rstd, rows, C, eps)
        self._rec(f"layernorm_fwd rows={rows}", ("layernorm_fwd",), 0.0)

    def layernorm_bwd(self, dy, x, mean, rstd, gamma_, dx, dgamma, dbeta, rows, C):
        torch.cuda.synchronize()
        d0 = dy.reshape(-1)[:rows * C].clone()
        self._sync("layernorm_bwd", dy, x, mean, rstd, gamma_, dx, dgamma, dbeta, rows, C)
        check_layernorm_bwd(d0, x, mean, rstd, gamma_, dx, dgamma, dbeta, rows, C)
        self._rec(f"layernorm_bwd rows={rows}", ("layernorm_bwd", dgamma is not None), 0.0)


AUDIT_CASES = [("C5_bench_options", BENCH_OPT, C5["B"]), ("skip_lfs_B32", SKIP_OPT, 32)]


@pytest.mark.parametrize("case", AUDIT_CASES, ids=[c[0] for c in AUDIT_CASES])
def test_audit_mlp_step(case):
    """One eager bf16-mode step at T = 60 with every audited launch checked as it runs.  Every GEMM variant of the derived list
    must occur, the skip matrix must be built and its gradients gathered through plan.skip_src, and losses, gradients and
    parameters must equal (torch.equal) the same step on plain CudaKernels with its concurrent lanes."""
    name, optkw, B = case
    audit = MlpAudit("cuda")

    def expect(plan):
        want = {gemm_variant(e, entry_kernel(e, True)) for e in backbone_launches(plan, B) if e["op"] == "gemm"}
        want |= {("act_fwd", ACT_RELU), ("act_fwd", ACT_TANH), ("act_bwd", ACT_RELU, True), ("act_bwd", ACT_RELU, False),
                 ("act_bwd", ACT_TANH, False), ("permute4", False), ("permute4", True), ("gather_add_cols", True),
                 ("build_concat", True), ("layernorm_fwd",), ("layernorm_bwd", True), ("layernorm_bwd", False)}
        # the skip matrix [h1 | h2 | ..] is built for the S + 1 decoder calls, its gradients gathered over the S reconstructions
        src = plan.skip_src
        return want, [("build_concat", 0, src[:plan.S + 1]), ("build_concat", H, src[:plan.S + 1]),
                      ("gather_add_cols", 0, src[:plan.S]), ("gather_add_cols", H, src[:plan.S])]

    def watched(eng, x):
        eng.K.eng = eng
        watch_backbone(eng)
    audit_step(TrainEngineMLP, CFG, optkw, C5["T"], B, audit, expect, name, prepare=watched)
    rec = {v for v in audit.seen if v[0] == "gemm-recurrent"}
    assert ("gemm-recurrent", torch.float32, "tf32") in rec and ("gemm-recurrent", torch.bfloat16, "tc") in rec, rec


def test_graph_replay_equals_eager_c5():
    """The C5 step replayed from a captured CUDA graph (restored to the initial state in place) equals the eager step."""
    eager, graph = (run_step(TrainEngineMLP, CFG, BENCH_OPT, CudaKernels("cuda"), C5["T"], C5["B"], 0, use_graph=g,
                             prepare=assert_concurrent)[1] for g in (False, True))
    assert_equal_steps(eager, graph, "C5 graph replay vs eager")


# ------------------------------------------------------------------ F. the whole C5 step against the float64 oracle

@pytest.fixture(scope="module")
def oracle_c5():
    """The oracle's C5 step (reference models/p2p_model.py, Mode A) in float64 on the device, from the engine's initial weights
    and inputs."""
    opt, probs, plan, x, eps = step_inputs(CFG, BENCH_OPT, C5["T"], C5["B"], 0)
    state = {m: {k: v.cuda() for k, v in sd.items()} for m, sd in O.build_state(CFG, seed=1, dtype=torch.float64).items()}
    adam = {m: O.new_adam_state(state[m]) for m in O.MODULES}
    t0 = time.time()
    ref = O.train_step(state, adam, x.double().cuda(), opt, "mlp", eps.double().cuda(), probs, mode="A")
    torch.cuda.synchronize()
    print(f"[oracle] float64 C5 step on the device: {time.time() - t0:.1f} s")
    grads = {m: {k: g.cpu() for k, g in gm.items()} for m, gm in ref["grads"].items()}
    del state, adam
    release()
    return ref["losses"], grads


MODES = [("fp32", torch.float32, 1e-4, 1 - 1e-5, None), ("bf16", torch.bfloat16, 1e-2, 0.995, 0.05)]


@pytest.mark.parametrize("mode", MODES, ids=[m[0] for m in MODES])
def test_c5_step_vs_float64_oracle(oracle_c5, mode):
    """Losses and every gradient tensor of one C5 step against the float64 oracle: fp32 mode to rtol 1e-4 and cosine
    >= 1 - 1e-5 (the thresholds of test_mlp_gpu.py), bf16 mode to rtol 1e-2, cosine >= 0.995 and norm ratio within 5 %
    (test_measured_gpu.py's thresholds for h36m at rnn_size 512)."""
    name, adt, rtol, mincos, norm_tol = mode
    ref_losses, ref_grads = oracle_c5
    opt, probs, plan, x, eps = step_inputs(CFG, BENCH_OPT, C5["T"], C5["B"], 0)
    eng = TrainEngineMLP(O.build_state(CFG, seed=1), CFG, opt, CudaKernels("cuda"), act_dtype=adt)
    got = eng.step(x.cuda(), probs=probs, eps=eps.cuda())
    torch.cuda.synchronize()
    np.testing.assert_allclose(got, np.array(ref_losses), rtol=rtol, atol=1e-7, err_msg=name)
    coss, bad = [], []
    for m in O.MODULES:
        for k, gref in ref_grads[m].items():
            g = eng.arena[m].g[k].detach().double().cpu()
            cos = torch.nn.functional.cosine_similarity(g.flatten(), gref.flatten(), dim=0).item()
            r = g.norm().item() / (gref.norm().item() + 1e-300)
            coss.append((cos, f"{m}.{k}", r))
            if cos < mincos:
                bad.append(f"{name} grad {m}.{k}: cosine {cos:.8f} < {mincos}")
            if norm_tol is not None and abs(r - 1) >= norm_tol:
                bad.append(f"{name} grad {m}.{k}: norm ratio {r:.4f}")
    coss.sort()
    print(f"[oracle] {name}: losses {got} vs {np.array(ref_losses)}; worst cosines "
          + ", ".join(f"{n} {1 - c:.2e} (norm {r:.5f})" for c, n, r in coss[:6]))
    assert not bad, "\n".join(bad)
