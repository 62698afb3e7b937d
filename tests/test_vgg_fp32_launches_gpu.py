"""The fp32 vgg_64 / vgg_128 training steps' kernel launches against float64 (P2PVG_PRECISION=fp32, the mode that gives
reference-level vgg gradients), at the shapes of the C3 benchmark configuration (vgg_64, T = 30, B = 128) and of vgg_128
(T = 30, B = 32).

In fp32 every 3x3 convolution is im2col3 -> gemm_simt (-> gather_add of the fp32 skip half), every data gradient im2col3 of
dy with mirrored taps -> gemm_simt, every weight gradient a CUDA-core GEMM over all pixels (split-K).  At C3 the vgg_col
buffer of a 64x64x64 layer holds 15.7M rows of pitch 576: 9.06e9 elements, past 2^33.

A whole eager fp32 step does not fit in 80 GB at C3 or at vgg_128 B = 32 (vgg_col plus vgg_dcol alone come to about 67 GiB
at those shapes; vgg_64 at B = 64 does not fit either), so
  A. the fp32 launch list tests/vgg_ref.py derives (precision "fp32") is compared with a recorded eager step at B = 32
     (vgg_64) and B = 8 (vgg_128), T = 30, and the step's peak device memory is printed;
  B. every distinct GEMM of the C3 and vgg_128 lists runs at its exact shape, with only its own operands allocated, against
     float64 (launch_audit.gemm32_at_shape);
  C. im2col3 bit-exact at the largest 64-channel launches of C3 and vgg_128 (9.06e9 elements, both tap signs), and the
     fp32 ends and skip gathers of vgg_128 (im2col3 / col2im3 of the 3-channel frames, gather_add / group_sum / add_indexed
     over 128x128x64 groups);
  E. audited fp32 steps at T = 30, at half the recorded step's batch (vgg_64 B = 16, vgg_128 B = 4: the audit also holds the
     plain step's results, 0 / 1 copies of every probed GEMM's operands and float64 references; it peaks at 27.7 / 31.6 GiB
     there, where the recorded step alone takes 50.2 / 51.2 GiB at twice the batch): every GEMM on the SIMT
     bound, im2col3 / col2im3 / gather_add / group_sum / add_indexed, pooling, upsampling and every BatchNorm entry point
     checked against float64 as they run, every skip gather reading plan.skip_src, bit-identical to the plain serial step
     and to its graph replay;
  F. a whole fp32 vgg_64 step at the audit batch (T = 30, B = 16) against the float64 oracle on the device (the oracle took
     5.0 s on an H100 80GB HBM3 at 700 W; the time is printed).
"""
import time

import numpy as np
import pytest
import torch

from oracle import p2p_oracle as O
from p2pvg_b200._lib import CudaKernels
from p2pvg_b200.engine import StepPlan
from p2pvg_b200.engine_vgg import TrainEngineVGG
from tests.launch_audit import K, memory_per_test  # noqa: F401  (fixtures)
from tests.launch_audit import (BENCH_OPT, SENTINEL, SKIP_OPT, SimtAudit, assert_equal_steps, assert_serial, audit_step,
                                gemm32_at_shape, gemm_ws_bytes, kernel_for, recorded_fp32_step, release, run_step, skip_seed,
                                step_inputs)
from tests.vgg_ref import (VggAudit, backward_launches, forward_launches, im2col3_ref, run_im2col3_col2im3, run_skip_index, vgg_cfg,
                           vgg_tables)

pytestmark = pytest.mark.gpu

T = 30
SHAPES = {"C3": dict(W0=64, B=128), "vgg128": dict(W0=128, B=32)}
LIST_B = {"C3": 32, "vgg128": 8}


def launches(name, B=None):
    c = SHAPES[name]
    p = StepPlan(T, np.zeros(T - 1), O.default_opt(**BENCH_OPT))
    B = B or c["B"]
    return (forward_launches(T, B, p.S, p.nskip, c["W0"], "fp32")
            + backward_launches(T, B, p.S, p.nskip, c["W0"], p.has_cpc, "fp32"))


# ------------------------------------------------------------------ A. the launch lists

@pytest.mark.parametrize("name", list(SHAPES))
def test_fp32_launch_list_matches_an_eager_step(name):
    """The derived fp32 list equals, call for call and in order, the backbone launches of one eager fp32 step, which runs
    serially."""
    c, B = SHAPES[name], LIST_B[name]
    plan, got, peak = recorded_fp32_step(TrainEngineVGG, vgg_cfg(c["W0"]), BENCH_OPT, T, B)
    L = launches(name, B)
    want = [e["key"] for e in L]
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, f"{name}: launch {i} is {g}, the derived list says {w} ({L[i]['name']})"
    assert len(got) == len(want), f"{name}: {len(got)} launches recorded, {len(want)} derived"
    print(f"[list] {name} fp32 B={B}: {len(got)} launches, in order; peak device memory of the step {peak:.2f} GiB")


# ------------------------------------------------------------------ B. every distinct GEMM at its exact shape

def _distinct_gemms():
    seen, out = set(), []
    for n in SHAPES:
        for e in launches(n):
            if e["op"] == "gemm" and e["key"] not in seen:
                seen.add(e["key"])
                out.append((n, e))
    return out


GEMMS = _distinct_gemms()


@pytest.mark.parametrize("cfg,e", GEMMS, ids=[f"{n}-{e['name'].replace(' ', '_')}-{e['M']}x{e['N']}x{e['K']}" for n, e in GEMMS])
def test_fp32_gemm_at_launch_shape(K, cfg, e):
    gemm32_at_shape(K, e, e["M"] * 5 + e["N"] * 3 + e["K"], cfg)


def test_fp32_gemm_coverage():
    """The C3 64x64x64 layers: forward over a [15.7M, 576] col operand (9.06e9 elements) and their weight gradient
    64 x 576 over 15.7M pixels in 33 splits."""
    geo = {(n, e["M"], e["N"], e["K"], e["a_mn"]) for n, e in GEMMS}
    assert ("C3", 3840 * 64 * 64, 64, 576, False) in geo and ("C3", 64, 576, 3840 * 64 * 64, True) in geo
    assert kernel_for(64, 576, 3840 * 64 * 64, True, True, 64, 576, 0, 0, False)[1] == 33


# ------------------------------------------------------------------ C. the lowering at the 64-channel and vgg_128 shapes

def _largest_im2col3():
    """Per list and tap sign, the im2col3 launch of >= 64 channels with the most output elements."""
    out = []
    for n in SHAPES:
        for sgn in (1, -1):
            L = [e["args"] for e in launches(n) if e["op"] == "im2col3" and e["args"][2] >= 64 and e["args"][4] == sgn]
            out.append((n,) + max(L, key=lambda a: a[0] * a[1] * a[1] * a[3]))
    return out


IM2COL3 = _largest_im2col3()


@pytest.mark.parametrize("case", IM2COL3, ids=[f"{c[0]}-N{c[1]}_{c[2]}x{c[2]}x{c[3]}_ld{c[4]}_sgn{c[5]}" for c in IM2COL3])
def test_im2col3_largest_launch(K, case):
    """im2col3 over a whole 64-channel launch (9.06e9 output elements at C3 and at vgg_128 B = 32), bit-exact against the
    gather chunk by chunk of images, nothing written past the end."""
    cfg, N, H, C, ld, sgn = case
    assert N * H * H * ld > 1 << 33
    x = torch.randn(N * H * H * C, device="cuda")
    n = N * H * H * ld
    col = torch.full((n + 64,), SENTINEL, device="cuda")
    K.im2col3(x, col, N, H, H, C, ld, sgn)
    torch.cuda.synchronize()
    assert (col[n:] == SENTINEL).all(), "im2col3 wrote past its output"
    xv, cv = x.view(N, H, H, C), col[:n].view(N * H * H, ld)
    per = max(1, (1 << 27) // (H * H * ld))
    for n0 in range(0, N, per):
        k = min(per, N - n0)
        assert torch.equal(cv[n0 * H * H:(n0 + k) * H * H], im2col3_ref(xv[n0:n0 + k], k, H, H, C, sgn, ld)), \
            f"{cfg} im2col3 sgn={sgn} images [{n0}, {n0 + k})"
    print(f"[exact] {cfg} im2col3 N={N} {H}x{H}x{C} ld={ld} sgn={sgn}: {n} elements ({n / 2 ** 33:.3f} x 2^33), bit-exact")


def test_fp32_vgg128_ends(K):
    """The fp32 3-channel ends of vgg_128 over all T B = 960 frames: im2col3 of the frames (row32 and generic paths, both tap
    signs) bit-exact, col2im3 of the last layer within 9 fp32 adds."""
    c = SHAPES["vgg128"]
    run_im2col3_col2im3(K, T * c["B"], c["W0"], torch.float32, "vgg128 fp32 ends")


def test_fp32_vgg128_skip_gathers(K):
    """gather_add of the fp32 skip half, group_sum of its gradient and add_indexed into the encoder at vgg_128's largest
    stage (30 groups of 32 x 128 x 128 x 64, three skip sources), against float64."""
    c = SHAPES["vgg128"]
    ga = [e["args"] for e in launches("vgg128") if e["op"] == "gather_add"]
    assert (T, c["B"] * 128 * 128 * 64) in ga
    run_skip_index(K, T, c["B"], 128, 64, torch.float32, True)


# ------------------------------------------------------------------ E. audited steps

class VggFp32Audit(SimtAudit, VggAudit):
    """VggAudit's lowering, pooling and skip-gather checks with SimtAudit's GEMM bound and BatchNorm checks; every fp32 skip
    gather logs the source table it read."""
    PRINT_RECORDS = False
    REPORT_GEMMS_ONLY = True

    def gather_add(self, dst, src, grp_src, G, n):
        self.skip_reads.append(grp_src.tolist()[:G])
        super().gather_add(dst, src, grp_src, G, n)


AUDIT = [("vgg64_bench_options", 64, BENCH_OPT, 16), ("vgg64_skip_lfs", 64, SKIP_OPT, 16), ("vgg128_bench_options", 128, BENCH_OPT, 4)]


@pytest.mark.parametrize("case", AUDIT, ids=[c[0] for c in AUDIT])
def test_audit_fp32_vgg_step(case):
    name, W0, optkw, B = case
    audit = VggFp32Audit("cuda")

    def expect(plan):
        L = (forward_launches(T, B, plan.S, plan.nskip, W0, "fp32") + backward_launches(T, B, plan.S, plan.nskip, W0, plan.has_cpc, "fp32"))
        want = {("maxpool2_fwd",), ("maxpool2_bwd",), ("upsample2_fwd",), ("upsample2_bwd",), ("group_sum",), ("add_indexed",),
                ("col2im3",), ("gather_add",), ("bn_fwd_stats",), ("bn_act", 1), ("bn_act", 2), ("bn_bwd", 1), ("bn_bwd", 2),
                ("bn_param_grad",), ("im2col3", "row32", 1), ("im2col3", "generic", 1), ("im2col3", "generic", -1)}
        for e in L:
            if e["op"] == "gemm":
                kern = kernel_for(e["M"], e["N"], e["K"], e["a_mn"], e["b_mn"], e["lda"], e["ldb"], 0, 0, False, gemm_ws_bytes(audit))
                want.add(("gemm", kern if isinstance(kern, str) else kern[0], e["a_mn"], e["b_mn"], e["bias"]))
        assert ("gemm", "simt-splitK", True, True, False) in want
        gathers = sum(1 for e in L if e["op"] == "gather_add")
        assert gathers == len(vgg_tables(W0)[1])   # one per decoder stage entry
        return want, [plan.skip_src] * gathers

    plan, plain = audit_step(TrainEngineVGG, vgg_cfg(W0), optkw, T, B, audit, expect, f"{name} fp32", act_dtype=torch.float32)
    np_seed = skip_seed(T) if optkw.get("skip_prob") else 0
    _, graph = run_step(TrainEngineVGG, vgg_cfg(W0), optkw, CudaKernels("cuda"), T, B, np_seed, use_graph=True,
                        act_dtype=torch.float32, prepare=assert_serial)
    assert_equal_steps(plain, graph, f"{name}: graph replay vs eager")


# ------------------------------------------------------------------ F. against the float64 oracle

def test_fp32_vgg64_step_vs_float64_oracle():
    """Losses to rtol 1e-4 and every gradient to cosine >= 1 - 1e-4 against the float64 oracle (DESIGN.md's fp32 vgg
    thresholds), the BatchNorm-cancelled biases exempt; at the vgg_64 audit batch, T = 30."""
    Tf, B = T, AUDIT[0][3]
    cfg = vgg_cfg(64)
    opt, probs, plan, x, eps = step_inputs(cfg, BENCH_OPT, Tf, B, 0)
    state = {m: {k: v.cuda() for k, v in sd.items()} for m, sd in O.build_state(cfg, seed=1, dtype=torch.float64).items()}
    adam = {m: O.new_adam_state(state[m]) for m in O.MODULES}
    t0 = time.time()
    ref = O.train_step(state, adam, x.double().cuda(), opt, "vgg", eps.double().cuda(), probs, mode="A")
    torch.cuda.synchronize()
    print(f"[oracle] float64 vgg_64 T={Tf} B={B} step on the device: {time.time() - t0:.1f} s")
    del state, adam
    release()
    eng = TrainEngineVGG(O.build_state(cfg, seed=1), cfg, opt, CudaKernels("cuda"), act_dtype=torch.float32)
    got = eng.step(x.cuda(), probs=probs, eps=eps.cuda())
    torch.cuda.synchronize()
    np.testing.assert_allclose(got, np.array(ref["losses"]), rtol=1e-4, atol=1e-7)
    worst = []
    for m in O.MODULES:
        for k, gref in ref["grads"][m].items():
            if k.endswith("main.0.bias") or k in ("c5.0.bias", "upc1.0.bias"):
                continue   # bias in front of a training-mode BatchNorm: exactly-zero true gradient (test_vgg_gpu.py)
            g = eng.arena[m].g[k].detach().double()
            cos = torch.nn.functional.cosine_similarity(g.flatten(), gref.flatten().to(g.device), dim=0).item()
            worst.append((cos, f"{m}.{k}"))
    worst.sort()
    print(f"[oracle] vgg_64: losses {got} vs {np.array(ref['losses'])}; worst cosines "
          + ", ".join(f"{n} {1 - cs:.2e}" for cs, n in worst[:5]))
    bad = [f"{n}: cosine {cs:.8f}" for cs, n in worst if cs < 1 - 1e-4]
    assert not bad, "\n".join(bad)
