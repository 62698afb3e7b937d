"""Parity of the CUDA train step (through the C ABI) with the CPU oracle and with the golden fixtures
written by the unmodified reference.  Tolerances: fp32 path — losses rtol 1e-4, gradient cosine >= 1-1e-5;
bf16 tensor-core path — losses rtol 2e-2, gradient cosine >= 0.995 (bf16 operands, fp32 accumulation).
Index / time-counter logic is bit-exact (tests/test_oracle_golden.py, tests/test_engine_emu.py)."""
import glob
import os

import numpy as np
import pytest
import torch

from oracle import p2p_oracle as O
from p2pvg_b200.engine import StepPlan, TrainEngine
from tests.test_engine_emu import CFG64, bn_cancelled_bias
from tests.test_oracle_golden import load_fixture

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def make_engine(state, cfg, opt, act_dtype, gemm="auto", mode="A"):
    from p2pvg_b200._lib import CudaKernels
    K = CudaKernels("cuda")
    K.set_gemm_impl(gemm)
    return TrainEngine(O.clone_state(state), cfg, opt, K, act_dtype=act_dtype, mode=mode)


def check(ref_losses, ref_grads, got, eng, rtol_loss, min_cos, what=""):
    np.testing.assert_allclose(got, np.array(ref_losses, dtype=np.float32), rtol=rtol_loss, atol=1e-6, err_msg=what)
    for m in O.MODULES:
        gmax = max(g.abs().max().item() for g in ref_grads[m].values())
        for k, gref in ref_grads[m].items():
            g = eng.arena[m].g[k].detach().cpu()
            if bn_cancelled_bias(m, k):
                assert g.abs().max().item() <= 3e-2 * gmax, f"{what} grad {m}.{k} should be ~0"
                continue
            cos = torch.nn.functional.cosine_similarity(g.flatten().double(), gref.flatten().double(), dim=0).item()
            assert cos >= min_cos, f"{what} grad {m}.{k}: cosine {cos:.6f}"
            r = g.norm().item() / (gref.norm().item() + 1e-30)
            assert abs(r - 1) < 50 * (1 - min_cos) + 1e-3, f"{what} grad {m}.{k}: norm ratio {r:.5f}"


CASES = [
    ("plain", CFG64, {}, 5, 3),
    ("skip", CFG64, dict(skip_prob=0.5), 8, 2),
    ("lfs", CFG64, dict(skip_prob=0.5, n_past=2, last_frame_skip=True), 7, 2),
    ("d128", dict(CFG64, channels=3, image_width=128), {}, 4, 2),
]


def inputs(name, cfg, opt, T, B):
    x = torch.rand(T, B, cfg["channels"], cfg["image_width"], cfg["image_width"], generator=torch.Generator().manual_seed(5))
    np.random.seed(5 if name == "lfs" else 0)
    probs = np.random.uniform(0, 1, T - 1)
    plan = StepPlan(T, probs, opt)
    eps = O.draw_eps(plan.S, B, cfg["z_dim"], seed=11)
    return x, probs, eps


@pytest.mark.parametrize("name,cfg,optkw,T,B", CASES)
def test_step_fp32_vs_oracle(name, cfg, optkw, T, B):
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    state = O.build_state(cfg, seed=1)
    opt = O.default_opt(**optkw)
    opt["batch_size"] = opt["batch_size"] or B
    eng = make_engine(state, cfg, opt, torch.float32)
    adam = {m: O.new_adam_state(state[m]) for m in O.MODULES}
    x, probs, eps = inputs(name, cfg, opt, T, B)
    ref = O.train_step(state, adam, x, opt, cfg["image_width"], eps, probs, mode="A")
    got = eng.step(x.cuda(), probs=probs, eps=eps.cuda())
    check(ref["losses"], ref["grads"], got, eng, 1e-4, 1 - 1e-5, what=f"{name}/fp32")
    for m in O.MODULES:  # post-step weights: Adam moves every element by ~lr*sign(g)
        for k, v in state[m].items():
            if O.is_param(k):
                dw = (eng.arena[m].p[k].cpu() - v).abs().max().item()
                assert dw <= 2.2e-3, f"weight {m}.{k} {dw}"
            elif v.is_floating_point():
                assert torch.allclose(eng.buffers[m][k].cpu(), v, rtol=1e-4, atol=1e-6), f"buffer {m}.{k}"
            else:
                assert torch.equal(eng.buffers[m][k].cpu(), v)


# batch >= 4: with 2 samples per BatchNorm group the normalised latent is exactly +-1, its input gradient is
# identically zero and what is left is rounding noise whose sign is arbitrary in bf16
CASES_BF16 = [(n, c, o, t, max(b, 4)) for n, c, o, t, b in CASES]


@pytest.mark.parametrize("name,cfg,optkw,T,B", CASES_BF16)
@pytest.mark.parametrize("gemm", ["simt", "tc"])
def test_step_bf16_vs_emulation(name, cfg, optkw, T, B, gemm):
    """bf16 path (CUDA-core GEMM and tensor-core wgmma GEMM) against the torch emulation run with the same bf16
    rounding points: isolates kernel errors from bf16 storage noise."""
    from tests.emu_backend import EmuKernels
    state = O.build_state(cfg, seed=1)
    opt = O.default_opt(**optkw)
    opt["batch_size"] = opt["batch_size"] or B
    eng = make_engine(state, cfg, opt, torch.bfloat16, gemm)
    if gemm == "tc":
        assert eng.K.has_tc_gemm(), "tensor-core GEMM unavailable on this device"
    emu = TrainEngine(O.clone_state(state), cfg, opt, EmuKernels("cuda"), act_dtype=torch.bfloat16)
    x, probs, eps = inputs(name, cfg, opt, T, B)
    try:
        got = eng.step(x.cuda(), probs=probs, eps=eps.cuda())
    finally:
        eng.K.set_gemm_impl("auto")
    want = emu.step(x.cuda(), probs=probs, eps=eps.cuda())
    grads = {m: {k: emu.arena[m].g[k].detach().cpu() for k in emu.arena[m].names} for m in O.MODULES}
    check(tuple(float(v) for v in want), grads, got, eng, 5e-3, 0.99, what=f"{name}/bf16-{gemm}")


@pytest.mark.parametrize("gemm", ["simt", "tc"])
def test_step_bf16_vs_oracle(gemm):
    """bf16 tensor-core path against the fp32 oracle at a batch where bf16 storage noise averages out."""
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    cfg, T, B = CFG64, 5, 16
    state = O.build_state(cfg, seed=1)
    opt = O.default_opt(batch_size=B)
    eng = make_engine(state, cfg, opt, torch.bfloat16, gemm)
    adam = {m: O.new_adam_state(state[m]) for m in O.MODULES}
    x, probs, eps = inputs("plain", cfg, opt, T, B)
    ref = O.train_step(state, adam, x, opt, 64, eps, probs, mode="A")
    try:
        got = eng.step(x.cuda(), probs=probs, eps=eps.cuda())
    finally:
        eng.K.set_gemm_impl("auto")
    check(ref["losses"], ref["grads"], got, eng, 2e-2, 0.98, what=f"oracle/bf16-{gemm}")


def digest_close(t, d, rtol, what):
    f = t.detach().double().reshape(-1).cpu()
    assert f.numel() == d["numel"]
    scale = max(d["absmax"], 1e-30)
    err = (f[d["idx"]] - d["samples"]).abs().max().item()
    assert err <= rtol * scale, f"{what}: {err:.3e} vs scale {scale:.3e}"
    assert abs(float(f.norm()) - d["l2"]) <= rtol * max(d["l2"], 1e-30), what


# the dcgan fixtures; vgg64_rgb and h36m_mlp are replayed by tests/test_vgg_gpu.py / tests/test_mlp_gpu.py
@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(GOLD, "step_d*.pt"))), ids=lambda p: os.path.basename(p)[5:-3])
def test_step_vs_reference_golden(path):
    """fp32 CUDA path against numbers produced by the reference's own P2PModel.forward."""
    fix = load_fixture(path)
    cfg, opt = fix["cfg"], dict(fix["opt"])
    state = O.build_state(cfg, seed=fix["init_seed"])
    eng = make_engine(state, cfg, opt, torch.float32)
    rec = fix["steps"][0]
    got = eng.step(rec["x"].cuda(), probs=rec["probs"].numpy(), eps=rec["eps"].cuda())
    np.testing.assert_allclose(got, np.array(rec["losses"], dtype=np.float32), rtol=1e-4, atol=1e-7)
    posts = [r for r in rec["tape"] if r["m"] == "posterior"]
    S, B, z = eng.S, eng.B, eng.z
    mu = eng.mu[:S * B * z].reshape(S, B, z).cpu()
    for s in range(S):
        assert torch.allclose(mu[s], posts[s]["mu"], rtol=1e-3, atol=1e-5)
    for m, digs in rec["grad_digest"].items():
        for k, d in digs.items():
            if bn_cancelled_bias(m, k):
                continue
            digest_close(eng.arena[m].g[k], d, 2e-2 if m in ("encoder", "decoder") else 2e-3, f"grad {m}.{k}")
    for m, bufs in rec["bn_buffers"].items():
        for k, v in bufs.items():
            b = eng.buffers[m][k].cpu()
            assert torch.allclose(b.double(), v.double(), rtol=1e-4, atol=1e-6), f"{m}.{k}"
