"""Host-side schedule (p2pvg_b200/engine.py) validated on CPU against the oracle, with the torch
emulation of the kernel ABI standing in for the CUDA library (tests/emu_backend.py)."""

import numpy as np
import pytest
import torch

from oracle import p2p_oracle as O
from p2pvg_b200.engine import TrainEngine, StepPlan
from tests.emu_backend import EmuKernels

CFG64 = dict(g_dim=128, z_dim=10, rnn_size=256, channels=1, image_width=64, predictor_rnn_layers=2,
             posterior_rnn_layers=1, prior_rnn_layers=1)


def run_pair(cfg, opt, T, B, steps=1, mode="A", np_seed=0, act_dtype=torch.float32):
    torch.set_num_threads(8)   # the split of torch's CPU reductions follows the thread count: the same on every host
    state = O.build_state(cfg, seed=1)
    opt = O.default_opt(**opt)
    if opt["batch_size"] is None:
        opt["batch_size"] = B
    eng = TrainEngine(O.clone_state(state), cfg, opt, EmuKernels("cpu"), act_dtype=act_dtype, mode=mode)
    adam = {m: O.new_adam_state(state[m]) for m in O.MODULES}
    gen = torch.Generator().manual_seed(5)
    results = []
    for it in range(steps):
        x = torch.rand(T, B, cfg["channels"], cfg["image_width"], cfg["image_width"], generator=gen)
        np.random.seed(np_seed + it)
        probs = np.random.uniform(0, 1, T - 1)
        plan = StepPlan(T, probs, opt)
        eps = O.draw_eps(plan.S, B, cfg["z_dim"], seed=11 + it)
        ref = O.train_step(state, adam, x, opt, cfg["image_width"], eps, probs, mode=mode)
        got = eng.step(x, probs=probs, eps=eps)
        results.append((ref, got, eng, state))
    return results


def bn_cancelled_bias(m, k):
    """Conv / ConvT biases that feed a training-mode BatchNorm have an exactly-zero true gradient; both
    implementations only produce rounding noise there."""
    if m == "encoder":
        return k.endswith(".0.bias")
    if m == "decoder":
        return k.endswith(".0.bias") and not k.startswith(("upc5.0", "upc6.0")) or k == "upc1.0.bias"
    return False


def compare(ref, got, eng, state, rtol_loss=1e-4, rtol_grad=2e-3, lr=1e-3, cancelled=None, cos_tol=1e-5, buf_atol=1e-6, max_bad_frac=0.0):
    bn_cancelled = cancelled if cancelled is not None else bn_cancelled_bias
    np.testing.assert_allclose(got, np.array(ref["losses"], dtype=np.float32), rtol=rtol_loss, atol=1e-7)
    for m in O.MODULES:
        gmax = max(g.abs().max().item() for g in ref["grads"][m].values())
        for k, gref in ref["grads"][m].items():
            g = eng.arena[m].g[k]
            if bn_cancelled(m, k):
                assert g.abs().max().item() <= 1e-4 * gmax, f"grad {m}.{k} should be ~0"
                continue
            scale = gref.abs().max().item() + 1e-12
            bad = ((g - gref).abs() > 10 * rtol_grad * scale).float().mean().item()
            err = (g - gref).abs().max().item() if bad > max_bad_frac else 0.0
            cos = torch.nn.functional.cosine_similarity(g.flatten().double(), gref.flatten().double(), dim=0).item()
            # BatchNorm makes many weight gradients sums of nearly cancelling terms: judge direction tightly
            # (cosine) and the worst element loosely
            assert cos >= 1 - cos_tol and err <= 10 * rtol_grad * scale, f"grad {m}.{k}: cos {cos:.8f} err {err:.3e} scale {scale:.3e}"
        for k, v in state[m].items():
            if O.is_param(k):
                w = eng.arena[m].p[k]
                dw = (w - v).abs()
                # Adam normalises the update to ~lr*sign(g): elements whose gradient is rounding noise may
                # move differently, but never by more than ~2 lr; everything else must agree tightly.
                assert dw.max().item() <= 2.2 * lr, f"weight {m}.{k}"
                gref = ref["grads"][m][k]
                solid = gref.abs() > 3e-2 * (gref.abs().max() + 1e-30)
                if not bn_cancelled(m, k) and solid.any():
                    assert (dw[solid] > 2e-5 + 0.1 * lr).float().mean().item() <= max_bad_frac, f"weight {m}.{k}: {dw[solid].max().item():.3e}"
            elif v.is_floating_point():
                assert torch.allclose(eng.buffers[m][k], v, rtol=1e-4, atol=buf_atol), f"buffer {m}.{k}"
            else:
                assert torch.equal(eng.buffers[m][k], v), f"buffer {m}.{k}"


def test_plain_two_steps():
    # run_pair compares step by step against live state, so evaluate each step right after it ran
    torch.manual_seed(0)
    res = run_pair(CFG64, {}, T=5, B=3, steps=1)
    compare(*res[0])
    res = run_pair(CFG64, {}, T=5, B=3, steps=2)
    ref, got, eng, state = res[1]
    np.testing.assert_allclose(got, np.array(ref["losses"], dtype=np.float32), rtol=2e-3)
    assert eng.arena["encoder"].step_t.item() == 2 and eng.buffers["encoder"]["c1.main.1.num_batches_tracked"].item() == 18


def test_skip_frames():
    (ref, got, eng, state), = run_pair(CFG64, dict(skip_prob=0.5), T=8, B=2, np_seed=0)
    assert eng.last_plan.S < 7
    compare(ref, got, eng, state)


def test_last_frame_skip_n_past2():
    (ref, got, eng, state), = run_pair(CFG64, dict(skip_prob=0.5, n_past=2, last_frame_skip=True), T=7, B=2, np_seed=5)
    assert eng.last_plan.nskip > 1
    compare(ref, got, eng, state)


def test_configured_batch_size_and_mode_b():
    (ref, got, eng, state), = run_pair(CFG64, dict(batch_size=5), T=4, B=2, mode="B")
    compare(ref, got, eng, state)


def test_dcgan128_rgb():
    cfg = dict(CFG64, channels=3, image_width=128)
    (ref, got, eng, state), = run_pair(cfg, {}, T=4, B=2)
    compare(ref, got, eng, state)
