"""vgg_64 backbone: host-side schedule (p2pvg_b200/engine_vgg.py) on CPU against the oracle."""

import numpy as np
import torch

from oracle import p2p_oracle as O
from p2pvg_b200.engine import StepPlan
from p2pvg_b200.engine_vgg import TrainEngineVGG
from tests.emu_vgg import EmuKernelsVGG
from tests.test_engine_emu import compare as _compare


def vgg_cancelled(m, k):
    """Conv biases in front of a training-mode BatchNorm (every vgg layer, c5 and upc1): exactly-zero gradient."""
    return m in ("encoder", "decoder") and (k.endswith("main.0.bias") or k in ("c5.0.bias", "c6.0.bias", "upc1.0.bias"))


def compare(*a, **kw):
    # 23 BatchNorm layers at batch 2-3 amplify fp32 summation-order noise, and among millions of pre-activations a few
    # sit within rounding of zero: their LeakyReLU slope flips between the two implementations and moves one output
    # channel's weight gradient.  Judge direction to 1e-4 and allow 0.5 % of the elements of a tensor to be outliers.
    args = dict(cancelled=vgg_cancelled, cos_tol=1e-4, rtol_grad=2e-3, buf_atol=1e-5, max_bad_frac=5e-3)
    args.update(kw)
    return _compare(*a, **args)


def make_cfg(channels, width=64):
    return dict(g_dim=128, z_dim=10, rnn_size=64, channels=channels, image_width=width, backbone="vgg", predictor_rnn_layers=2,
                posterior_rnn_layers=1, prior_rnn_layers=1)


def run(optkw, T, B, channels=3, np_seed=0, mode="A", width=64):
    torch.set_num_threads(8)   # the split of torch's CPU reductions follows the thread count: the same on every host
    cfg = make_cfg(channels, width)
    state = O.build_state(cfg, seed=1)
    opt = O.default_opt(**optkw)
    opt["batch_size"] = opt["batch_size"] or B
    eng = TrainEngineVGG(O.clone_state(state), cfg, opt, EmuKernelsVGG("cpu"), mode=mode)
    adam = {m: O.new_adam_state(state[m]) for m in O.MODULES}
    x = torch.rand(T, B, channels, width, width, generator=torch.Generator().manual_seed(5))
    np.random.seed(np_seed)
    probs = np.random.uniform(0, 1, T - 1)
    plan = StepPlan(T, probs, opt)
    eps = O.draw_eps(plan.S, B, 10, seed=11)
    ref = O.train_step(state, adam, x, opt, "vgg", eps, probs, mode=mode)
    got = eng.step(x, probs=probs, eps=eps)
    return ref, got, eng, state


def test_vgg_plain_rgb():
    compare(*run({}, T=4, B=2))


def test_vgg_skip_and_last_frame_skip_gray():
    ref, got, eng, state = run(dict(skip_prob=0.5, n_past=2, last_frame_skip=True), T=6, B=2, channels=1, np_seed=3)
    assert eng.last_plan.S < 5 and eng.last_plan.nskip > 1
    compare(ref, got, eng, state)


def test_vgg128_plain_gray():
    """models/vgg_128.py: the 5-stage 128x128 variant through the same schedule."""
    # 29 BatchNorm layers at batch 2: the fp32 summation-order noise floor is ~2x that of vgg_64
    compare(*run({}, T=3, B=2, channels=1, width=128), cos_tol=2e-4, rtol_grad=5e-3, max_bad_frac=2e-2)
