"""h36m pose backbone: host-side schedule (p2pvg_b200/engine_mlp.py) on CPU against the oracle."""

import numpy as np
import torch

from oracle import p2p_oracle as O
from p2pvg_b200.engine import StepPlan
from p2pvg_b200.engine_mlp import TrainEngineMLP
from tests.emu_mlp import EmuKernelsMLP
from tests.test_engine_emu import compare as _compare


def compare(*a):
    return _compare(*a, cancelled=lambda m, k: False)  # no BatchNorm in this backbone

CFG = dict(g_dim=128, z_dim=10, rnn_size=64, backbone="mlp", predictor_rnn_layers=2, posterior_rnn_layers=1, prior_rnn_layers=1)


def run(optkw, T, B, np_seed=0, mode="A"):
    torch.set_num_threads(8)   # the split of torch's CPU reductions follows the thread count: the same on every host
    state = O.build_state(CFG, seed=1)
    opt = O.default_opt(**optkw)
    opt["batch_size"] = opt["batch_size"] or B
    eng = TrainEngineMLP(O.clone_state(state), CFG, opt, EmuKernelsMLP("cpu"), mode=mode)
    adam = {m: O.new_adam_state(state[m]) for m in O.MODULES}
    x = torch.randn(T, B, 17, 3, generator=torch.Generator().manual_seed(5))
    np.random.seed(np_seed)
    probs = np.random.uniform(0, 1, T - 1)
    plan = StepPlan(T, probs, opt)
    eps = O.draw_eps(plan.S, B, 10, seed=11)
    ref = O.train_step(state, adam, x, opt, "mlp", eps, probs, mode=mode)
    got = eng.step(x, probs=probs, eps=eps)
    return ref, got, eng, state


def test_mlp_plain():
    compare(*run({}, T=6, B=5))


def test_mlp_skip_and_last_frame_skip():
    ref, got, eng, state = run(dict(skip_prob=0.5, n_past=2, last_frame_skip=True), T=9, B=3, np_seed=3)
    assert eng.last_plan.S < 8 and eng.last_plan.nskip > 1
    compare(ref, got, eng, state)


def test_mlp_mode_b():
    compare(*run(dict(skip_prob=0.4), T=7, B=4, np_seed=1, mode="B"))
