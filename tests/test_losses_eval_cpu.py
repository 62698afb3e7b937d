"""Held-out scoring (P2PModel.p2p_losses) without a GPU: the eval-mode restatement against the reference's own eval-mode
forward (tests/golden/losses_eval.pt), the engines' evaluate_losses schedule through the emulated kernels against that
restatement for every backbone, and the argument checks."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import p2p_oracle as O
from p2pvg_b200.engine import StepPlan, TrainEngine
from p2pvg_b200.engine_mlp import TrainEngineMLP
from p2pvg_b200.engine_vgg import TrainEngineVGG
from tests.emu_seq_losses import EmuKernelsEval, EmuKernelsMLPEval, EmuKernelsVGGEval
from tests.loss_eval_ref import forward_losses_eval

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "losses_eval.pt")
FIX = torch.load(GOLDEN, weights_only=False)


def fixture_inputs(fx):
    """(state with the fixture's BatchNorm buffers, x, width tag) of a losses_eval.pt case."""
    state = O.build_state(fx["cfg"], seed=fx["init_seed"])
    for m, bufs in fx["bn_buffers"].items():
        for k, v in bufs.items():
            state[m][k] = v.clone()
    if "x" in fx:
        x = fx["x"]
    else:
        x = torch.rand(*fx["x_shape"], generator=torch.Generator().manual_seed(fx["x_seed"]))
    cfg = fx["cfg"]
    width = {"mlp": "mlp", "vgg": "vgg"}.get(cfg["backbone"], cfg["image_width"])
    return state, x, width


@pytest.mark.parametrize("case", sorted(FIX))
def test_eval_oracle_reproduces_reference(case):
    torch.set_num_threads(8)
    fx = FIX[case]
    state, x, width = fixture_inputs(fx)
    ref = forward_losses_eval(state, x, fx["opt"], width, fx["eps"], fx["probs"].numpy())
    np.testing.assert_allclose(ref["losses"], fx["losses"], rtol=2e-5, atol=1e-9)
    # the executed steps and their time counters, as the reference's posterior received them (fp32 fill_ of the doubles)
    assert len(ref["steps"]) == len(fx["counters"])
    got = torch.tensor([[tuc, dt] for _, tuc, dt in ref["steps"]], dtype=torch.float32)
    assert torch.equal(got, fx["counters"])


ENGINES = {"dcgan": (TrainEngine, EmuKernelsEval), "vgg": (TrainEngineVGG, EmuKernelsVGGEval), "mlp": (TrainEngineMLP, EmuKernelsMLPEval)}


def emu_engine(fx, state):
    cfg = dict(fx["cfg"])
    cls, kern = ENGINES[cfg["backbone"]]
    opt = dict(fx["opt"])
    return cls(O.clone_state(state), cfg, opt, kern("cpu"))


def snapshot(eng):
    return [t.clone() for t in (eng.pool["flat"], eng.pool["grad"], eng.pool["m"], eng.pool["v"])] + \
        [eng.arena[m].step_t.clone() for m in eng.arena] + [v.clone() for m in eng.buffers for v in eng.buffers[m].values()]


@pytest.mark.parametrize("case", sorted(FIX))
def test_evaluate_losses_emulated_matches_oracle(case):
    """The engines' eval-mode schedule (eval BatchNorm coefficients, no statistics, no update) through the emulated kernels
    gives the restatement's scalars and per-row values, leaves every arena, step counter and buffer as it was, and its
    per-row values add up to the scalars."""
    torch.set_num_threads(8)
    fx = FIX[case]
    state, x, width = fixture_inputs(fx)
    ref = forward_losses_eval(state, x, fx["opt"], width, fx["eps"], fx["probs"].numpy())
    eng = emu_engine(fx, state)
    before = snapshot(eng)
    plan, per, out = eng.evaluate_losses(x, probs=fx["probs"].numpy(), eps=fx["eps"])
    # fp32 layers summed in another order: KL (a sum of nearly cancelling terms, ~1e-4 here) is held to an absolute 1e-7
    np.testing.assert_allclose(out.numpy(), ref["losses"], rtol=1e-4, atol=1e-7)
    np.testing.assert_allclose(out.numpy(), fx["losses"], rtol=1e-4, atol=1e-7)
    np.testing.assert_allclose(per.numpy(), ref["per_seq"].double().numpy(), rtol=1e-4, atol=1e-7)
    assert per.dtype == out.dtype == torch.float64 and tuple(per.shape) == (4, x.shape[1])
    np.testing.assert_allclose([per[0].mean(), per[1].sum(), per[2].mean(), per[3].mean()], out.numpy(), rtol=1e-12)
    assert plan.tgt_frame == [i for i, _, _ in ref["steps"]]
    for a, b in zip(before, snapshot(eng)):
        assert torch.equal(a, b)


def test_kld_divides_by_configured_batch():
    """h36m: B = 10 rows under opt.batch_size = 16 -- the per-row KL shares are row sums / 16."""
    fx = FIX["h36m_mlp"]
    assert fx["opt"]["batch_size"] == 16 and fx["x"].shape[1] == 10
    state, x, width = fixture_inputs(fx)
    eng = emu_engine(fx, state)
    _, per, _ = eng.evaluate_losses(x, probs=fx["probs"].numpy(), eps=fx["eps"])
    opt10 = dict(fx["opt"], batch_size=10)
    _, per10, _ = TrainEngineMLP(O.clone_state(state), fx["cfg"], opt10, EmuKernelsMLPEval("cpu")).evaluate_losses(
        x, probs=fx["probs"].numpy(), eps=fx["eps"])
    np.testing.assert_allclose(per[1].numpy() * 16, per10[1].numpy() * 10, rtol=1e-12)
    np.testing.assert_allclose(per[0].numpy(), per10[0].numpy(), rtol=0)


def test_replayed_skip_pattern_tables():
    """Two skip patterns of one signature (same T, S, distinct-skip count) differ only in the index tables."""
    opt = O.default_opt(skip_prob=0.5, batch_size=2)
    a, b = StepPlan(8, np.array([0.9, 0.1, 0.9, 0.9, 0.9, 0.9, 0.9]), opt), StepPlan(8, np.array([0.9, 0.9, 0.1, 0.9, 0.9, 0.9, 0.9]), opt)
    assert a.key == b.key and a.tgt_frame != b.tgt_frame


def _model(training):
    from p2pvg_b200.models import dcgan_64
    from p2pvg_b200.models.p2p_model import P2PModel
    opt = types.SimpleNamespace(dataset="mnist", backbone_net=dcgan_64, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0,
                                weight_align=0.5, skip_prob=0.5, n_past=1, last_frame_skip=False, batch_size=2)
    m = P2PModel(2, 1, 128, 10, 256, 1, 1, 2, opt=opt)
    return m.train() if training else m.eval()


@pytest.mark.parametrize("what,message", [("training", "needs every module in eval mode"),
                                          ("partly_training", "needs every module in eval mode"),
                                          ("cpu", "runs on a CUDA device"), ("short", "T >= 2 frames")])
def test_p2p_losses_rejections_before_any_draw(what, message):
    model = _model(what == "training")
    if what == "partly_training":
        model.decoder.train()
    x = torch.rand(1 if what == "short" else 4, 2, 1, 64, 64)
    st, rng = np.random.get_state(), torch.get_rng_state()
    with pytest.raises(ValueError, match=message):
        model.p2p_losses(x)
    assert torch.equal(torch.get_rng_state(), rng)
    st2 = np.random.get_state()
    assert st[0] == st2[0] and np.array_equal(st[1], st2[1]) and st[2:] == st2[2:]
    assert model._engine is None


def test_eval_buffers_leave_step_graphs_valid():
    """Held-out calls that grow from call to call -- in T, in B, and in executed steps beyond any the training steps had --
    never re-allocate a buffer the step may have captured: graph_generation() and every step buffer stay as they were."""
    torch.set_num_threads(8)
    cfg = dict(g_dim=128, z_dim=10, rnn_size=64, channels=1, image_width=64, predictor_rnn_layers=2, posterior_rnn_layers=1,
               prior_rnn_layers=1)
    opt = O.default_opt(skip_prob=0.5, batch_size=3)
    state = O.build_state(cfg, seed=1)
    eng = TrainEngine(O.clone_state(state), cfg, opt, EmuKernelsEval("cpu"))
    gen = torch.Generator().manual_seed(2)
    probs_train = np.array([0.9, 0.1, 0.1, 0.9, 0.9, 0.9, 0.9])   # T = 8 with two skipped steps: S = 5
    eng.step(torch.rand(8, 3, 1, 64, 64, generator=gen), probs=probs_train, eps=O.draw_eps(5, 3, 10, seed=1))
    gen0, bufs0 = eng.graph_generation(), dict(eng._bufs)
    for T, B in ((4, 2), (6, 2), (8, 3)):   # growing held-out batches, the last one without skips (S = 7 > 5)
        probs = np.full(T - 1, 0.9)
        eng.evaluate_losses(torch.rand(T, B, 1, 64, 64, generator=gen), probs=probs, eps=O.draw_eps(T - 1, B, 10, seed=T))
        assert eng.graph_generation() == gen0
        assert all(eng._bufs[k] is t for k, t in bufs0.items())
    # a step after them still matches the oracle
    x = torch.rand(8, 3, 1, 64, 64, generator=gen)
    eps = O.draw_eps(5, 3, 10, seed=7)
    got = eng.step(x, probs=probs_train, eps=eps)
    ref_state = O.clone_state(state)
    adam = {m: O.new_adam_state(ref_state[m]) for m in O.MODULES}
    O.train_step(ref_state, adam, torch.rand(8, 3, 1, 64, 64, generator=torch.Generator().manual_seed(2)), opt, 64,
                 O.draw_eps(5, 3, 10, seed=1), probs_train)
    ref = O.train_step(ref_state, adam, x, opt, 64, eps, probs_train)
    np.testing.assert_allclose(got, np.array(ref["losses"], dtype=np.float32), rtol=1e-4, atol=1e-7)
