"""Held-out scoring on the GPU: TrainEngine*.evaluate_losses / P2PModel.p2p_losses and the p2pvg_seq_losses kernel."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import p2p_oracle as O
from tests.loss_eval_ref import forward_losses_eval, seq_losses_ref

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "losses_eval.pt")


@pytest.fixture(scope="module")
def K():
    from p2pvg_b200._lib import CudaKernels
    return CudaKernels("cuda:0")


@pytest.fixture(autouse=True)
def exact_reference():
    """The float32 reference on the GPU runs without TF32."""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def engine(K, cfg, opt, state, adt):
    from p2pvg_b200.engine import TrainEngine
    from p2pvg_b200.engine_mlp import TrainEngineMLP
    from p2pvg_b200.engine_vgg import TrainEngineVGG
    cls = {"mlp": TrainEngineMLP, "vgg": TrainEngineVGG}.get(cfg.get("backbone"), TrainEngine)
    return cls(O.clone_state(state), cfg, opt, K, act_dtype=adt)


def width_of(cfg):
    return {"mlp": "mlp", "vgg": "vgg"}.get(cfg.get("backbone"), cfg.get("image_width"))


def restated_seq(eng, plan):
    """p2pvg_seq_losses' float64 restatement on the engine's own buffers of the call just made."""
    rec, sig = eng.decoded()
    return seq_losses_ref(rec, sig, eng.x_nhwc, eng.ix["tgt_idx"], eng.S, eng.B, eng.frame_elems, eng.mu, eng.lv, eng.mu_p, eng.lv_p,
                          eng.z, eng.Hlat, eng.ix["in_idx"], eng.h_pred, eng.g, plan.has_cpc, float(eng.opt["batch_size"]), float(eng.T))


def fixture_inputs(fx):
    state = O.build_state(fx["cfg"], seed=fx["init_seed"])
    for m, bufs in fx["bn_buffers"].items():
        for k, v in bufs.items():
            state[m][k] = v.clone()
    x = fx["x"] if "x" in fx else torch.rand(*fx["x_shape"], generator=torch.Generator().manual_seed(fx["x_seed"]))
    return state, x


FIX = torch.load(GOLDEN, weights_only=False)


@pytest.mark.parametrize("case", sorted(FIX))
def test_fp32_every_backbone_matches_oracle_and_fixture(K, case):
    fx = FIX[case]
    state, x = fixture_inputs(fx)
    ref = forward_losses_eval(state, x, fx["opt"], width_of(fx["cfg"]), fx["eps"], fx["probs"].numpy())
    eng = engine(K, fx["cfg"], dict(fx["opt"]), state, torch.float32)
    plan, per, out = eng.evaluate_losses(x.cuda(), probs=fx["probs"].numpy(), eps=fx["eps"].cuda())
    got = out.cpu().numpy()
    np.testing.assert_allclose(got, ref["losses"], rtol=1e-4, atol=1e-7)
    np.testing.assert_allclose(got, fx["losses"], rtol=1e-4, atol=1e-7)
    rper, rout = restated_seq(eng, plan)
    np.testing.assert_allclose(per.cpu().numpy(), rper.cpu().numpy(), rtol=1e-4, atol=1e-9)
    np.testing.assert_allclose(got, rout.cpu().numpy(), rtol=1e-4, atol=1e-9)
    np.testing.assert_allclose(per.cpu().numpy(), ref["per_seq"].double().numpy(), rtol=1e-4, atol=1e-7)
    p = per.cpu().double()
    np.testing.assert_allclose([p[0].mean(), p[1].sum(), p[2].mean(), p[3].mean()], got, rtol=1e-12)


def random_bn(state, seed):
    """Non-trivial running statistics (eval mode must not look like mean 0 / variance 1)."""
    g = torch.Generator().manual_seed(seed)
    for m in ("encoder", "decoder"):
        for k, v in state[m].items():
            if k.endswith("running_mean"):
                v.copy_(0.1 * torch.randn(v.shape, generator=g))
            elif k.endswith("running_var"):
                v.copy_(0.5 + torch.rand(v.shape, generator=g))
    return state


MEASURED = {
    "d64_T30_B16": (dict(g_dim=128, z_dim=10, rnn_size=256, channels=1, image_width=64), dict(), 30, 16),
    "d64_T30_B16_skip": (dict(g_dim=128, z_dim=10, rnn_size=256, channels=1, image_width=64), dict(skip_prob=0.5), 30, 16),
    "vgg64_T6_B32": (dict(g_dim=128, z_dim=10, rnn_size=256, channels=3, image_width=64, backbone="vgg", vgg_width=64), dict(), 6, 32),
    "h36m_R512_T12_B32": (dict(g_dim=128, z_dim=10, rnn_size=512, backbone="mlp"), dict(skip_prob=0.3), 12, 32),
}


def measured_case(name):
    cfg, optkw, T, B = MEASURED[name]
    cfg = dict(cfg, predictor_rnn_layers=2, posterior_rnn_layers=1, prior_rnn_layers=1)
    state = random_bn(O.build_state(cfg, seed=1), 3)
    opt = O.default_opt(batch_size=B, **optkw)
    gen = torch.Generator().manual_seed(5)
    if cfg.get("backbone") == "mlp":
        x = torch.randn(T, B, 17, 3, generator=gen)
    else:
        x = torch.rand(T, B, cfg["channels"], 64, 64, generator=gen)
    probs = np.random.RandomState(7).uniform(0, 1, T - 1)
    S = len(O.skip_schedule(T, probs, opt["skip_prob"], opt["n_past"]))
    eps = O.draw_eps(S, B, 10, seed=9)
    return cfg, opt, state, x, probs, eps


@pytest.mark.parametrize("name", sorted(MEASURED))
def test_bf16_measured_shapes(K, name):
    cfg, opt, state, x, probs, eps = measured_case(name)
    gstate = {m: {k: v.cuda() for k, v in sd.items()} for m, sd in state.items()}
    ref = forward_losses_eval(gstate, x.cuda(), opt, width_of(cfg), eps.cuda(), probs)
    eng = engine(K, cfg, dict(opt), state, torch.bfloat16)
    if "skip" in name:
        assert len(O.skip_schedule(x.shape[0], probs, opt["skip_prob"], 1)) < x.shape[0] - 1
    plan, per, out = eng.evaluate_losses(x.cuda(), probs=probs, eps=eps.cuda(), use_graph=True)
    np.testing.assert_allclose(out.cpu().numpy(), ref["losses"], rtol=1e-2, atol=1e-6)
    rper, _ = restated_seq(eng, plan)
    np.testing.assert_allclose(per.cpu().numpy(), rper.cpu().numpy(), rtol=1e-4, atol=1e-9)


def test_graph_replay_other_skip_pattern_and_repeat(K):
    """Eager, capture, replay; a second skip pattern of the same signature replays and equals its eager run; two calls with the
    same draws are bit-identical."""
    cfg, opt, state, x, _, _ = measured_case("d64_T30_B16_skip")
    x = x[:8].cuda()
    pa = np.array([0.9, 0.9, 0.1, 0.9, 0.9, 0.9, 0.9])
    pb = np.array([0.9, 0.9, 0.9, 0.1, 0.9, 0.9, 0.9])
    eps = O.draw_eps(6, x.shape[1], 10, seed=4).cuda()
    eng = engine(K, cfg, dict(opt), state, torch.bfloat16)
    for _ in range(3):
        plan_a, per_a, out_a = eng.evaluate_losses(x, probs=pa, eps=eps, use_graph=True)
    assert plan_a.S == 6
    graphs = [v for v in eng._eval_graphs.values() if v != "warm"]
    assert len(graphs) == 1
    plan_b, per_b, out_b = eng.evaluate_losses(x, probs=pb, eps=eps, use_graph=True)
    assert plan_b.key == plan_a.key and plan_b.tgt_frame != plan_a.tgt_frame
    assert [v for v in eng._eval_graphs.values() if v != "warm"] == graphs   # replayed, not captured again
    _, per_e, out_e = eng.evaluate_losses(x, probs=pb, eps=eps, use_graph=False)
    torch.testing.assert_close(out_b, out_e, rtol=1e-6, atol=0)
    torch.testing.assert_close(per_b, per_e, rtol=1e-6, atol=0)
    _, per_b2, out_b2 = eng.evaluate_losses(x, probs=pb, eps=eps, use_graph=True)
    assert torch.equal(out_b, out_b2) and torch.equal(per_b, per_b2)
    assert not torch.equal(out_a, out_b)


def make_model(seed=1):
    from p2pvg_b200.models import dcgan_64
    from p2pvg_b200.models.p2p_model import P2PModel
    opt = types.SimpleNamespace(dataset="mnist", backbone_net=dcgan_64, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0,
                                weight_align=0.5, skip_prob=0.0, n_past=1, last_frame_skip=False, batch_size=4)
    torch.manual_seed(seed)
    return P2PModel(4, 1, 128, 10, 256, 1, 1, 2, opt=opt).cuda()


def model_state(model):
    out = []
    for m in ("frame_predictor", "posterior", "prior", "encoder", "decoder"):
        mod = getattr(model, m)
        out += [t.detach().clone() for t in mod.state_dict().values()]
        out += [p.grad.detach().clone() for p in mod.parameters() if p.grad is not None]
        osd = getattr(model, m + "_optimizer").state_dict()
        for st in osd["state"].values():
            out += [st["exp_avg"].clone(), st["exp_avg_sq"].clone(), torch.tensor(float(st["step"]))]
    return out


def test_p2p_losses_leaves_training_untouched():
    """Every parameter, gradient, Adam moment and step and BatchNorm buffer is unchanged; the captured training graph is
    replayed afterwards (no re-capture); with injected draws, forward after p2p_losses equals forward alone, bit for bit."""
    T, B = 6, 4
    gen = torch.Generator().manual_seed(3)
    batches = [torch.rand(T, B, 1, 64, 64, generator=gen).cuda() for _ in range(4)]
    held_out = torch.rand(T, B - 1, 1, 64, 64, generator=gen).cuda()
    models = [make_model(), make_model()]
    results = []
    for idx, model in enumerate(models):
        model.train()
        for it in range(3):
            np.random.seed(100 + it)
            torch.manual_seed(200 + it)
            model(batches[it])
        eng = model._engine
        graphs = {k: v for k, v in eng._graphs.items() if v != "warm"}
        assert len(graphs) == 1, "the training graph of the one signature was captured"
        gen0 = eng.graph_generation()
        if idx == 0:
            model.eval()
            before = model_state(model)
            # held-out batches growing from call to call (shorter and narrower first), all no larger than the training batch
            v2 = model.p2p_losses(held_out[:T - 2, :2])
            assert eng.graph_generation() == gen0
            v = model.p2p_losses(held_out)
            assert eng.graph_generation() == gen0
            model.p2p_losses(held_out)   # captured, then replayed
            model.p2p_losses(held_out)
            assert eng.graph_generation() == gen0
            assert all(eng._graphs.get(k) is g for k, g in graphs.items())
            after = model_state(model)
            assert len(before) == len(after) and all(torch.equal(a, b) for a, b in zip(before, after))
            assert set(v) == {"mse", "kld", "cpc", "align", "per_sequence", "steps"}
            assert all(v["per_sequence"][k].shape == (B - 1,) and v["per_sequence"][k].dtype == torch.float64 for k in ("mse", "kld", "cpc", "align"))
            assert v["steps"][0] == 1 and v["steps"][-1] == T - 1 and all(np.isfinite([v[k] for k in ("mse", "kld", "cpc", "align")]))
            assert v2["per_sequence"]["mse"].shape == (2,) and v2["steps"] == list(range(1, T - 2))
            model.train()
        np.random.seed(300)
        torch.manual_seed(400)
        losses = model(batches[3])
        torch.cuda.synchronize()
        assert eng.graph_generation() == gen0
        now = {k: v for k, v in eng._graphs.items() if v != "warm"}
        assert set(now) == set(graphs) and all(now[k] is graphs[k] for k in graphs)   # replayed, not re-captured
        results.append((np.array(losses), [p.detach().clone() for p in model.parameters()]))
    assert np.array_equal(results[0][0], results[1][0])
    assert all(torch.equal(a, b) for a, b in zip(results[0][1], results[1][1]))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("shape", [(1, 1, 1, 64), (1, 5, 3, 64), (4, 1, 4, 128), (3, 7, 1, 128), (6, 2, 3, 128), (2, 3, 4, 64),
                                   (5, 9, "pose", 0)])
def test_seq_losses_kernel_against_float64(K, dtype, shape):
    S, B, C, W = shape
    pose = C == "pose"
    if pose and dtype == torch.bfloat16:
        pytest.skip("pose predictions are fp32")
    E = 51 if pose else C * W * W
    T, z, g = S + 3, 10, 128
    gen = torch.Generator().manual_seed(S * 100 + B)
    dev = "cuda"
    rec = (torch.randn((S + 1) * B * E, generator=gen) * 2).to(dev, dtype)
    x = (torch.randn(T * B * E, generator=gen) if pose else torch.rand(T * B * E, generator=gen)).to(dev)
    tgt = torch.tensor(list(range(1, S + 1)) + [T - 1], dtype=torch.int32, device=dev)
    in_idx = torch.tensor(list(range(S)) + [S - 1], dtype=torch.int32, device=dev)
    mu, lv, mu_p, lv_p = [(0.5 * torch.randn(S * B * z, generator=gen)).to(dev) for _ in range(4)]
    H = torch.randn(T * B * g, generator=gen).tanh().to(dev)
    h_pred = torch.randn((S + 1) * B * g, generator=gen).tanh().to(dev)
    partial = torch.zeros((S + 1) * B * 3, dtype=torch.float64, device=dev)
    counter = torch.zeros(1, dtype=torch.int32, device=dev)
    per = torch.zeros(4 * B, dtype=torch.float64, device=dev)
    out = torch.zeros(4, dtype=torch.float64, device=dev)
    args = (rec, not pose, x, tgt, S, B, E, mu, lv, mu_p, lv_p, z, H, in_idx, h_pred, g, True, 7.0, float(T))
    K.seq_losses(*args, partial, counter, per, out)
    rper, rout = seq_losses_ref(*args)
    np.testing.assert_allclose(per.view(4, B).cpu().numpy(), rper.cpu().numpy(), rtol=1e-4, atol=1e-12)
    np.testing.assert_allclose(out.cpu().numpy(), rout.cpu().numpy(), rtol=1e-4, atol=1e-12)
    assert int(counter.item()) == 0   # rearmed for the next launch
    per2, out2 = torch.zeros_like(per), torch.zeros_like(out)
    K.seq_losses(*args, partial, counter, per2, out2)
    assert torch.equal(per, per2) and torch.equal(out, out2)
