"""Pose generation on the GPU (h36m_mlp backbone): the fused p2pvg_pose_mlp kernel against the composed eager forward, the
eager and the graph-replayed p2p_generate against the reference's own poses (tests/golden/pose_gen_h36m.pt) and the CPU
oracle, and the contracts of P2PModel.p2p_generate_graphed restated for poses.

Tolerances: the pose path is exact fp32 in both P2PVG_PRECISION modes (the eager pose forward runs exact fp32 GEMMs, the
fused kernel exact fp32 FFMA), so both modes share one bound: 3e-4 absolute on generated poses (1e-4 relative to the
input poses' std of 3), 1e-4 relative + 1e-4 absolute for single kernel calls and written-back LSTM states."""
import contextlib
import os
import types

import numpy as np
import pytest
import torch

from oracle import p2p_oracle as O

pytestmark = pytest.mark.gpu
FIX = os.path.join(os.path.dirname(__file__), "golden", "pose_gen_h36m.pt")
POSE_ATOL = 3e-4
MODS = ("frame_predictor", "posterior", "prior")


@contextlib.contextmanager
def precision(p):
    prev = os.environ.get("P2PVG_PRECISION")
    os.environ["P2PVG_PRECISION"] = p
    try:
        yield
    finally:
        if prev is None:
            del os.environ["P2PVG_PRECISION"]
        else:
            os.environ["P2PVG_PRECISION"] = prev


def pose_opt(B, n_past=1, lfs=False, skip_prob=0.5):
    from p2pvg_b200.models import h36m_mlp
    return types.SimpleNamespace(dataset="h36m", backbone_net=h36m_mlp, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0,
                                 weight_align=0.5, skip_prob=skip_prob, n_past=n_past, last_frame_skip=lfs, batch_size=B)


def pose_model(state, opt, cfg):
    from p2pvg_b200.models.p2p_model import P2PModel
    model = P2PModel(opt.batch_size, 1, cfg["g_dim"], cfg["z_dim"], cfg["rnn_size"], 1, 1, 2, opt=opt)
    for m in O.MODULES:
        getattr(model, m).load_state_dict(state[m])
    return model.cuda().eval()


def fixture_model(fix, case):
    o = case["opt"]
    opt = pose_opt(o["batch_size"], o["n_past"], o["last_frame_skip"], o["skip_prob"])
    return pose_model(O.build_state(fix["cfg"], seed=fix["init_seed"]), opt, fix["cfg"])


def perturbed_state(cfg, seed):
    """The reference initialisation (N(0, 0.02) weights) with every parameter moved by N(0, 0.05): poses then depend
    visibly on z and the LSTM state."""
    state = O.build_state(cfg, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    for m in O.MODULES:
        for v in state[m].values():
            if v.is_floating_point():
                v.add_(0.05 * torch.randn(v.shape, generator=g))
    return state


def run(fn, np_seed, draws):
    from p2pvg_b200.infer import eps_stream
    np.random.seed(np_seed)
    with eps_stream(draws) as es:
        out = fn()
        assert len(es.draws) == 0, "fewer gaussian-LSTM calls than executed steps"
    return out


def n_exec_of(np_seed, len_output, len_x, opt, skip_frame, eval_cp_ix=None):
    from p2pvg_b200.gen_engine import plan_slots
    probs = np.random.RandomState(np_seed).uniform(0, 1, len_output - 1)
    return len(plan_slots(len_output, len_x, probs, opt.skip_prob, opt.n_past, skip_frame,
                          len_output - 1 if eval_cp_ix is None else eval_cp_ix))


def draws_for(n_exec, rows, z, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(rows, z, generator=g) for _ in range(2 * n_exec)]


def poses_close(a, b, what, atol=POSE_ATOL):
    e = (a.float().cpu() - b.float().cpu()).abs().max().item()
    assert e <= atol, f"{what}: max {e:.3e}"


def hidden_of(model):
    return {m: [(h.clone(), c.clone()) for h, c in getattr(model, m).hidden] for m in MODS}


def hidden_close(a, b, what=""):
    for m in a:
        for (ha, ca), (hb, cb) in zip(a[m], b[m]):
            assert torch.allclose(ha, hb, rtol=1e-4, atol=1e-4) and torch.allclose(ca, cb, rtol=1e-4, atol=1e-4), (what, m)


# ---- 1. the fused kernel against the composed eager forward ---------------------------------------------------------------
@pytest.mark.parametrize("g", [32, 128, 256])
@pytest.mark.parametrize("rows", [1, 8, 9, 33, 200, 300])
def test_pose_mlp_kernel(rows, g):
    from p2pvg_b200.infer import kernels_for, mlp_decoder_forward, mlp_encoder_forward
    from p2pvg_b200.models import h36m_mlp
    torch.manual_seed(rows * 1000 + g)
    enc = h36m_mlp.encoder(out_dim=g, h_dim=g).cuda()
    dec = h36m_mlp.decoder(in_dim=g, h_dim=g).cuda()
    for mod in (enc, dec):   # non-trivial LayerNorm affine parameters
        for n, p in mod.named_parameters():
            if "norm" in n:
                p.data.add_(0.2 * torch.randn_like(p))
    K = kernels_for("cuda")
    # encoder on frame idx[0] = 2 of a [3][rows][51] segment
    seg = 3 * torch.randn(3, rows, 17, 3, device="cuda")
    idx = torch.tensor([2], dtype=torch.int32, device="cuda")
    h = torch.full((rows, g), float("nan"), device="cuda")
    h1, h2 = torch.full_like(h, float("nan")), torch.full_like(h, float("nan"))
    K.pose_mlp(enc, False, seg, h, rows, src_idx=idx, h1=h1, h2=h2)
    rh, (r1, r2) = mlp_encoder_forward(enc, seg[2])
    for got, ref, what in ((h, rh, "h"), (h1, r1, "h1"), (h2, r2, "h2")):
        assert torch.allclose(got, ref, rtol=1e-4, atol=1e-4), (what, (got - ref).abs().max().item())
    # decoder with skips from a source of nsrc < rows rows (output row r reads skip row r % nsrc)
    nsrc = max(1, rows // 4) if rows > 1 else 1
    vec = torch.tanh(torch.randn(rows, g, device="cuda"))
    s1, s2 = torch.randn(nsrc, g, device="cuda"), torch.randn(nsrc, g, device="cuda")
    out = torch.full((rows, 17, 3), float("nan"), device="cuda")
    K.pose_mlp(dec, True, vec, out, rows, skips=[s1, s2], nsrc=nsrc)
    tile = torch.arange(rows, device="cuda") % nsrc
    ref = mlp_decoder_forward(dec, vec, [s1[tile], s2[tile]])
    assert torch.allclose(out, ref, rtol=1e-4, atol=1e-4), (out - ref).abs().max().item()
    # full-size skip source
    s1, s2 = torch.randn(rows, g, device="cuda"), torch.randn(rows, g, device="cuda")
    K.pose_mlp(dec, True, vec, out, rows, skips=[s1, s2], nsrc=rows)
    ref = mlp_decoder_forward(dec, vec, [s1, s2])
    assert torch.allclose(out, ref, rtol=1e-4, atol=1e-4), (out - ref).abs().max().item()


def test_pose_mlp_rejects_bad_arguments():
    from p2pvg_b200._lib import KernelError
    from p2pvg_b200.infer import kernels_for
    from p2pvg_b200.models import h36m_mlp
    dec = h36m_mlp.decoder(in_dim=128, h_dim=128).cuda()
    K = kernels_for("cuda")
    vec, out = torch.zeros(4, 128, device="cuda"), torch.zeros(4, 17, 3, device="cuda")
    with pytest.raises(KernelError, match="skips"):
        K.pose_mlp(dec, True, vec, out, 4, skips=None, nsrc=0)
    big = h36m_mlp.decoder(in_dim=1024, h_dim=1024).cuda()   # 256 KB of shared memory per CTA
    with pytest.raises(KernelError, match="shared memory"):
        K.pose_mlp(big, True, torch.zeros(4, 1024, device="cuda"), out, 4, skips=[torch.zeros(4, 1024, device="cuda")] * 2, nsrc=4)


# ---- 2 / 3. eager and graphed against the reference's poses -------------------------------------------------------------
def check_against_fixture(generate):
    fix = torch.load(FIX, weights_only=False)
    for case in fix["cases"]:
        model = fixture_model(fix, case)
        x = case["x"].cuda()
        for r in case["runs"]:
            draws = [r["eps"][s, j] for s in range(r["n_exec"]) for j in (0, 1)]
            seq = run(lambda: generate(model, x, case["len_output"], case["eval_cp_ix"], r["model_mode"], r["skip_frame"]),
                      r["np_seed"], draws)
            what = f"{case['case']} {r['model_mode']}/skip_frame={r['skip_frame']}"
            assert len(seq) == case["len_output"], what
            assert [bool((f == 0).all()) for f in seq] == r["zero_frames"], what
            for i, (f, ref) in enumerate(zip(seq, r["poses"])):
                assert tuple(f.shape) == tuple(ref.shape), what
                poses_close(f, ref, f"{what} frame {i}")


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_eager_matches_reference_fixture(prec):
    with precision(prec):
        check_against_fixture(lambda m, x, L, cp, mode, sf: m.p2p_generate((None, x, None), L, cp, model_mode=mode, skip_frame=sf))


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
def test_graphed_matches_reference_fixture(prec):
    with precision(prec):
        check_against_fixture(lambda m, x, L, cp, mode, sf: m.p2p_generate_graphed((None, x, None), L, cp, model_mode=mode,
                                                                                   skip_frame=sf))


# ---- 4. graphed against the CPU oracle at rnn_size 512 ------------------------------------------------------------------
@pytest.mark.parametrize("lfs", [False, True])
@pytest.mark.parametrize("n_past", [1, 2])
def test_graphed_matches_oracle(n_past, lfs):
    from p2pvg_b200.gen_engine import plan_slots
    T, B = 5, 3
    cfg = dict(g_dim=128, z_dim=10, rnn_size=512, backbone="mlp", predictor_rnn_layers=2, posterior_rnn_layers=1, prior_rnn_layers=1)
    state = perturbed_state(cfg, seed=20 + n_past)
    opt = pose_opt(B, n_past, lfs)
    model = pose_model(O.clone_state(state), opt, cfg)
    oopt = dict(skip_prob=0.5, n_past=n_past, last_frame_skip=lfs)
    x = 3 * torch.randn(T, B, 17, 3, generator=torch.Generator().manual_seed(3))
    for len_output, eval_cp_ix, skip_frame in ((T - 2, T - 2, False), (T, T - 1, True), (T + 3, T + 1, True)):
        for mode in ("full", "posterior", "prior"):
            np_seed = 11 + len_output
            probs = np.random.RandomState(np_seed).uniform(0, 1, len_output - 1)
            S = len(plan_slots(len_output, T, probs, 0.5, n_past, skip_frame, eval_cp_ix))
            draws = draws_for(S, B, 10, seed=len_output)
            got = run(lambda: model.p2p_generate_graphed(x.cuda(), len_output, eval_cp_ix, model_mode=mode, skip_frame=skip_frame),
                      np_seed, draws)
            eps = torch.stack([torch.stack([draws[2 * s], draws[2 * s + 1]]) for s in range(S)]) if S else torch.zeros(0, 2, B, 10)
            ref = O.p2p_generate(state, list(x), len_output, eval_cp_ix, oopt, "mlp", eps, probs, model_mode=mode, skip_frame=skip_frame)
            assert len(got) == len(ref) == len_output
            for i, (a, b) in enumerate(zip(got, ref)):
                poses_close(a, b, f"len_output={len_output} {mode} frame {i}")


# ---- 5. the engine's contracts -----------------------------------------------------------------------------------------
def contract_model(n_past=1, lfs=False, B=3, seed=30):
    cfg = dict(g_dim=128, z_dim=10, rnn_size=512, backbone="mlp", predictor_rnn_layers=2, posterior_rnn_layers=1, prior_rnn_layers=1)
    model = pose_model(perturbed_state(cfg, seed), pose_opt(B, n_past, lfs), cfg)
    x = 3 * torch.randn(6, B, 17, 3, generator=torch.Generator().manual_seed(seed)).cuda()
    return model, x


def test_one_graph_two_skip_patterns_no_aliasing():
    from p2pvg_b200.gen_engine import plan_slots
    with precision("fp32"):
        model, x = contract_model()
        L, T, cp = 9, x.shape[0], 8
        pats = {}
        for sd in range(300):
            probs = np.random.RandomState(sd).uniform(0, 1, L - 1)
            pl = plan_slots(L, T, probs, model.opt.skip_prob, model.opt.n_past, True, cp)
            pats.setdefault(len(pl), {}).setdefault(tuple(p[0] for p in pl), sd)
        S, by_pat = max(((k, v) for k, v in pats.items() if len(v) >= 2), key=lambda kv: len(kv[1]))
        outs = []
        for j, sd in enumerate(list(by_pat.values())[:2]):
            draws = draws_for(S, x.shape[1], 10, seed=40 + j)
            got = run(lambda: model.p2p_generate_graphed(x, L, cp, skip_frame=True), sd, draws)
            ref = run(lambda: model.p2p_generate(x, L, cp, skip_frame=True), sd, draws)
            for i, (a, b) in enumerate(zip(got, ref)):
                poses_close(a, b, f"pattern {j} frame {i}")
            outs.append((got, [f.clone() for f in got]))
        assert len(model._gen_engine._graphs) == 1, "both calls must replay one graph"
        for a, b in zip(*outs[0]):
            assert torch.equal(a, b), "a returned pose aliases graph memory"


def test_training_steps_between_calls():
    with precision("fp32"):
        model, x = contract_model()
        L, cp = 8, 7
        S = n_exec_of(0, L, x.shape[0], model.opt, False)
        draws = draws_for(S, x.shape[1], 10, 2)
        before = [f.clone() for f in run(lambda: model.p2p_generate_graphed(x, L, cp), 0, draws)]
        for step in range(2):
            model.train()
            model((None, x, None))   # TrainEngineMLP: parameters move into the training arena (step 0), then update in place
            torch.cuda.synchronize()
            model.eval()
            n_graphs = len(model._gen_engine._graphs)
            got = [f.clone() for f in run(lambda: model.p2p_generate_graphed(x, L, cp), 0, draws)]
            if step == 1:
                assert len(model._gen_engine._graphs) == n_graphs, "stable parameter addresses: the cached graph is reused"
            hg = hidden_of(model)
            ref = run(lambda: model.p2p_generate(x, L, cp), 0, draws)
            assert max((a - b).abs().max().item() for a, b in zip(got[1:], before[1:])) > 1e-4, "the update was not picked up"
            for i, (a, b) in enumerate(zip(got, ref)):
                poses_close(a, b, f"step {step} frame {i}")
            hidden_close(hg, hidden_of(model), f"step {step}")
            before = got


@pytest.mark.parametrize("n_past,lfs", [(1, False), (2, True)])
def test_numpy_stream_and_hidden_state(n_past, lfs):
    with precision("fp32"):
        model, x = contract_model(n_past, lfs)
        L, cp, B = 9, 8, x.shape[1]
        S = n_exec_of(7, L, x.shape[0], model.opt, True)
        draws = draws_for(S, B, 10, 3)
        run(lambda: model.p2p_generate_graphed(x, L, cp, skip_frame=True), 7, draws)
        after_graphed = np.random.uniform()
        run(lambda: model.p2p_generate(x, L, cp, skip_frame=True), 7, draws)
        assert np.random.uniform() == after_graphed
        g = torch.Generator().manual_seed(4)
        start = {m: [(torch.randn(B, getattr(model, m).hidden_size, generator=g).cuda(),
                      torch.randn(B, getattr(model, m).hidden_size, generator=g).cuda()) for _ in range(getattr(model, m).n_layers)]
                 for m in MODS}
        res = {}
        for name, fn in (("graphed", model.p2p_generate_graphed), ("graphed again", model.p2p_generate_graphed),
                         ("eager", model.p2p_generate)):
            for m, hc in start.items():
                getattr(model, m).hidden = [(h.clone(), c.clone()) for h, c in hc]
            seq = run(lambda: fn(x, L, cp, skip_frame=True, init_hidden=False), 7, draws)
            res[name] = ([f.clone() for f in seq], hidden_of(model))
        for a, b, e in zip(res["graphed"][0], res["graphed again"][0], res["eager"][0]):
            assert torch.equal(a, b)
            poses_close(a, e, "init_hidden=False")
        hidden_close(res["graphed"][1], res["eager"][1], "written-back .hidden")


def test_nsample_equals_looped_calls():
    with precision("fp32"):
        model, x = contract_model()
        L, cp, B, ns = 9, 8, x.shape[1], 4
        S = n_exec_of(5, L, x.shape[0], model.opt, True)
        d = torch.randn(ns, S, 2, B, 10, generator=torch.Generator().manual_seed(9))
        looped = [run(lambda: model.p2p_generate_graphed(list(x), L, cp, skip_frame=True), 5,
                      [d[s, i, j] for i in range(S) for j in (0, 1)]) for s in range(ns)]
        batched = run(lambda: model.p2p_generate_graphed(x, L, cp, skip_frame=True, nsample=ns), 5,
                      [d[:, i, j].reshape(ns * B, 10) for i in range(S) for j in (0, 1)])
        eager = run(lambda: model.p2p_generate_samples(x, ns, L, cp, skip_frame=True), 5,
                    [d[:, i, j].reshape(ns * B, 10) for i in range(S) for j in (0, 1)])
        assert len(batched) == ns and all(len(b) == L for b in batched)
        for s in range(ns):
            for a, b, e in zip(batched[s], looped[s], eager[s]):
                assert a.shape == b.shape == (B, 17, 3)
                assert torch.allclose(a, b, rtol=1e-4, atol=1e-5)
                poses_close(a, e, f"sample {s}")


# ---- 6. launch budget ---------------------------------------------------------------------------------------------------
def test_launch_budget_per_step():
    """K.launches over the first call of a signature counts the warm-up run and the captured body (two bodies)."""
    from p2pvg_b200.infer import kernels_for
    with precision("fp32"):
        model, x = contract_model()
        K = kernels_for("cuda")
        rest = []
        for L in (4, 7, 12):
            S = L - 1   # skip_frame=False, n_past=1: every step executes and decodes
            n0 = K.launches
            run(lambda: model.p2p_generate_graphed(x, L, L - 1), 0, draws_for(S, x.shape[1], 10, L))
            body = (K.launches - n0) // 2
            assert (K.launches - n0) % 2 == 0
            assert body <= 4 * S + 4, (L, body)
            rest.append(body - 4 * S)
            n1 = K.launches
            run(lambda: model.p2p_generate_graphed(x, L, L - 1), 0, draws_for(S, x.shape[1], 10, L))
            assert K.launches == n1, "a replay launches nothing from the host"
        assert len(set(rest)) == 1, f"the per-call constant depends on the number of steps: {rest}"
