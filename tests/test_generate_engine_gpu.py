"""P2PModel.p2p_generate_graphed (p2pvg_b200/gen_engine.py): one CUDA-graph replay per call against the reference's frames
(tests/golden/gen_*.pt), the CPU oracle (dcgan_128, 3 channels), and the eager p2p_generate fed the same draws; plus the
eval-BatchNorm epilogue of p2pvg_conv_gemm against GEMM + bn_eval_coeffs + bn_act.  Tolerances as test_generate_gpu.py:
fp32 2e-4 max / 2e-5 mean, bf16 4e-2 max / 6e-3 mean on frames in [0, 1]."""
import contextlib
import os
import types

import numpy as np
import pytest
import torch

from oracle import p2p_oracle as O
from tests.test_generate_gpu import GEN, build_model

pytestmark = pytest.mark.gpu
TOL = {"fp32": (2e-4, 2e-5), "bf16": (4e-2, 6e-3)}


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


def close(a, b, prec, what=""):
    tmax, tmean = TOL[prec]
    e = (a.float().cpu() - b.float().cpu()).abs()
    assert e.max().item() <= tmax and e.mean().item() <= tmean, f"{what}: max {e.max().item():.3e} mean {e.mean().item():.3e}"


def draws_for(n_exec, rows, z, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(rows, z, generator=g) for _ in range(2 * n_exec)]


def run(fn, np_seed, draws):
    from p2pvg_b200.infer import eps_stream
    np.random.seed(np_seed)
    with eps_stream(draws) as es:
        out = fn()
        assert len(es.draws) == 0, "fewer gaussian-LSTM calls than executed steps"
    return out


def n_exec_of(np_seed, len_output, len_x, opt, skip_frame):
    from p2pvg_b200.gen_engine import plan_slots
    probs = np.random.RandomState(np_seed).uniform(0, 1, len_output - 1)
    return len(plan_slots(len_output, len_x, probs, opt.skip_prob, opt.n_past, skip_frame, len_output - 1))


# ---- 1. the reference's own frames ----------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("path", GEN, ids=lambda p: os.path.basename(p)[4:-3])
def test_graphed_matches_reference_fixtures(path, prec):
    fix = torch.load(path, weights_only=False)
    tmax, tmean = TOL[prec]
    with precision(prec):
        model = build_model(fix)
        x = fix["x"].cuda()
        for r in fix["runs"]:
            draws = [r["eps"][s, j] for s in range(r["n_exec"]) for j in (0, 1)]
            seq = run(lambda: model.p2p_generate_graphed(x, fix["len_output"], fix["eval_cp_ix"], model_mode=r["model_mode"],
                                                         skip_frame=r["skip_frame"]), r["np_seed"], draws)
            what = f"{prec} {r['model_mode']}/skip_frame={r['skip_frame']}"
            assert len(seq) == fix["len_output"]
            assert [bool((f == 0).all()) for f in seq] == r["zero_frames"], what
            for i, (f, d) in enumerate(zip(seq, r["digests"])):
                v = f.detach().double().reshape(-1).cpu()
                assert (v[d["idx"]] - d["samples"]).abs().max().item() <= tmax, f"{what} frame {i}"
            for f, ref in ((seq[-1], r["last"]), (seq[len(seq) // 2], r["mid"])):
                close(f, ref, prec, what)


# ---- 2. dcgan_128, three channels, against the CPU oracle -------------------------------------------------------------
def model128(n_past, lfs, seed=5):
    from p2pvg_b200.models import dcgan_128
    from p2pvg_b200.models.p2p_model import P2PModel
    cfg = dict(g_dim=128, z_dim=10, rnn_size=256, channels=3, image_width=128, predictor_rnn_layers=2,
               posterior_rnn_layers=1, prior_rnn_layers=1)
    opt = types.SimpleNamespace(dataset="mnist", backbone_net=dcgan_128, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0,
                                weight_align=0.5, skip_prob=0.5, n_past=n_past, last_frame_skip=lfs, batch_size=2)
    model = P2PModel(2, 3, 128, 10, 256, 1, 1, 2, opt=opt)
    state = O.build_state(cfg, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    for m in ("encoder", "decoder"):   # non-trivial running statistics
        for k, v in state[m].items():
            if k.endswith("running_mean"):
                v.copy_(0.1 * torch.randn(v.shape, generator=g))
            elif k.endswith("running_var"):
                v.copy_(0.5 + torch.rand(v.shape, generator=g))
    for m in O.MODULES:
        getattr(model, m).load_state_dict(state[m])
    return model.cuda().eval(), state, dict(skip_prob=0.5, n_past=n_past, last_frame_skip=lfs)


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("lfs", [False, True])
@pytest.mark.parametrize("n_past", [1, 2])
def test_dcgan128_rgb_matches_oracle(n_past, lfs, prec):
    T, B = 5, 2
    x = torch.rand(T, B, 3, 128, 128, generator=torch.Generator().manual_seed(3))
    with precision(prec):
        model, state, oopt = model128(n_past, lfs)
        for len_output, eval_cp_ix, skip_frame in ((T - 2, T - 2, False), (T, T - 2, True), (T + 2, T + 1, True)):
            np_seed = 11 + len_output
            probs = np.random.RandomState(np_seed).uniform(0, 1, len_output - 1)
            from p2pvg_b200.gen_engine import plan_slots
            S = len(plan_slots(len_output, T, probs, 0.5, n_past, skip_frame, eval_cp_ix))
            draws = draws_for(S, B, 10, seed=len_output)
            got = run(lambda: model.p2p_generate_graphed(x.cuda(), len_output, eval_cp_ix, skip_frame=skip_frame), np_seed, draws)
            eps = torch.stack([torch.stack([draws[2 * s], draws[2 * s + 1]]) for s in range(S)]) if S else torch.zeros(0, 2, B, 10)
            ref = O.p2p_generate(state, list(x), len_output, eval_cp_ix, oopt, 128, eps, probs, skip_frame=skip_frame)
            assert len(got) == len(ref) == len_output
            for i, (a, b) in enumerate(zip(got, ref)):
                close(a, b, prec, f"len_output={len_output} frame {i}")


# ---- 3. one graph, many calls ----------------------------------------------------------------------------------------
def test_one_graph_many_calls_tables_not_baked():
    fix = torch.load(GEN[0], weights_only=False)
    with precision("fp32"):
        model = build_model(fix)
        x = fix["x"].cuda()
        L, T = fix["len_output"], x.shape[0]
        opt = model.opt
        # two NumPy seeds with the same number of executed steps but different skip patterns
        pats = {}
        for sd in range(200):
            probs = np.random.RandomState(sd).uniform(0, 1, L - 1)
            from p2pvg_b200.gen_engine import plan_slots
            pl = plan_slots(L, T, probs, opt.skip_prob, opt.n_past, True, fix["eval_cp_ix"])
            pats.setdefault(len(pl), {}).setdefault(tuple(p[0] for p in pl), sd)
        S, by_pat = max(((k, v) for k, v in pats.items() if len(v) >= 2), key=lambda kv: len(kv[1]))
        seeds = list(by_pat.values())[:2]
        outs = []
        for j, sd in enumerate(seeds):
            draws = draws_for(S, x.shape[1], 10, seed=40 + j)
            got = run(lambda: model.p2p_generate_graphed(x, L, fix["eval_cp_ix"], skip_frame=True), sd, draws)
            ref = run(lambda: model.p2p_generate(x, L, fix["eval_cp_ix"], skip_frame=True), sd, draws)
            for a, b in zip(got, ref):
                close(a, b, "fp32")
            outs.append((got, [f.clone() for f in got]))
        assert len(model._gen_engine._graphs) == 1, "both calls must replay one graph"
        first, snapshot = outs[0]
        for a, b in zip(first, snapshot):
            assert torch.equal(a, b), "a returned frame aliases graph memory"


# ---- 4. a training step between two calls ------------------------------------------------------------------------------
def test_fresh_weights_after_training_step():
    fix = torch.load(GEN[0], weights_only=False)
    with precision("fp32"):
        model = build_model(fix)
        x = fix["x"].cuda()
        L, cp = fix["len_output"], fix["eval_cp_ix"]
        S = n_exec_of(0, L, x.shape[0], model.opt, False)
        draws = draws_for(S, x.shape[1], 10, 2)
        before = run(lambda: model.p2p_generate_graphed(x, L, cp), 0, draws)
        model.train()
        model(x)                       # re-points parameters into the training arena and updates them + running statistics
        torch.cuda.synchronize()
        model.eval()
        got = run(lambda: model.p2p_generate_graphed(x, L, cp), 0, draws)
        ref = run(lambda: model.p2p_generate(x, L, cp), 0, draws)
        assert max((a - b).abs().max().item() for a, b in zip(got[1:], before[1:])) > 1e-3, "the update was not picked up"
        # the graphed path encodes the ground truth time-batched (other GEMM row counts, so other fp32 summation orders
        # than the per-frame eager calls); after the update the autoregressive steps amplify that to a few 1e-5 on average
        for a, b in zip(got, ref):
            e = (a - b).abs()
            assert e.max().item() <= 2e-4 and e.mean().item() <= 5e-5, (e.max().item(), e.mean().item())


# ---- 5. NumPy stream and hidden state ----------------------------------------------------------------------------------
def test_numpy_stream_and_hidden_state():
    fix = torch.load(GEN[1], weights_only=False)
    with precision("fp32"):
        model = build_model(fix)
        x = fix["x"].cuda()
        L, cp, B = fix["len_output"], fix["eval_cp_ix"], x.shape[1]
        S = n_exec_of(7, L, x.shape[0], model.opt, True)
        draws = draws_for(S, B, 10, 3)
        run(lambda: model.p2p_generate_graphed(x, L, cp, skip_frame=True), 7, draws)
        after_graphed = np.random.uniform()
        run(lambda: model.p2p_generate(x, L, cp, skip_frame=True), 7, draws)
        assert np.random.uniform() == after_graphed
        # init_hidden=False: start from a non-zero .hidden, leave the final state in .hidden
        g = torch.Generator().manual_seed(4)
        start = {m: [(torch.randn(B, getattr(model, m).hidden_size, generator=g).cuda(),
                      torch.randn(B, getattr(model, m).hidden_size, generator=g).cuda()) for _ in range(getattr(model, m).n_layers)]
                 for m in ("frame_predictor", "posterior", "prior")}
        res = {}
        for name, fn in (("graphed", model.p2p_generate_graphed), ("eager", model.p2p_generate)):
            for m, hc in start.items():
                getattr(model, m).hidden = [(h.clone(), c.clone()) for h, c in hc]
            seq = run(lambda: fn(x, L, cp, skip_frame=True, init_hidden=False), 7, draws)
            res[name] = (seq, {m: [(h.clone(), c.clone()) for h, c in getattr(model, m).hidden] for m in start})
        for a, b in zip(res["graphed"][0], res["eager"][0]):
            close(a, b, "fp32")
        for m in start:
            for (h1, c1), (h2, c2) in zip(res["graphed"][1][m], res["eager"][1][m]):
                assert torch.allclose(h1, h2, rtol=1e-4, atol=1e-5) and torch.allclose(c1, c2, rtol=1e-4, atol=1e-5), m


# ---- 6. batched samples ------------------------------------------------------------------------------------------------
def test_nsample_equals_looped_graphed_calls():
    fix = torch.load(GEN[0], weights_only=False)
    with precision("fp32"):
        model = build_model(fix)
        x = fix["x"].cuda()
        L, cp, B, ns = fix["len_output"], fix["eval_cp_ix"], x.shape[1], 3
        S = n_exec_of(5, L, x.shape[0], model.opt, True)
        g = torch.Generator().manual_seed(9)
        d = torch.randn(ns, S, 2, B, 10, generator=g)
        looped = [run(lambda: model.p2p_generate_graphed(x, L, cp, skip_frame=True), 5, [d[s, i, j] for i in range(S) for j in (0, 1)])
                  for s in range(ns)]
        batched = run(lambda: model.p2p_generate_graphed(x, L, cp, skip_frame=True, nsample=ns), 5,
                      [d[:, i, j].reshape(ns * B, 10) for i in range(S) for j in (0, 1)])
        eager = run(lambda: model.p2p_generate_samples(x, ns, L, cp, skip_frame=True), 5,
                    [d[:, i, j].reshape(ns * B, 10) for i in range(S) for j in (0, 1)])
        assert len(batched) == ns and all(len(b) == L for b in batched)
        for s in range(ns):
            for a, b, e in zip(batched[s], looped[s], eager[s]):
                assert a.shape == b.shape and torch.allclose(a.float(), b.float(), rtol=1e-4, atol=2e-5)
                close(a, e, "fp32")


# ---- 7. the eval-BatchNorm epilogue ------------------------------------------------------------------------------------
# (kind, Ck, Cn, small-map size) at the dcgan_64 / dcgan_128 layer shapes
EPI_SHAPES = [(0, 64, 128, 16), (0, 128, 256, 8), (0, 256, 512, 4), (0, 512, 512, 2),
              (2, 512, 256, 4), (2, 256, 128, 8), (2, 128, 64, 16), (2, 512, 512, 2)]


@pytest.mark.parametrize("B", [1, 16, 100])
@pytest.mark.parametrize("kind,Ck,Cn,H", EPI_SHAPES)
def test_conv_gemm_eval_epilogue(kind, Ck, Cn, H, B):
    from p2pvg_b200._lib import ACT_LRELU, ACT_TANH, kernels_for
    K = kernels_for("cuda")
    g = torch.Generator(device="cuda").manual_seed(Ck + Cn + H + B)
    Hin = 2 * H if kind == 0 else H
    Hout = H if kind == 0 else 2 * H
    a = torch.randn(B * Hin * Hin * Ck, device="cuda", generator=g).bfloat16()
    w = (0.05 * torch.randn(16 * Ck * Cn, device="cuda", generator=g)).bfloat16()
    bias = torch.randn(Cn, device="cuda", generator=g)
    gamma, beta = 1 + 0.1 * torch.randn(Cn, device="cuda", generator=g), 0.1 * torch.randn(Cn, device="cuda", generator=g)
    rmean, rvar = 0.1 * torch.randn(Cn, device="cuda", generator=g), 0.5 + torch.rand(Cn, device="cuda", generator=g)
    sc, sh = torch.empty(Cn, device="cuda"), torch.empty(Cn, device="cuda")
    K.bn_eval_coeffs(gamma, beta, rmean, rvar, Cn, sc, sh)
    M = B * Hout * Hout
    for act in (ACT_LRELU, ACT_TANH):
        for add in (False, True):
            addend = torch.randn(M * Cn, device="cuda", generator=g).bfloat16() if add else None
            kw = dict(bias=bias, addend=addend, grp_src=torch.zeros(1, dtype=torch.int32, device="cuda") if add else None,
                      imgs_per_group=B if add else 0)
            raw = torch.empty(M * Cn, device="cuda")
            K.conv_gemm(kind, a, w, raw, B, H, H, Ck, Cn, **kw)
            ref = torch.empty_like(raw)
            K.bn_act(raw, ref, sc, sh, 1, M, Cn, act)
            got = torch.empty_like(raw)
            K.conv_gemm(kind, a, w, got, B, H, H, Ck, Cn, eval_scale=sc, eval_shift=sh, act=act, **kw)
            torch.cuda.synchronize()
            assert torch.allclose(got, ref, rtol=1e-5, atol=1e-5), (act, add, (got - ref).abs().max().item())
            got16 = torch.empty(M * Cn, device="cuda", dtype=torch.bfloat16)
            K.conv_gemm(kind, a, w, got16, B, H, H, Ck, Cn, eval_scale=sc, eval_shift=sh, act=act, **kw)
            assert torch.allclose(got16.float(), ref, rtol=1e-2, atol=1e-2)


def test_conv_gemm_eval_epilogue_rejects_statistics():
    from p2pvg_b200._lib import ACT_LRELU, KernelError, kernels_for
    K = kernels_for("cuda")
    a = torch.zeros(2 * 32 * 32 * 64, device="cuda", dtype=torch.bfloat16)
    w = torch.zeros(16 * 64 * 128, device="cuda", dtype=torch.bfloat16)
    c = torch.empty(2 * 16 * 16 * 128, device="cuda", dtype=torch.bfloat16)
    sc = torch.ones(128, device="cuda")
    sp = torch.zeros(4 * 128 * 2, device="cuda")
    with pytest.raises(KernelError, match="eval"):
        K.conv_gemm(0, a, w, c, 2, 16, 16, 64, 128, stat_partial=sp, eval_scale=sc, eval_shift=sc, act=ACT_LRELU)


# ---- state on a fresh signature -------------------------------------------------------------------------------------
@pytest.mark.parametrize("init_hidden", [True, False])
def test_first_call_of_a_signature_starts_from_the_given_state(init_hidden):
    """The first call of a signature (warm-up + capture + replay) must start from zeros or the caller's .hidden exactly like
    every later call: frames and written-back .hidden of call 1 (fresh graph) and call 2 (cached graph) are bit-equal, and
    equal the eager path's."""
    fix = torch.load(GEN[1], weights_only=False)
    mods = ("frame_predictor", "posterior", "prior")
    with precision("fp32"):
        model = build_model(fix)
        x = fix["x"].cuda()
        L, cp, B = fix["len_output"], fix["eval_cp_ix"], x.shape[1]
        S = n_exec_of(7, L, x.shape[0], model.opt, True)
        draws = draws_for(S, B, 10, 3)
        g = torch.Generator().manual_seed(4)
        start = {m: [(torch.randn(B, getattr(model, m).hidden_size, generator=g).cuda(),
                      torch.randn(B, getattr(model, m).hidden_size, generator=g).cuda()) for _ in range(getattr(model, m).n_layers)]
                 for m in mods}
        res = []
        for fn in (model.p2p_generate_graphed, model.p2p_generate_graphed, model.p2p_generate):
            for m, hc in start.items():
                getattr(model, m).hidden = [(h.clone(), c.clone()) for h, c in hc]
            seq = run(lambda: fn(x, L, cp, skip_frame=True, init_hidden=init_hidden), 7, draws)
            res.append(([f.clone() for f in seq], {m: [(h.clone(), c.clone()) for h, c in getattr(model, m).hidden] for m in mods}))
        assert len(model._gen_engine._graphs) == 1
        (f1, h1), (f2, h2), (fe, he) = res
        for a, b, e in zip(f1, f2, fe):
            assert torch.equal(a, b)
            close(a, e, "fp32")
        for m in mods:
            for (ha, ca), (hb, cb), (hx, cx) in zip(h1[m], h2[m], he[m]):
                assert torch.equal(ha, hb) and torch.equal(ca, cb), m
                assert torch.allclose(ha, hx, rtol=1e-4, atol=1e-5) and torch.allclose(ca, cx, rtol=1e-4, atol=1e-5), m


def hidden_close(model_hidden_a, model_hidden_b, what=""):
    for m in model_hidden_a:
        for (ha, ca), (hb, cb) in zip(model_hidden_a[m], model_hidden_b[m]):
            assert torch.allclose(ha, hb, rtol=1e-4, atol=2e-5) and torch.allclose(ca, cb, rtol=1e-4, atol=2e-5), (what, m)


def hidden_of(model):
    return {m: [(h.clone(), c.clone()) for h, c in getattr(model, m).hidden] for m in ("frame_predictor", "posterior", "prior")}


@pytest.mark.parametrize("mode", ["full", "posterior", "prior"])
def test_latent_path_matches_eager(mode):
    """The frames of randomly initialised weights hardly depend on z; the LSTM states do.  After a call with skipped
    frames and ground truth running out (posterior falls back to h_cpaw), the written-back states of all three modules
    equal the eager path's, per model_mode (which z feeds the predictor)."""
    fix = torch.load(GEN[1], weights_only=False)
    with precision("fp32"):
        model = build_model(fix)
        x = fix["x"].cuda()
        L = x.shape[0] + 3
        S = n_exec_of(2, L, x.shape[0], model.opt, True)
        draws = draws_for(S, x.shape[1], 10, 8)
        run(lambda: model.p2p_generate_graphed(x, L, L - 2, model_mode=mode, skip_frame=True), 2, draws)
        hg = hidden_of(model)
        run(lambda: model.p2p_generate(x, L, L - 2, model_mode=mode, skip_frame=True), 2, draws)
        hidden_close(hg, hidden_of(model), mode)


def test_cached_graph_picks_up_a_second_training_step():
    """With the parameters already in the training arena (stable addresses), a training step between two calls reuses the
    cached graph, whose in-graph weight re-pack and BatchNorm coefficients must see the updated values."""
    fix = torch.load(GEN[0], weights_only=False)
    with precision("bf16"):
        model = build_model(fix)
        x = fix["x"].cuda()
        L, cp = fix["len_output"], fix["eval_cp_ix"]
        model.train()
        model(x)
        model.eval()
        S = n_exec_of(0, L, x.shape[0], model.opt, False)
        draws = draws_for(S, x.shape[1], 10, 2)
        before = run(lambda: model.p2p_generate_graphed(x, L, cp), 0, draws)
        before = [f.clone() for f in before]
        n_graphs = len(model._gen_engine._graphs)
        model.train()
        model(x)
        torch.cuda.synchronize()
        model.eval()
        got = run(lambda: model.p2p_generate_graphed(x, L, cp), 0, draws)
        hg = hidden_of(model)
        assert len(model._gen_engine._graphs) == n_graphs, "the second call must reuse the cached graph"
        ref = run(lambda: model.p2p_generate(x, L, cp), 0, draws)
        assert max((a - b).abs().max().item() for a, b in zip(got[1:], before[1:])) > 1e-3, "the update was not picked up"
        for a, b in zip(got, ref):
            close(a, b, "bf16")
        for m, hc in hg.items():
            for (ha, ca), (hb, cb) in zip(hc, hidden_of(model)[m]):
                assert (ha - hb).abs().max().item() < 2e-2 and (ca - cb).abs().max().item() < 2e-2, m


# ---- the fused LSTM step kernel ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 16, 33, 200])
@pytest.mark.parametrize("L", [1, 2, 3])
@pytest.mark.parametrize("R", [64, 128, 256, 512])
def test_lstm_step_kernel(R, L, B):
    """p2pvg_lstm_step (two gaussian modules in one launch, then one Linear+tanh module) against the composed exact-fp32
    sequence embed GEMM -> (GEMM W_ih, GEMM W_hh + addend, lstm_pointwise_fwd) x L -> head GEMMs + act / reparam_kl_fwd.
    The state is updated in place."""
    from p2pvg_b200._lib import ACT_TANH, LSTM_HEAD_GAUSSIAN, LSTM_HEAD_LINEAR_TANH
    from p2pvg_b200.infer import kernels_for
    K = kernels_for("cuda")
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(R * 100 + L * 10 + B)
    ga, gb, zd, go = 128, 10, 10, 128
    T = 3
    A = torch.randn(T * B, ga, device=dev, generator=g)
    Bm = torch.randn(2 * B, gb, device=dev, generator=g)
    idx = torch.tensor([2, 1], dtype=torch.int32, device=dev)
    sc = torch.tensor([0.4, 0.2], device=dev)
    in_dim = ga + gb + 2
    X = torch.cat([A[2 * B:3 * B], Bm[B:2 * B], sc[0].expand(B, 1), sc[1].expand(B, 1)], 1).contiguous()

    def rnd(*shape, s=0.1):
        return s * torch.randn(*shape, device=dev, generator=g)

    def module(head):
        mod = dict(w_e=rnd(R, in_dim), b_e=rnd(R), layers=[(rnd(4 * R, R), rnd(4 * R), rnd(4 * R, R), rnd(4 * R)) for _ in range(L)],
                   h=[rnd(B, R, s=0.5) for _ in range(L)], c=[rnd(B, R, s=0.5) for _ in range(L)], head=head)
        n = zd if head == LSTM_HEAD_GAUSSIAN else go
        mod.update(w_o=rnd(n, R), b_o=rnd(n), w_o2=rnd(n, R), b_o2=rnd(n), eps=torch.randn(B, n, device=dev, generator=g), n=n)
        return mod

    def reference(mod):
        E = torch.empty(B, R, device=dev)
        K.gemm(X, mod["w_e"], E, B, R, in_dim, bias=mod["b_e"])
        inp, hs, cs = E, [], []
        for l, (wi, bi, wh, bh) in enumerate(mod["layers"]):
            pre, gates = torch.empty(B, 4 * R, device=dev), torch.empty(B, 4 * R, device=dev)
            K.gemm(inp, wi, pre, B, 4 * R, R, bias=bi)
            K.gemm(mod["h"][l], wh, gates, B, 4 * R, R, bias=bh, addend=pre)
            c, h = torch.empty(B, R, device=dev), torch.empty(B, R, device=dev)
            K.lstm_pointwise_fwd(gates, mod["c"][l], c, h, B, R)
            hs.append(h)
            cs.append(c)
            inp = h
        n = mod["n"]
        out = torch.empty(B, n, device=dev)
        K.gemm(inp, mod["w_o"], out, B, n, R, bias=mod["b_o"])
        if mod["head"] == LSTM_HEAD_LINEAR_TANH:
            K.act_fwd(out, out.numel(), ACT_TANH)
            return out, hs, cs
        lv = torch.empty(B, n, device=dev)
        K.gemm(inp, mod["w_o2"], lv, B, n, R, bias=mod["b_o2"])
        z, zz = torch.empty_like(out), torch.empty_like(out)
        K.reparam_kl_fwd(out, lv, out, lv, mod["eps"], mod["eps"], z, zz, B * n, torch.zeros(4, device=dev))
        return z, hs, cs

    def operands(mod):
        hs, cs = [h.clone() for h in mod["h"]], [c.clone() for c in mod["c"]]
        w = torch.tensor([t.data_ptr() for lw in mod["layers"] for t in lw], dtype=torch.int64, device=dev)
        st = torch.tensor([t.data_ptr() for l in range(L) for t in (hs[l], cs[l], hs[l], cs[l])], dtype=torch.int64, device=dev)
        out = torch.full((B, mod["n"]), float("nan"), device=dev)
        d = dict(seg_a=A, idx_a=idx[:1], ga=ga, seg_b=Bm, idx_b=idx[1:], gb=gb, tuc=sc[:1], dt=sc[1:], w_embed=mod["w_e"],
                 b_embed=mod["b_e"], layers=L, layer_w=w, state=st, head=mod["head"], out_dim=mod["n"], w_out=mod["w_o"],
                 b_out=mod["b_o"], w_out2=mod["w_o2"], b_out2=mod["b_o2"], eps=mod["eps"], out=out)
        return d, (out, hs, cs, w, st)

    mods = [module(LSTM_HEAD_GAUSSIAN), module(LSTM_HEAD_GAUSSIAN), module(LSTM_HEAD_LINEAR_TANH)]
    ops = [operands(m) for m in mods]
    K.lstm_step([ops[0][0], ops[1][0]], B, R)
    K.lstm_step([ops[2][0]], B, R)
    torch.cuda.synchronize()
    for mod, (_, (out, hs, cs, _, _)) in zip(mods, ops):
        ref, rh, rc = reference(mod)
        torch.cuda.synchronize()
        assert torch.allclose(out, ref, rtol=1e-5, atol=1e-5), (out - ref).abs().max().item()
        for l in range(L):
            assert torch.allclose(hs[l], rh[l], rtol=1e-5, atol=1e-5) and torch.allclose(cs[l], rc[l], rtol=1e-5, atol=1e-5), l
