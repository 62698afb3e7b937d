"""P2PModel.p2p_generate_multi_cp and p2p_evaluate(cp_ixs=...) (p2pvg_b200/gen_engine.py): the chain of segments as ONE
CUDA-graph replay against the reference's own hand-chained p2p_generate calls (tests/golden/multi_cp_gen.pt) and against
the looped p2p_generate_graphed calls it stands for, for every backbone in both P2PVG_PRECISION modes.

Tolerances: against the reference as the other generation tests (fp32 2e-4 worst / 2e-5 mean, bf16 4e-2 / 6e-3 on frames
in [0, 1]; 3e-4 absolute on poses in both modes); against the looped calls as the nsample test of
test_generate_engine_gpu.py (frames rtol 1e-4 + atol 2e-5, written-back LSTM state rtol 1e-4 + atol 1e-5)."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import p2p_oracle as O
from p2pvg_b200 import metrics
from tests.test_generate_engine_gpu import TOL, close, precision, run
from tests.test_metrics_gpu import make_model
from tests.test_pose_generate_gpu import POSE_ATOL, pose_model, pose_opt

pytestmark = pytest.mark.gpu
FIX = os.path.join(os.path.dirname(__file__), "golden", "multi_cp_gen.pt")
MODS = ("frame_predictor", "posterior", "prior")


def load():
    return torch.load(FIX, weights_only=False)


def case_frames(c):
    g = torch.Generator().manual_seed(c["x_seed"])
    if c["backbone"] == "mlp":
        return 3 * torch.randn(*c["x_shape"], generator=g)
    return torch.rand(*c["x_shape"], generator=g)


def case_model(c):
    if c["backbone"] == "mlp":
        o = c["opt"]
        return pose_model(O.build_state(c["cfg"], seed=c["init_seed"]), pose_opt(o["batch_size"], o["n_past"],
                                                                              o["last_frame_skip"], o["skip_prob"]), c["cfg"])
    if c["backbone"] == "vgg":
        from tests.test_vgg_generate_gpu import build_model
    else:
        from tests.test_generate_gpu import build_model
    return build_model(c)


def hidden_of(model):
    return {m: [(h.clone(), c.clone()) for h, c in getattr(model, m).hidden] for m in MODS}


def n_exec_chain(np_seed, cps, lens, opt, skip_frame):
    from p2pvg_b200.gen_engine import plan_slots
    rs, n = np.random.RandomState(np_seed), 0
    for k, (a, b) in enumerate(zip(cps, cps[1:])):
        L = lens[k] if lens else b - a + 1
        n += len(plan_slots(L, b - a + 1, rs.uniform(0, 1, L - 1), opt.skip_prob, opt.n_past, skip_frame, L - 1))
    return n


def looped(model, x, cps, lens, mode="full", skip_frame=False, ns=1):
    """The calls p2p_generate_multi_cp stands for."""
    out = []
    for k, (a, b) in enumerate(zip(cps, cps[1:])):
        L = lens[k] if lens else b - a + 1
        out.append(model.p2p_generate_graphed(x[a:b + 1], L, L - 1, model_mode=mode, skip_frame=skip_frame, init_hidden=k == 0,
                                              nsample=ns))
    return out


def flat(res, ns):
    """[(segment, sample, frame index, tensor)] of a chain result."""
    return [(k, s, i, f) for k, seg in enumerate(res) for s, seq in enumerate([seg] if ns == 1 else seg) for i, f in enumerate(seq)]


def assert_same_as_looped(got, ref, ns, what=""):
    a, b = flat(got, ns), flat(ref, ns)
    assert [t[:3] for t in a] == [t[:3] for t in b], what
    for (k, s, i, fa), (_, _, _, fb) in zip(a, b):
        assert fa.shape == fb.shape and torch.allclose(fa.float(), fb.float(), rtol=1e-4, atol=2e-5), \
            f"{what} segment {k} sample {s} frame {i}: {(fa.float() - fb.float()).abs().max().item():.3e}"


def assert_hidden_same(ha, hb, what=""):
    for m in MODS:
        for (h1, c1), (h2, c2) in zip(ha[m], hb[m]):
            assert torch.allclose(h1, h2, rtol=1e-4, atol=1e-5) and torch.allclose(c1, c2, rtol=1e-4, atol=1e-5), (what, m)


# ---- 1. the reference's own chained calls ------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("case", range(4))
def test_chain_matches_reference_fixture(case, prec):
    c = load()["cases"][case]
    tmax, _ = TOL[prec]
    with precision(prec):
        model = case_model(c)
        x = case_frames(c).cuda()
        for r in c["runs"]:
            draws = [r["eps"][s, j] for s in range(r["n_exec"]) for j in (0, 1)]
            what = f"{c['case']} {prec} {r['model_mode']}/skip_frame={r['skip_frame']}"
            res = run(lambda: model.p2p_generate_multi_cp(x, c["cp_ixs"], c["len_outputs"], model_mode=r["model_mode"],
                                                          skip_frame=r["skip_frame"]), r["np_seed"], draws)
            assert [len(seq) for seq in res] == c["len_outputs"], what
            assert [[bool((f == 0).all()) for f in seq] for seq in res] == r["zero_frames"], what
            for k, seq in enumerate(res):
                if c["backbone"] == "mlp":
                    for i, (f, ref) in enumerate(zip(seq, r["poses"][k])):
                        e = (f.float().cpu() - ref.float()).abs().max().item()
                        assert e <= POSE_ATOL, f"{what} segment {k} pose {i}: {e:.3e}"
                    continue
                for i, (f, d) in enumerate(zip(seq, r["digests"][k])):
                    v = f.detach().double().reshape(-1).cpu()
                    assert (v[d["idx"]] - d["samples"]).abs().max().item() <= tmax, f"{what} segment {k} frame {i}"
                if "last" in r:
                    close(seq[-1], r["last"][k], prec, f"{what} segment {k} last frame")


# ---- 2. the looped p2p_generate_graphed calls ----------------------------------------------------------------------------
CONFIGS = [("dcgan_64", 1, 1, False), ("dcgan_64", 1, 2, True), ("dcgan_128", 3, 1, False), ("vgg_64", 3, 2, True),
           ("vgg_128", 1, 1, False), ("h36m_mlp", 1, 1, False), ("h36m_mlp", 1, 2, True)]


def config_model(backbone, C, n_past, lfs, B=2):
    """test_metrics_gpu.make_model (every parameter moved by N(0, 0.05), so that samples differ visibly), with the vgg
    backbones moved by N(0, 0.02) only: at 0.05 their 13 convolution layers turn chaotic (eager and graphed looped calls of
    the same model then differ by 0.1 in fp32), and the fp32 skip-half GEMM, whose split-K depends on the number of rows,
    sums in another order for a chain's batched sources than for one segment's."""
    if backbone.startswith("vgg"):
        from p2pvg_b200.models import vgg_64, vgg_128
        from p2pvg_b200.models.p2p_model import P2PModel
        opt = types.SimpleNamespace(dataset="mnist", backbone_net=vgg_64 if backbone == "vgg_64" else vgg_128, lr=1e-3, beta1=0.9,
                                    beta=1e-4, weight_cpc=100.0, weight_align=0.5, skip_prob=0.5, n_past=n_past,
                                    last_frame_skip=lfs, batch_size=B)
        torch.manual_seed(0)
        model = P2PModel(B, C, 128, 10, 256, 1, 1, 2, opt=opt)
        g = torch.Generator().manual_seed(1)
        with torch.no_grad():
            for p in model.parameters():
                p.add_(0.02 * torch.randn(p.shape, generator=g))
        return model.cuda().eval()
    model = make_model(backbone, C, B, n_past)
    model.opt.last_frame_skip = lfs
    return model


def clip(model, T, B, seed):
    g = torch.Generator().manual_seed(seed)
    if model.is_pose:
        return torch.randn(T, B, 17, 3, generator=g).cuda()
    enc = model.encoder
    return torch.rand(T, B, enc.nc, enc.image_width, enc.image_width, generator=g).cuda()


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("backbone,C,n_past,lfs", CONFIGS, ids=[f"{b}-C{c}-np{n}{'-lfs' if l else ''}" for b, c, n, l in CONFIGS])
def test_chain_equals_looped_calls(backbone, C, n_past, lfs, prec):
    """Unequal segments, one len_output longer than its slice (the posterior falls back to h_cpaw), skipped frames; nsample
    1 and 3.  Same frames, same eps consumption, same NumPy stream afterwards, same final .hidden."""
    T, B = 9, 2
    cps, lens = [0, 3, 5, 8], [4, 6, 4]
    with precision(prec):
        model = config_model(backbone, C, n_past, lfs, B)
        x = clip(model, T, B, seed=T + n_past)
        for ns, mode, skip_frame in ((1, "full", True), (3, "prior", True), (3, "posterior", False)):
            what = f"{backbone} {prec} nsample={ns} {mode} skip_frame={skip_frame}"
            S = n_exec_chain(5, cps, lens, model.opt, skip_frame)
            g = torch.Generator().manual_seed(ns)
            draws = [torch.randn(ns * B, model.z_dim, generator=g) for _ in range(2 * S)]
            got = run(lambda: model.p2p_generate_multi_cp(x, cps, lens, model_mode=mode, skip_frame=skip_frame, nsample=ns), 5, draws)
            after_chain, h_chain = np.random.uniform(), hidden_of(model)
            ref = run(lambda: looped(model, x, cps, lens, mode, skip_frame, ns), 5, draws)
            assert np.random.uniform() == after_chain, what
            assert_same_as_looped(got, ref, ns, what)
            assert_hidden_same(h_chain, hidden_of(model), what)


# ---- 3. one replay, tables not baked, memory --------------------------------------------------------------------------
def test_one_replay_per_chain_and_tables_not_baked(monkeypatch):
    T, B, cps = 9, 2, [0, 2, 5, 8]
    with precision("fp32"):
        model = config_model("dcgan_64", 1, 1, False, B)
        replays = []
        real = torch.cuda.CUDAGraph.replay
        monkeypatch.setattr(torch.cuda.CUDAGraph, "replay", lambda self: (replays.append(1), real(self))[1])
        eng = model._graphed_engine()
        for j in range(3):   # same signature (skip_frame=False), other frames and eps on every call
            x = clip(model, T, B, seed=40 + j)
            S = n_exec_chain(j, cps, None, model.opt, False)
            g = torch.Generator().manual_seed(50 + j)
            draws = [torch.randn(B, model.z_dim, generator=g) for _ in range(2 * S)]
            replays.clear()
            got = run(lambda: model.p2p_generate_multi_cp(x, cps), j, draws)
            assert len(replays) == 1, "a chain is one graph replay"
            h = hidden_of(model)
            ref = run(lambda: looped(model, x, cps, None), j, draws)
            assert_same_as_looped(got, ref, 1, f"call {j}")
            assert_hidden_same(h, hidden_of(model), f"call {j}")
            if j == 0:
                first = [[f.clone() for f in seq] for seq in got]
                n_graphs, mem = len(eng._graphs), eng.memory_bytes()
        for a, b in zip(first, got):
            assert not all(torch.equal(fa, fb) for fa, fb in zip(a[1:], b[1:])), "the frames of call 0 came back"
        # the cache holds the chain beside the three single-call signatures of the looped calls, within MAX_GRAPHS
        assert len(eng._graphs) == n_graphs and mem > 0
        eng.clear()
        assert eng.memory_bytes() == 0 and len(eng._graphs) == 0


def test_chain_shares_the_graph_cache_with_single_calls():
    from p2pvg_b200.gen_engine import MAX_GRAPHS
    T, B = 9, 1
    with precision("fp32"):
        model = config_model("dcgan_64", 1, 1, False, B)
        eng = model._graphed_engine()
        x = clip(model, T, B, seed=3)
        for cps in ([0, 4, 8], [0, 2, 8], [0, 3, 6, 8], [0, 1, 8], [0, 5, 8]):
            model.p2p_generate_multi_cp(x, cps)
            assert len(eng._graphs) <= MAX_GRAPHS
        model.p2p_generate_graphed(x, T, T - 1)
        assert len(eng._graphs) == MAX_GRAPHS


# ---- 4. a training step between two calls ------------------------------------------------------------------------------
def test_training_step_between_two_chains_is_picked_up():
    c = load()["cases"][0]
    cps, lens = c["cp_ixs"], c["len_outputs"]
    with precision("bf16"):
        model = case_model(c)
        x = case_frames(c).cuda()
        model.train()
        model(x)                     # parameters now live in the training arena (stable addresses)
        model.eval()
        S = n_exec_chain(3, cps, lens, model.opt, True)
        g = torch.Generator().manual_seed(3)
        draws = [torch.randn(x.shape[1], model.z_dim, generator=g) for _ in range(2 * S)]
        before = run(lambda: model.p2p_generate_multi_cp(x, cps, lens, skip_frame=True), 3, draws)
        before = [[f.clone() for f in seq] for seq in before]
        eng = model._graphed_engine()
        n_graphs = len(eng._graphs)
        model.train()
        model(x)
        torch.cuda.synchronize()
        model.eval()
        got = run(lambda: model.p2p_generate_multi_cp(x, cps, lens, skip_frame=True), 3, draws)
        h = hidden_of(model)
        assert len(eng._graphs) == n_graphs, "the second chain must reuse the cached graph"
        assert max((a - b).abs().max().item() for sa, sb in zip(got, before) for a, b in zip(sa[1:], sb[1:])) > 1e-3, \
            "the update was not picked up"
        ref = run(lambda: looped(model, x, cps, lens, skip_frame=True), 3, draws)
        assert_same_as_looped(got, ref, 1, "after a training step")
        assert_hidden_same(h, hidden_of(model), "after a training step")


# ---- 5. scoring ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("backbone,C,n_past", [("dcgan_64", 1, 1), ("dcgan_128", 3, 2), ("vgg_64", 3, 1), ("vgg_128", 1, 2),
                                               ("h36m_mlp", 1, 2)])
def test_evaluate_cp_ixs(backbone, C, n_past, prec):
    T, B, ns = 10, 2, 3
    cps = [0, 4, 6, 9] if n_past == 1 else [0, 3, 6, 9]
    with precision(prec):
        model = config_model(backbone, C, n_past, False, B)
        x = clip(model, T, B, seed=7)
        S = n_exec_chain(8, cps, None, model.opt, False)
        g = torch.Generator().manual_seed(8)
        draws = [torch.randn(ns * B, model.z_dim, generator=g) for _ in range(2 * S)]
        ev = run(lambda: model.p2p_evaluate(x, nsample=ns, cp_ixs=cps), 8, draws)
        h = hidden_of(model)
        res = run(lambda: model.p2p_generate_multi_cp(x, cps, nsample=ns), 8, draws)
        for m in MODS:   # the same draws give the same generation, bit for bit
            for (h1, c1), (h2, c2) in zip(h[m], getattr(model, m).hidden):
                assert torch.equal(h1, h2) and torch.equal(c1, c2), m
        want = [a + i for a, b in zip(cps, cps[1:]) for i in range(n_past, b - a + 1)]
        assert ev["frames"] == want and set(cps[1:]) <= set(want)
        # the frames and their clip indices, scored by the public metrics functions
        pred, gts = [], []
        for k, (a, b) in enumerate(zip(cps, cps[1:])):
            for i in range(n_past, b - a + 1):
                pred.append(torch.stack([res[k][s][i] for s in range(ns)]))   # [ns, B, ...]
                gts.append(x[a + i])
        P = torch.stack(pred).reshape(-1, *x.shape[2:]).contiguous()          # (frame, sample, b)
        Gt = torch.stack(gts).unsqueeze(1).expand(-1, ns, -1, *([-1] * (x.dim() - 2))).reshape(-1, *x.shape[2:]).contiguous()
        ref = metrics.pose_metrics(P, Gt) if model.is_pose else metrics.frame_metrics(P, Gt)
        for key, v in ref.items():
            v = v.view(len(want), ns, B).permute(1, 0, 2)
            assert ev[key].shape == (ns, len(want), B)
            assert torch.allclose(ev[key], v, rtol=1e-9, atol=1e-9, equal_nan=True), key
        # one segment is p2p_evaluate over the whole clip under the same draws
        S1 = n_exec_chain(9, [0, T - 1], None, model.opt, False)
        d1 = [torch.randn(ns * B, model.z_dim, generator=g) for _ in range(2 * S1)]
        one = run(lambda: model.p2p_evaluate(x, nsample=ns, cp_ixs=[0, T - 1]), 9, d1)
        whole = run(lambda: model.p2p_evaluate(x, nsample=ns), 9, d1)
        assert one["frames"] == whole["frames"] == list(range(n_past, T))
        for key in (metrics.POSE_METRICS if model.is_pose else metrics.FRAME_METRICS):
            assert torch.equal(one[key], whole[key]), key
