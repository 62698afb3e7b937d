"""P2PModel.p2p_generate_graphed for the vgg_64 / vgg_128 backbones (p2pvg_b200/gen_engine_vgg.py): one CUDA-graph replay per
call against the reference's frames (tests/golden/vgg_gen.pt), the CPU oracle (vgg_128, 3 channels) and the eager
p2p_generate fed the same draws; its launch composition; and the kernels it adds or newly reaches against float64: the two
thin-end kernels p2pvg_vgg_first_eval / p2pvg_vgg_last_eval and the eval-BatchNorm epilogue of p2pvg_conv_gemm kind 3.

Tolerances on frames in [0, 1], as for dcgan (test_generate_engine_gpu.py): fp32 2e-4 max / 2e-5 mean, bf16 4e-2 max /
6e-3 mean."""
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import p2p_oracle as O
from tests.test_generate_engine_gpu import TOL, close, draws_for, n_exec_of, precision, run
from tests.test_vgg_generate_cpu import case_frames, full_frames, load

pytestmark = pytest.mark.gpu


def build_model(c):
    """The fixture case's P2PModel (vgg_64 / vgg_128) on the GPU in eval mode: the reference's initial weights (same init
    seed) and the fixture's BatchNorm buffers."""
    from p2pvg_b200.models import vgg_64, vgg_128
    from p2pvg_b200.models.p2p_model import P2PModel
    o, cfg = c["opt"], c["cfg"]
    opt = types.SimpleNamespace(dataset="mnist", backbone_net=vgg_128 if cfg["vgg_width"] == 128 else vgg_64, **o)
    torch.manual_seed(c["init_seed"])
    model = P2PModel(o["batch_size"], cfg["channels"], cfg["g_dim"], cfg["z_dim"], cfg["rnn_size"], 1, 1, 2, opt=opt)
    ref = O.build_state(cfg, seed=c["init_seed"])
    for m in ("encoder", "decoder"):
        sd = getattr(model, m).state_dict()
        for k, v in ref[m].items():
            assert torch.equal(sd[k], v), f"{m}.{k}"
    for m, bufs in c["bn_buffers"].items():
        mod = getattr(model, m)
        for k, v in bufs.items():
            owner, _, leaf = k.rpartition(".")
            getattr(mod.get_submodule(owner), leaf).copy_(v)
    return model.cuda().eval()


def errors(a, b):
    e = (a.float().cpu() - b.float().cpu()).abs()
    return e.max().item(), e.mean().item()


# ---- 1. the reference's own frames ----------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("case", range(3))
def test_graphed_matches_reference_fixture(case, prec):
    """Every run of the fixture: zero-frame pattern exact, the digest samples of every frame within the worst-pixel bound,
    and the frames stored in full within both bounds.  The eager p2p_generate's errors on the same frames are printed beside
    the graphed ones."""
    c = load()["cases"][case]
    tmax, _ = TOL[prec]
    with precision(prec):
        model = build_model(c)
        x = case_frames(c).cuda()
        for r in c["runs"]:
            draws = [r["eps"][s, j] for s in range(r["n_exec"]) for j in (0, 1)]
            what = f"{c['case']} {prec} {r['model_mode']}/skip_frame={r['skip_frame']}"
            kw = dict(model_mode=r["model_mode"], skip_frame=r["skip_frame"])
            seq = run(lambda: model.p2p_generate_graphed(x, c["len_output"], c["eval_cp_ix"], **kw), r["np_seed"], draws)
            eager = run(lambda: model.p2p_generate(x, c["len_output"], c["eval_cp_ix"], **kw), r["np_seed"], draws)
            refs = full_frames(seq, r)
            dig = [max(abs(float(v)) for v in (f.detach().double().reshape(-1).cpu()[d["idx"]] - d["samples"])) for f, d in
                   zip(seq, r["digests"])]
            dig_e = [max(abs(float(v)) for v in (f.detach().double().reshape(-1).cpu()[d["idx"]] - d["samples"])) for f, d in
                     zip(eager, r["digests"])]
            print(f"{what}: digest samples worst graphed {max(dig):.2e} eager {max(dig_e):.2e}; full frames graphed "
                  f"{[f'{m:.2e}/{a:.2e}' for m, a in (errors(f, ref) for f, ref in refs)]}, eager "
                  f"{[f'{m:.2e}/{a:.2e}' for m, a in (errors(f, ref) for f, ref in full_frames(eager, r))]}")
            assert len(seq) == c["len_output"]
            assert [bool((f == 0).all()) for f in seq] == r["zero_frames"], what
            for i, (f, d) in enumerate(zip(seq, r["digests"])):
                v = f.detach().double().reshape(-1).cpu()
                assert (v[d["idx"]] - d["samples"]).abs().max().item() <= tmax, f"{what} frame {i}"
            for f, ref in refs:
                close(f, ref, prec, what)


# ---- 2. vgg_128, three channels, against the CPU oracle ---------------------------------------------------------------
def model128(n_past, lfs, seed=5):
    from p2pvg_b200.models import vgg_128
    from p2pvg_b200.models.p2p_model import P2PModel
    cfg = dict(g_dim=128, z_dim=10, rnn_size=256, channels=3, image_width=128, backbone="vgg", vgg_width=128,
               predictor_rnn_layers=2, posterior_rnn_layers=1, prior_rnn_layers=1)
    opt = types.SimpleNamespace(dataset="mnist", backbone_net=vgg_128, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0,
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


@pytest.mark.parametrize("lfs", [False, True])
@pytest.mark.parametrize("n_past", [1, 2])
def test_vgg128_rgb_matches_oracle(n_past, lfs):
    from p2pvg_b200.gen_engine import plan_slots
    T, B = 4, 2
    x = torch.rand(T, B, 3, 128, 128, generator=torch.Generator().manual_seed(3))
    for prec in ("fp32", "bf16"):
        with precision(prec):
            model, state, oopt = model128(n_past, lfs)
            for len_output, eval_cp_ix, skip_frame in ((T, T - 1, True), (T + 2, T + 1, True)):
                np_seed = 11 + len_output
                probs = np.random.RandomState(np_seed).uniform(0, 1, len_output - 1)
                S = len(plan_slots(len_output, T, probs, 0.5, n_past, skip_frame, eval_cp_ix))
                draws = draws_for(S, B, 10, seed=len_output)
                got = run(lambda: model.p2p_generate_graphed(x.cuda(), len_output, eval_cp_ix, skip_frame=skip_frame), np_seed, draws)
                eps = torch.stack([torch.stack([draws[2 * s], draws[2 * s + 1]]) for s in range(S)])
                ref = O.p2p_generate(state, list(x), len_output, eval_cp_ix, oopt, "vgg", eps, probs, skip_frame=skip_frame)
                assert len(got) == len(ref) == len_output
                for i, (a, b) in enumerate(zip(got, ref)):
                    close(a, b, prec, f"{prec} len_output={len_output} frame {i}")


# ---- 3. against the eager path with the same draws ----------------------------------------------------------------------
def hidden_of(model):
    return {m: [(h.clone(), c.clone()) for h, c in getattr(model, m).hidden] for m in ("frame_predictor", "posterior", "prior")}


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("case", [0, 1])
def test_graphed_matches_eager(case, prec):
    """nsample = 1 against p2p_generate, nsample = 3 against p2p_generate_samples and against three looped graphed calls
    (bf16: the skip half is read as the kind-3 addend of image n % nsrc), and init_hidden=False with the written-back .hidden."""
    c = load()["cases"][case]
    with precision(prec):
        model = build_model(c)
        x = case_frames(c).cuda()
        L, cp, B, ns = c["len_output"], c["eval_cp_ix"], x.shape[1], 3
        S = n_exec_of(5, L, x.shape[0], model.opt, True)
        draws = draws_for(S, B, 10, 1)
        got = run(lambda: model.p2p_generate_graphed(x, L, cp, skip_frame=True), 5, draws)
        ref = run(lambda: model.p2p_generate(x, L, cp, skip_frame=True), 5, draws)
        for i, (a, b) in enumerate(zip(got, ref)):
            close(a, b, prec, f"nsample=1 frame {i}")
        d = torch.randn(ns, S, 2, B, 10, generator=torch.Generator().manual_seed(9))
        looped = [run(lambda: model.p2p_generate_graphed(x, L, cp, skip_frame=True), 5, [d[s, i, j] for i in range(S) for j in (0, 1)])
                  for s in range(ns)]
        looped = [[f.clone() for f in seq] for seq in looped]
        tiled = [d[:, i, j].reshape(ns * B, 10) for i in range(S) for j in (0, 1)]
        batched = run(lambda: model.p2p_generate_graphed(x, L, cp, skip_frame=True, nsample=ns), 5, tiled)
        eager = run(lambda: model.p2p_generate_samples(x, ns, L, cp, skip_frame=True), 5, tiled)
        assert len(batched) == ns and all(len(b) == L for b in batched)
        for s in range(ns):
            for i, (a, b, e) in enumerate(zip(batched[s], looped[s], eager[s])):
                assert a.shape == b.shape == e.shape
                close(a, b, prec, f"sample {s} frame {i} vs looped graphed")
                close(a, e, prec, f"sample {s} frame {i} vs eager samples")
        g = torch.Generator().manual_seed(4)
        start = {m: [(torch.randn(B, getattr(model, m).hidden_size, generator=g).cuda(),
                      torch.randn(B, getattr(model, m).hidden_size, generator=g).cuda()) for _ in range(getattr(model, m).n_layers)]
                 for m in ("frame_predictor", "posterior", "prior")}
        res = {}
        for name, fn in (("graphed", model.p2p_generate_graphed), ("eager", model.p2p_generate)):
            for m, hc in start.items():
                getattr(model, m).hidden = [(h.clone(), c_.clone()) for h, c_ in hc]
            seq = run(lambda: fn(x, L, cp, skip_frame=True, init_hidden=False), 5, draws)
            res[name] = ([f.clone() for f in seq], hidden_of(model))
        for a, b in zip(res["graphed"][0], res["eager"][0]):
            close(a, b, prec, "init_hidden=False")
        tol = 1e-4 if prec == "fp32" else 2e-2
        for m in start:
            for (h1, c1), (h2, c2) in zip(res["graphed"][1][m], res["eager"][1][m]):
                assert (h1 - h2).abs().max().item() < tol and (c1 - c2).abs().max().item() < tol, m


# ---- 4. one graph, many calls; training steps in between ---------------------------------------------------------------
def test_one_graph_two_skip_patterns_no_aliasing():
    from p2pvg_b200.gen_engine import plan_slots
    c = load()["cases"][0]
    with precision("bf16"):
        model = build_model(c)
        x = case_frames(c).cuda()
        L, T, opt = c["len_output"], x.shape[0], model.opt
        pats = {}
        for sd in range(300):
            probs = np.random.RandomState(sd).uniform(0, 1, L - 1)
            pl = plan_slots(L, T, probs, opt.skip_prob, opt.n_past, True, c["eval_cp_ix"])
            pats.setdefault(len(pl), {}).setdefault(tuple(p[0] for p in pl), sd)
        S, by_pat = max(((k, v) for k, v in pats.items() if len(v) >= 2), key=lambda kv: len(kv[1]))
        outs = []
        for j, sd in enumerate(list(by_pat.values())[:2]):
            draws = draws_for(S, x.shape[1], 10, seed=40 + j)
            got = run(lambda: model.p2p_generate_graphed(x, L, c["eval_cp_ix"], skip_frame=True), sd, draws)
            ref = run(lambda: model.p2p_generate(x, L, c["eval_cp_ix"], skip_frame=True), sd, draws)
            for a, b in zip(got, ref):
                close(a, b, "bf16")
            outs.append((got, [f.clone() for f in got]))
        assert len(model._gen_engine._graphs) == 1, "both calls must replay one graph"
        for a, b in zip(*outs[0]):
            assert torch.equal(a, b), "a returned frame aliases graph memory"
        assert model._gen_engine.memory_bytes() > 0


def test_training_steps_between_calls_are_picked_up():
    """A training step between two calls changes the frames; after a second step the cached graph is reused (the parameters
    stay in the training arena) and still matches the eager path on the updated weights."""
    c = load()["cases"][1]
    with precision("bf16"):
        model = build_model(c)
        x = case_frames(c).cuda()
        L, cp = c["len_output"], c["eval_cp_ix"]
        S = n_exec_of(0, L, x.shape[0], model.opt, False)
        draws = draws_for(S, x.shape[1], 10, 2)
        before = [f.clone() for f in run(lambda: model.p2p_generate_graphed(x, L, cp), 0, draws)]
        for step in range(2):
            model.train()
            model(x)
            torch.cuda.synchronize()
            model.eval()
            n_graphs = len(model._gen_engine._graphs)
            got = [f.clone() for f in run(lambda: model.p2p_generate_graphed(x, L, cp), 0, draws)]
            if step == 1:
                assert len(model._gen_engine._graphs) == n_graphs, "the second step must reuse the cached graph"
            ref = run(lambda: model.p2p_generate(x, L, cp), 0, draws)
            assert max((a - b).abs().max().item() for a, b in zip(got[1:], before[1:])) > 1e-3, "the update was not picked up"
            for a, b in zip(got, ref):
                close(a, b, "bf16", f"after step {step}")
            before = got


# ---- 5. launch composition ---------------------------------------------------------------------------------------------
def _recording_backend():
    from p2pvg_b200._lib import CudaKernels

    class Recording(CudaKernels):
        def __init__(self, dev):
            super().__init__(dev)
            self.calls = []

        def __getattribute__(self, name):
            attr = object.__getattribute__(self, name)
            if name.startswith("_") or name in ("calls", "launches", "lib", "device", "ws_gen", "gemm_workspace", "bn_workspace") \
                    or not callable(attr):
                return attr
            calls = object.__getattribute__(self, "calls")

            def rec(*a, **kw):
                calls.append((name, a, kw))
                return attr(*a, **kw)
            return rec
    return Recording("cuda")


@pytest.mark.parametrize("case", [0, 1, 2])
def test_launch_composition_bf16(case, monkeypatch):
    """Per captured run: every >= 64-channel 3x3 layer of every encode and decode is exactly one conv_gemm kind-3 launch with
    the eval epilogue (LeakyReLU), each skip half one plain kind-3 launch, each thin end one launch; no im2col3, col2im3,
    gather_add or explicit 4x4 lowering."""
    from p2pvg_b200 import infer
    from p2pvg_b200._lib import ACT_LRELU
    from p2pvg_b200.engine_vgg import VGG_DEC, VGG_DEC_128, VGG_ENC, VGG_ENC_128
    from p2pvg_b200.gen_engine import plan_slots
    c = load()["cases"][case]
    K = _recording_backend()
    monkeypatch.setattr(infer, "kernels_for", lambda dev: K)
    with precision("bf16"):
        model = build_model(c)
        x = case_frames(c).cuda()
        L, cp, T = c["len_output"], c["eval_cp_ix"], x.shape[0]
        r = c["runs"][1]
        draws = [r["eps"][s, j] for s in range(r["n_exec"]) for j in (0, 1)]
        run(lambda: model.p2p_generate_graphed(x, L, cp, skip_frame=True), r["np_seed"], draws)
    W = c["cfg"]["vgg_width"]
    ENC, DEC = (VGG_ENC_128, VGG_DEC_128) if W == 128 else (VGG_ENC, VGG_DEC)
    enc_shapes = [(cin, cout, W >> i) for i, st in enumerate(ENC) for j, (cin, cout) in enumerate(st) if cin is not None]
    dec_shapes = [(cin // 2 if j == 0 else cin, cout, 8 << k) for k, st in enumerate(DEC) for j, (cin, cout) in enumerate(st)]
    n_past, lfs = c["opt"]["n_past"], c["opt"]["last_frame_skip"]
    S = len(plan_slots(L, T, r["probs"].numpy(), c["opt"]["skip_prob"], n_past, True, cp))
    n_tf = min(n_past - 1, L - 1)
    n_dec = max(S - n_tf, 0)
    n_enc = 1 + max(n_dec - 1, 0)
    n_halves = (n_dec if lfs else 1) if n_dec else 0
    names = [k for k, _, _ in K.calls]
    for banned in ("im2col3", "col2im3", "gather_add", "im2col", "col2im", "act_fwd"):
        assert banned not in names, banned
    runs = 2   # the uncaptured warm-up and the captured run of the first call
    conv = [(a, kw) for k, a, kw in K.calls if k == "conv_gemm"]
    assert all(a[0] == 3 for a, _ in conv)
    ev = sorted((a[7], a[8], a[5]) for a, kw in conv if kw.get("eval_scale") is not None)
    assert all(kw.get("act") == ACT_LRELU for a, kw in conv if kw.get("eval_scale") is not None)
    assert ev == sorted(runs * (n_enc * enc_shapes + n_dec * dec_shapes))
    plain = sorted((a[7], a[8], a[5]) for a, kw in conv if kw.get("eval_scale") is None)
    halves = [(cin // 2, cout, 8 << k) for k, st in enumerate(DEC) for cin, cout in st[:1]]
    assert plain == sorted(runs * n_halves * halves)
    assert names.count("vgg_first_eval") == runs * n_enc
    assert names.count("vgg_last_eval") == runs * n_dec
    assert len(model._gen_engine._graphs) == 1


# ---- 6. kernels against float64 -----------------------------------------------------------------------------------------
def _lrelu(v):
    return torch.where(v > 0, v, 0.2 * v)


@pytest.mark.parametrize("N", [1, 7, 130])
@pytest.mark.parametrize("W", [64, 128])
@pytest.mark.parametrize("nc", [1, 3])
def test_vgg_first_eval_kernel(nc, W, N):
    from p2pvg_b200._lib import kernels_for
    K = kernels_for("cuda")
    g = torch.Generator().manual_seed(nc * 1000 + W + N)
    x = torch.rand(N, nc, W, W, generator=g)
    w, bias = 0.3 * torch.randn(64, nc, 3, 3, generator=g), 0.1 * torch.randn(64, generator=g)
    scale, shift = 1 + 0.2 * torch.randn(64, generator=g), 0.1 * torch.randn(64, generator=g)
    ref = F.conv2d(x.double(), w.double(), bias.double(), padding=1)
    ref = _lrelu(ref * scale.double()[:, None, None] + shift.double()[:, None, None]).permute(0, 2, 3, 1).contiguous()
    mag = (F.conv2d(x.double(), w.double().abs(), bias.double().abs(), padding=1) * scale.double().abs()[:, None, None]
           + shift.double().abs()[:, None, None]).permute(0, 2, 3, 1)
    xd, wd, bd, sd, hd = (t.cuda() for t in (x, w, bias, scale, shift))
    for dt in (torch.float32, torch.bfloat16):
        y = torch.full((N, W, W, 64), float("nan"), device="cuda", dtype=dt)
        K.vgg_first_eval(xd, nc, wd, bd, sd, hd, y, N, W, W)
        got = y.double().cpu()
        bound = 30 * 2.0 ** -24 * mag + (2.0 ** -8) * ref.abs() * (dt == torch.bfloat16)   # 28 fp32 FFMA, one bf16 rounding
        err = (got - ref).abs()
        assert (err <= bound + 1e-12).all(), (str(dt), (err - bound).max().item())


@pytest.mark.parametrize("N", [1, 7, 130])
@pytest.mark.parametrize("W", [64, 128])
@pytest.mark.parametrize("nc", [1, 3])
def test_vgg_last_eval_kernel(nc, W, N):
    from p2pvg_b200._lib import kernels_for
    K = kernels_for("cuda")
    g = torch.Generator().manual_seed(nc * 2000 + W + N)
    d = torch.randn(N, W, W, 64, generator=g)
    w, bias = 0.05 * torch.randn(64, nc, 3, 3, generator=g), 0.1 * torch.randn(nc, generator=g)
    wd, bd = w.cuda(), bias.cuda()
    for dt in (torch.float32, torch.bfloat16):
        dq = d.to(dt)
        pre = F.conv_transpose2d(dq.double().permute(0, 3, 1, 2), w.double(), bias.double(), padding=1)
        ref = torch.sigmoid(pre)
        mag = F.conv_transpose2d(dq.double().abs().permute(0, 3, 1, 2), w.double().abs(), bias.double().abs(), padding=1)
        out = torch.full((N, nc, W, W), float("nan"), device="cuda")
        K.vgg_last_eval(dq.cuda(), wd, bd, out, nc, N, W, W)
        err = (out.double().cpu() - ref).abs()
        bound = 0.25 * 600 * 2.0 ** -24 * mag + 1e-6   # sigmoid' <= 1/4: fp32 accumulation of 577 terms, then expf
        assert (err <= bound).all(), (str(dt), (err - bound).max().item())


def _vgg_conv3_shapes():
    """(Ck, Cn, H) of every >= 64-channel 3x3 layer of vgg_64 and vgg_128, the decoder stage entries with Ck = the up half."""
    from p2pvg_b200.engine_vgg import VGG_DEC, VGG_DEC_128, VGG_ENC, VGG_ENC_128
    out = set()
    for W, ENC, DEC in ((64, VGG_ENC, VGG_DEC), (128, VGG_ENC_128, VGG_DEC_128)):
        out |= {(cin, cout, W >> i) for i, st in enumerate(ENC) for cin, cout in st if cin is not None}
        out |= {(cin // 2 if j == 0 else cin, cout, 8 << k) for k, st in enumerate(DEC) for j, (cin, cout) in enumerate(st)}
    return sorted(out)


@pytest.mark.parametrize("B", [1, 16, 100])
@pytest.mark.parametrize("Ck,Cn,H", _vgg_conv3_shapes())
def test_conv_gemm_kind3_eval_epilogue(Ck, Cn, H, B):
    """kind 3 with the eval-BatchNorm epilogue against kind 3 with a raw fp32 output + bn_act, with no addend and with a bf16
    or fp32 addend of nsrc images read through grp_src (image n adds addend image n % nsrc): covers the 64 -> 64 resident-
    weight ring, 128-row tiles spanning several 8 x 8 images, and multi-round persistent schedules (B = 100)."""
    from p2pvg_b200._lib import ACT_LRELU, ACT_TANH, kernels_for
    K = kernels_for("cuda")
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(Ck + 7 * Cn + 31 * H + B)
    M = B * H * H
    a = torch.randn(M * Ck, device=dev, generator=g).bfloat16()
    w = (0.05 * torch.randn(9 * Ck * Cn, device=dev, generator=g)).bfloat16()
    bias = torch.randn(Cn, device=dev, generator=g)
    gamma, beta = 1 + 0.1 * torch.randn(Cn, device=dev, generator=g), 0.1 * torch.randn(Cn, device=dev, generator=g)
    rmean, rvar = 0.1 * torch.randn(Cn, device=dev, generator=g), 0.5 + torch.rand(Cn, device=dev, generator=g)
    sc, sh = torch.empty(Cn, device=dev), torch.empty(Cn, device=dev)
    K.bn_eval_coeffs(gamma, beta, rmean, rvar, Cn, sc, sh)
    nsrc = max(B // 4, 1)
    grp = torch.zeros(B // nsrc, dtype=torch.int32, device=dev)
    for add_dt in (None, torch.bfloat16, torch.float32):
        addend = None if add_dt is None else torch.randn(nsrc * H * H * Cn, device=dev, generator=g).to(add_dt)
        kw = dict(bias=bias, addend=addend, grp_src=grp if addend is not None else None, imgs_per_group=nsrc if addend is not None else 0)
        raw = torch.empty(M * Cn, device=dev)
        K.conv_gemm(3, a, w, raw, B, H, H, Ck, Cn, **kw)
        for act in (ACT_LRELU, ACT_TANH):
            ref = torch.empty_like(raw)
            K.bn_act(raw, ref, sc, sh, 1, M, Cn, act)
            got = torch.full_like(raw, float("nan"))
            K.conv_gemm(3, a, w, got, B, H, H, Ck, Cn, eval_scale=sc, eval_shift=sh, act=act, **kw)
            torch.cuda.synchronize()
            assert torch.allclose(got, ref, rtol=1e-5, atol=1e-5), (str(add_dt), act, (got - ref).abs().max().item())
            got16 = torch.full((M * Cn,), float("nan"), device=dev, dtype=torch.bfloat16)
            K.conv_gemm(3, a, w, got16, B, H, H, Ck, Cn, eval_scale=sc, eval_shift=sh, act=act, **kw)
            assert torch.allclose(got16.float(), ref, rtol=2 ** -8, atol=1e-5), (str(add_dt), act)
    # the addend really is image n % nsrc: the raw output minus the addend-free output is the addend, tiled
    if B > 1:
        addend = torch.randn(nsrc * H * H * Cn, device=dev, generator=g)
        with_add, without = torch.empty(M * Cn, device=dev), torch.empty(M * Cn, device=dev)
        K.conv_gemm(3, a, w, with_add, B, H, H, Ck, Cn, bias=bias, addend=addend, grp_src=grp, imgs_per_group=nsrc)
        K.conv_gemm(3, a, w, without, B, H, H, Ck, Cn, bias=bias)
        diff = (with_add - without).view(B // nsrc, nsrc * H * H * Cn)
        assert torch.allclose(diff, addend.expand_as(diff), atol=1e-4)


# ---- 7. frames that do not fit --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("frames", ["vgg128_frames", "poses"])
def test_frame_shape_rejected_on_cuda_model(frames):
    c = load()["cases"][0]
    model = build_model(c)
    B = c["opt"]["batch_size"]
    x = [torch.zeros(B, 3, 128, 128, device="cuda")] * 3 if frames == "vgg128_frames" else [torch.zeros(B, 17, 3, device="cuda")] * 3
    with pytest.raises(ValueError, match="^p2p_generate_graphed"):
        model.p2p_generate_graphed(x, 4, 3)
