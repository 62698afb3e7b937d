"""P2PModel.p2p_generate_lengths (p2pvg_b200/gen_engine.py) and generate.generate_video: every output length in ONE
CUDA-graph replay against the looped p2p_generate_graphed calls it stands for, for every backbone in both P2PVG_PRECISION
modes; p2pvg_lstm_step with per-row counters against one launch per group; the composition kernel p2pvg_vis_tiles against
the reference generate.py's pictures (tests/golden/generate_ref.pt) and its rejections; generate_video's random streams
against generate.py's loop of eager calls.

Tolerances against the looped calls as test_multi_cp_gpu.py (frames rtol 1e-4 + atol 2e-5, written-back LSTM state rtol 1e-4
+ atol 1e-5), with its models (the vgg backbones moved by N(0, 0.02) only: the fp32 GEMM's split-K depends on the number of
rows, and a replay runs each step on the rows of every length still generating)."""
import hashlib
import os
import sys
import types

import numpy as np
import pytest
import torch

from tests.test_generate_engine_gpu import TOL, precision, run
from tests.test_multi_cp_gpu import MODS, clip, config_model, hidden_of

pytestmark = pytest.mark.gpu
FIX = os.path.join(os.path.dirname(__file__), "golden", "generate_ref.pt")


def looped(model, x, lens, mode="full", ns=1):
    return [model.p2p_generate_graphed(x, L, L - 1, model_mode=mode, nsample=ns) for L in lens]


def flat(res, ns):
    return [(k, s, i, f) for k, seq in enumerate(res) for s, sq in enumerate([seq] if ns == 1 else seq) for i, f in enumerate(sq)]


def assert_same(got, ref, ns, what=""):
    a, b = flat(got, ns), flat(ref, ns)
    assert [t[:3] for t in a] == [t[:3] for t in b], what
    for (k, s, i, fa), (_, _, _, fb) in zip(a, b):
        assert fa.shape == fb.shape and torch.allclose(fa.float(), fb.float(), rtol=1e-4, atol=2e-5), \
            f"{what} length {k} sample {s} frame {i}: {(fa.float() - fb.float()).abs().max().item():.3e}"


def assert_hidden_same(ha, hb, what=""):
    for m in MODS:
        for (h1, c1), (h2, c2) in zip(ha[m], hb[m]):
            assert h1.shape == h2.shape, (what, m)
            assert torch.allclose(h1, h2, rtol=1e-4, atol=1e-5) and torch.allclose(c1, c2, rtol=1e-4, atol=1e-5), (what, m)


def draws_for(lens, rows, z, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(rows, z, generator=g) for L in lens for _ in range(2 * (L - 1))]


# ---- 1. per-row counters in p2pvg_lstm_step ------------------------------------------------------------------------------
def test_lstm_step_counter_rows_equals_one_launch_per_group():
    from p2pvg_b200._lib import LSTM_HEAD_GAUSSIAN, kernels_for
    dev = torch.device("cuda")
    K = kernels_for(dev)
    g = torch.Generator().manual_seed(0)
    R, ga, zd, gr, nG, L = 256, 128, 10, 6, 3, 2
    rows = gr * nG
    rnd = lambda *s: (0.1 * torch.randn(*s, generator=g)).to(dev)   # noqa: E731
    w = [(rnd(4 * R, R if l else R), rnd(4 * R), rnd(4 * R, R), rnd(4 * R)) for l in range(L)]
    w_embed, b_embed, w_out, b_out, w_out2, b_out2 = rnd(R, 2 * ga + 2), rnd(R), rnd(zd, R), rnd(zd), rnd(zd, R), rnd(zd)
    seg = rnd(3 * rows, ga)
    idx = torch.tensor([1, 2], dtype=torch.int32, device=dev)
    tuc, dt = rnd(nG).abs(), rnd(nG).abs()
    eps = rnd(rows, zd)
    h0, c0 = rnd(L, rows, R), rnd(L, rows, R)

    def launch(r0, r1, counters, cr):
        n = r1 - r0
        # the group's rows as a batch of its own: the segment rows [r0, r1) of each index, its own state and eps
        sg = seg.view(3, rows, ga)[:, r0:r1].contiguous().view(-1, ga)
        hs, cs = h0[:, r0:r1].clone(), c0[:, r0:r1].clone()
        wp = torch.tensor([t.data_ptr() for l in range(L) for t in w[l]], dtype=torch.int64, device=dev)
        sp = torch.tensor([t.data_ptr() for l in range(L) for t in (hs[l], cs[l], hs[l], cs[l])], dtype=torch.int64, device=dev)
        out = torch.zeros(n, zd, device=dev)
        K.lstm_step([dict(seg_a=sg, idx_a=idx[:1], ga=ga, seg_b=sg, idx_b=idx[1:], gb=ga, tuc=counters[0], dt=counters[1],
                          w_embed=w_embed, b_embed=b_embed, layers=L, layer_w=wp, state=sp, head=LSTM_HEAD_GAUSSIAN, out_dim=zd,
                          w_out=w_out, b_out=b_out, w_out2=w_out2, b_out2=b_out2, eps=eps[r0:r1].contiguous(), out=out,
                          counter_rows=cr)], n, R)
        return out, hs, cs

    got = launch(0, rows, (tuc, dt), gr)
    for q in range(nG):
        ref = launch(q * gr, (q + 1) * gr, (tuc[q:q + 1], dt[q:q + 1]), 0)
        assert torch.equal(got[0][q * gr:(q + 1) * gr], ref[0]), q
        assert torch.equal(got[1][:, q * gr:(q + 1) * gr], ref[1]) and torch.equal(got[2][:, q * gr:(q + 1) * gr], ref[2]), q
    with pytest.raises(RuntimeError, match="counter_rows"):
        launch(0, rows, (tuc, dt), -1)


# ---- 2. the looped p2p_generate_graphed calls ----------------------------------------------------------------------------
CONFIGS = [("dcgan_64", 1, 1, False), ("dcgan_64", 1, 2, True), ("dcgan_128", 3, 1, False), ("vgg_64", 3, 2, True),
           ("vgg_128", 1, 1, False), ("h36m_mlp", 1, 1, False), ("h36m_mlp", 1, 2, True)]


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("backbone,C,n_past,lfs", CONFIGS, ids=[f"{b}-C{c}-np{n}{'-lfs' if l else ''}" for b, c, n, l in CONFIGS])
def test_lengths_equal_looped_calls(backbone, C, n_past, lfs, prec):
    """Unsorted lengths with a duplicate, one below len(x) and one above; nsample 1 and 3; all three model modes.  Same
    frames, same eps consumption, same NumPy stream afterwards, same final .hidden (the last length's rows)."""
    T, B = 6, 2
    lens = [4, 9, 2, 9, 6]
    with precision(prec):
        model = config_model(backbone, C, n_past, lfs, B)
        x = clip(model, T, B, seed=T + n_past)
        for ns, mode in ((1, "full"), (3, "prior"), (3, "posterior")):
            what = f"{backbone} {prec} nsample={ns} {mode}"
            draws = draws_for(lens, ns * B, model.z_dim, seed=ns)
            got = run(lambda: model.p2p_generate_lengths(x, lens, model_mode=mode, nsample=ns), 5, draws)
            after, h = np.random.uniform(), hidden_of(model)
            ref = run(lambda: looped(model, x, lens, mode, ns), 5, draws)
            assert np.random.uniform() == after, what
            assert [len(seq if ns == 1 else seq[0]) for seq in got] == lens, what
            assert_same(got, ref, ns, what)
            assert_hidden_same(h, hidden_of(model), what)


# ---- 3. one replay, tables not baked, a training step between two calls --------------------------------------------------
def test_one_replay_per_call_and_tables_not_baked(monkeypatch):
    T, B, lens = 8, 2, [5, 8, 3]
    with precision("fp32"):
        model = config_model("dcgan_64", 1, 1, False, B)
        replays = []
        real = torch.cuda.CUDAGraph.replay
        monkeypatch.setattr(torch.cuda.CUDAGraph, "replay", lambda self: (replays.append(1), real(self))[1])
        eng = model._graphed_engine()
        for j in range(3):   # one signature; other frames and eps on every call
            x = clip(model, T, B, seed=40 + j)
            draws = draws_for(lens, B, model.z_dim, seed=50 + j)
            replays.clear()
            got = run(lambda: model.p2p_generate_lengths(x, lens), j, draws)
            assert len(replays) == 1, "every length in one graph replay"
            h = hidden_of(model)
            ref = run(lambda: looped(model, x, lens), j, draws)
            assert_same(got, ref, 1, f"call {j}")
            assert_hidden_same(h, hidden_of(model), f"call {j}")
            if j == 0:
                first = [[f.clone() for f in seq] for seq in got]
                mem = eng.memory_bytes()
        for a, b in zip(first, got):
            assert not all(torch.equal(fa, fb) for fa, fb in zip(a[1:], b[1:])), "the frames of call 0 came back"
        assert mem > 0 and any(k.startswith("Hsrc") and k != "Hsrc" for G in eng._graphs.values() for k in G.bufs)


def test_training_step_between_two_calls_is_picked_up():
    T, B, lens = 6, 2, [6, 3]
    with precision("bf16"):
        model = config_model("dcgan_64", 1, 1, False, B)
        x = clip(model, T, B, seed=3)
        model.train()
        model(x)                     # parameters now live in the training arena (stable addresses)
        model.eval()
        draws = draws_for(lens, B, model.z_dim, seed=3)
        before = [[f.clone() for f in seq] for seq in run(lambda: model.p2p_generate_lengths(x, lens), 3, draws)]
        eng = model._graphed_engine()
        n_graphs = len(eng._graphs)
        model.train()
        model(x)
        torch.cuda.synchronize()
        model.eval()
        got = run(lambda: model.p2p_generate_lengths(x, lens), 3, draws)
        assert len(eng._graphs) == n_graphs, "the second call must reuse the cached graph"
        assert max((a - b).abs().max().item() for sa, sb in zip(got, before) for a, b in zip(sa[1:], sb[1:])) > 1e-3
        assert_same(got, run(lambda: looped(model, x, lens), 3, draws), 1, "after a training step")


def test_rejections_before_any_draw():
    T, B = 4, 1
    model = config_model("dcgan_64", 1, 2, False, B)
    x = clip(model, T, B, seed=1)
    for bad in ([], [1, 5], [5, "a"], None, [2.5], [True, 4]):
        st = np.random.get_state()
        rng = torch.cuda.get_rng_state()
        with pytest.raises(ValueError):
            model.p2p_generate_lengths(x, bad)
        assert np.random.get_state()[2] == st[2] and np.array_equal(np.random.get_state()[1], st[1])
        assert torch.equal(torch.cuda.get_rng_state(), rng)
    with pytest.raises(ValueError):
        model.p2p_generate_lengths(x[:1], [5])   # len(x) < min(n_past, L)
    with pytest.raises(ValueError):
        model.p2p_generate_lengths(x, [5], model_mode="both")
    with pytest.raises(ValueError):
        model.p2p_generate_lengths(x, [5], nsample=0)


# ---- 4. generate_video -----------------------------------------------------------------------------------------------------
def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


class Recorder:
    """A stand-in for imageio (mimsave recorded) and torchvision's save_image (tensors recorded)."""

    def __init__(self):
        self.files = []
        self.imageio = types.SimpleNamespace(mimsave=self.mimsave)

    def mimsave(self, name, frames):
        self.files.append((name, [np.asarray(f) for f in frames]))

    def save_image(self, t, name, **kw):
        assert not kw
        self.files.append((name, t.detach().cpu().clone()))


@pytest.fixture
def recorder(monkeypatch):
    import torchvision.utils as vutils
    rec = Recorder()
    monkeypatch.setitem(sys.modules, "imageio", rec.imageio)
    monkeypatch.setattr(vutils, "save_image", rec.save_image)
    return rec


def digest_of(name, v):
    return sha(v.numpy()) if torch.is_tensor(v) else [sha(f) for f in v]


def test_composition_kernel_matches_reference_fixture():
    from p2pvg_b200 import generate
    from tests.generate_ref import stub_samples
    for c in torch.load(FIX, weights_only=False)["composition"]:
        seq, samples = stub_samples(c)
        seq, dev_samples = seq.cuda(), {L: s.cuda() for L, s in samples.items()}
        lens, ns = c["lens"], c["nsamples"]
        store1 = torch.cat([dev_samples[L].reshape(-1, *seq.shape[2:]) for L in lens]).contiguous()   # [L][sample][t]
        base = np.cumsum([0] + [ns * L for L in lens])
        H = int(seq.shape[3])
        plan = generate.plan_video(len(seq), lens, c["idxs"], H, lambda t: (0, t),
                                   lambda k, s, t: (1, int(base[k]) + s * lens[k] + t))
        pics = generate.compose(seq.reshape(-1, *seq.shape[2:]).contiguous(), store1, plan, int(seq.shape[2]), H)
        got = {}
        for L, idx, (gt, block, gif) in zip(lens, c["idxs"], pics):
            names = generate.file_names("OUT", L, len(idx))
            gt, block, gif = gt.cpu(), block.cpu(), gif.cpu().numpy()
            vals = [gt] + [block[:, ix * H:(ix + 1) * H] for ix in range(len(idx))] + [block] + \
                [[f[:, ix * H:(ix + 1) * H] for f in gif] for ix in range(len(idx))] + [list(gif)]
            got.update({n: digest_of(n, v.contiguous() if torch.is_tensor(v) else v) for n, v in zip(names, vals)})
        assert list(got) == [n for n, _ in c["files"]], c["name"]
        for n, d in c["files"]:
            assert got[n] == d, f"{c['name']} {n}"


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("case", range(2), ids=["d64_c3", "vgg64_c3"])
def test_generate_video_matches_reference_generation(case, prec, recorder, monkeypatch):
    """The reference generate.py on its real P2PModel: the pictures within the generation tolerance with the reference's
    eps injected in its order (per length, per eager call, per step, posterior then prior), the same files, and NumPy's
    stream left where the script leaves it."""
    from p2pvg_b200 import generate
    from tests.generate_ref import fixture_model, video_frames
    c = torch.load(FIX, weights_only=False)["generation"][case]
    tmax, _ = TOL[prec]
    draws = iter(c["eps"])
    monkeypatch.setattr(generate, "_eps", lambda B, z, dev, n, nb: torch.stack(
        [torch.stack([next(draws).reshape(B, z)[:nb] for _ in (0, 1)]) for _ in range(n)]).to(dev))
    with precision(prec):
        model = fixture_model(c)
        seq = torch.from_numpy((video_frames(c) / 255.).astype(np.float32)).permute(0, 3, 1, 2).unsqueeze(1).cuda()
        np.random.set_state(c["np_before"])
        generate.generate_video(model, seq, "OUT")
    assert next(draws, None) is None, "every reference draw is used"
    after = np.random.get_state()
    assert after[2] == c["np_after"][2] and np.array_equal(after[1], c["np_after"][1])
    assert [n for n, _ in recorder.files] == [n for n, _ in c["files"]]
    for (n, v), (_, d) in zip(recorder.files, c["files"]):
        if torch.is_tensor(v):
            assert v.numel() == d["numel"], n
            e = (v.double().reshape(-1)[d["idx"]] - d["samples"]).abs().max().item()
            assert e <= tmax, f"{c['name']} {prec} {n}: {e:.3e}"
        else:   # GIF frames: the uint8 truncation of v * 255, so an error e in v moves a value by at most 1 + 255 e
            f = torch.from_numpy(np.stack(v)).double().reshape(-1)
            assert f.numel() == d["numel"], n
            e = (f[d["idx"]] - d["samples"]).abs().max().item()
            assert e <= 1 + 255 * tmax, f"{c['name']} {prec} {n}: {e}"


def test_generate_video_equals_the_eager_loop(tmp_path, recorder):
    """generate_video against generate.py's loop restated over the eager path (tests/generate_ref.generate_ref) from the same
    NumPy and CUDA seeds: the same files, pictures within the fp32 generation tolerance, and both random streams left in the
    same state."""
    from p2pvg_b200 import generate
    from tests.generate_ref import generate_ref
    B = 1
    with precision("fp32"):
        model = config_model("dcgan_64", 3, 1, False, B)
        seq = clip(model, 12, B, seed=2)
        np.random.seed(9)
        torch.cuda.manual_seed(9)
        pics = generate.generate_video(model, seq, str(tmp_path / "out"))
        np_got, rng_got = np.random.get_state(), torch.cuda.get_rng_state()
        got = list(recorder.files)
        recorder.files.clear()
        np.random.seed(9)
        torch.cuda.manual_seed(9)
        generate_ref(model, seq, str(tmp_path / "out"), recorder.save_image, recorder.mimsave)
    ref = recorder.files
    want = [n for L in generate.GEN_LENGTHS for n in generate.file_names(str(tmp_path / "out"), L, 5)]
    assert [n for n, _ in got] == want == [n for n, _ in ref] and len(want) == 3 * 13
    np_ref = np.random.get_state()
    assert np_got[2] == np_ref[2] and np.array_equal(np_got[1], np_ref[1])
    assert torch.equal(rng_got, torch.cuda.get_rng_state())
    tmax, tmean = TOL["fp32"]
    for (n, a), (_, b) in zip(got, ref):
        if torch.is_tensor(a):
            e = (a.double() - b.double()).abs()
            assert a.shape == b.shape and e.max().item() <= tmax and e.mean().item() <= tmean, f"{n}: {e.max().item():.3e}"
        else:
            assert len(a) == len(b), n
            for fa, fb in zip(a, b):
                assert fa.shape == fb.shape and np.abs(fa.astype(np.int16) - fb.astype(np.int16)).max() <= 1, n
    assert [tuple(p[0].shape) for p in pics] == [(3, 64, max(12, L) * 64) for L in generate.GEN_LENGTHS]


def test_cli_writes_generate_py_s_files(tmp_path, monkeypatch):
    """python -m p2pvg_b200.generate on a checkpoint written by P2PModel.save and a stub imageio video: the model is built
    from states['opt'] with the checkpoint's weights, and the files are generate.py's, with the pictures generate_video
    makes from the same seed."""
    import torchvision.utils as vutils
    from p2pvg_b200 import generate
    from tests.generate_ref import video_frames
    model = config_model("vgg_64", 3, 1, False, 1)
    model.opt.backbone, model.opt.image_width, model.opt.channels = "vgg", 64, 3
    for k, v in dict(g_dim=128, z_dim=10, rnn_size=256, prior_rnn_layers=1, posterior_rnn_layers=1, predictor_rnn_layers=2).items():
        setattr(model.opt, k, v)
    ckpt = str(tmp_path / "model.pth")
    model.save(ckpt, 3)
    c = dict(video_seed=5, T=8, H=64, C=3)
    rec = Recorder()
    rec.imageio.get_reader = lambda name: iter(list(video_frames(c)))
    monkeypatch.setitem(sys.modules, "imageio", rec.imageio)
    monkeypatch.setattr(vutils, "save_image", rec.save_image)
    built = []
    real = generate.generate_video
    monkeypatch.setattr(generate, "generate_video", lambda m, seq, root, **kw: (built.append((m, seq)), real(m, seq, root, **kw))[1])
    np.random.seed(4)
    generate.main(["--ckpt", ckpt, "--video", "clip.mp4", "--output_root", str(tmp_path / "gen"), "--seed", "7"])
    m, seq = built[0]
    assert not m.training
    for name in ("encoder", "decoder", "frame_predictor", "posterior", "prior"):
        for (k, a), b in zip(getattr(m, name).state_dict().items(), getattr(model, name).state_dict().values()):
            assert torch.equal(a.cpu(), b.cpu()), f"{name}.{k}"
    assert tuple(seq.shape) == (8, 1, 3, 64, 64) and seq.is_cuda
    assert torch.equal(seq.cpu(), torch.from_numpy((video_frames(c) / 255.).astype(np.float32)).permute(0, 3, 1, 2).unsqueeze(1))
    names = [n for n, _ in rec.files]
    assert names == [n for L in generate.GEN_LENGTHS for n in generate.file_names(str(tmp_path / "gen"), L, 5)]
    # the same seed through the function API gives the same pictures
    cli = list(rec.files)
    rec.files.clear()
    np.random.seed(4)
    torch.cuda.manual_seed_all(7)
    real(m, seq, str(tmp_path / "gen"))
    for (n, a), (_, b) in zip(cli, rec.files):
        assert (torch.equal(a, b) if torch.is_tensor(a) else all(np.array_equal(x, y) for x, y in zip(a, b))), n


def test_generate_video_one_channel(tmp_path, recorder):
    """1-channel frames are repeated to 3 channels; the borders and layout as for 3 channels."""
    from p2pvg_b200 import generate
    model = config_model("dcgan_64", 1, 1, False, 1)
    seq = clip(model, 7, 1, seed=4)
    pics = generate.generate_video(model, seq, str(tmp_path), gen_lengths=(5, 9), nsamples=3, ndisplays=2)
    gt, block, gif = pics[1]
    assert gt.shape == (3, 64, 9 * 64) and block.shape == (3, 128, 9 * 64) and gif.shape == (9, 64, 128, 3)
    for c in range(3):   # interior: the input frame, replicated to 3 channels
        assert torch.equal(gt[c, 3:61, 64 + 3:128 - 3], seq[1, 0, 0, 3:61, 3:61])
    assert torch.equal(gt[:, 0, 0], torch.tensor([1.0, 165 / 255, 0.0], device=gt.device))   # orange on frame 0
    assert torch.equal(gt[:, 0, 6 * 64], torch.tensor([1.0, 0.0, 0.0], device=gt.device))    # red from frame seq_len - 1 on
    assert torch.equal(gif.float(), torch.trunc(block.view(3, 2, 64, 9, 64).permute(3, 2, 1, 4, 0).reshape(9, 64, 128, 3) * 255))


# ---- 5. rejections of the composition kernel --------------------------------------------------------------------------------
def test_vis_tiles_rejects_malformed_tables():
    from p2pvg_b200._lib import kernels_for
    dev = torch.device("cuda")
    K = kernels_for(dev)
    store = torch.rand(4, 3, 8, 8, device=dev)
    out_f, out_u8 = torch.full((3 * 8 * 16,), -1.0, device=dev), torch.zeros(3 * 8 * 16, dtype=torch.uint8, device=dev)
    tables = torch.empty(16, dtype=torch.int64, device=dev)
    images = np.array([[0, 0, 8, 16], [0, 1, 8, 16]], np.int64)
    good = np.array([[0, 1, 1, 0, 0, 0], [0, 2, 2, 1, 0, 8]], np.int32)
    K.vis_tiles(store, 4, None, 0, 3, 8, good, images, tables, out_f, out_u8)
    torch.cuda.synchronize()
    assert (out_f.view(3, 8, 16)[:, :, :8] >= 0).all()
    bad_tiles = [(0, 4, 0, 0, 0, 0), (1, 0, 0, 0, 0, 0), (0, 0, 3, 0, 0, 0), (0, 0, 0, 2, 0, 0), (0, 0, 0, 0, 1, 0),
                 (0, 0, 0, 0, 0, 9), (0, -2, 0, 0, 0, 0), (0, 0, 0, 0, -1, 0)]
    for t in bad_tiles:
        out_f.fill_(-1.0)
        with pytest.raises(RuntimeError, match="vis_tiles"):
            K.vis_tiles(store, 4, None, 0, 3, 8, np.array([t], np.int32), images, tables, out_f, out_u8)
        torch.cuda.synchronize()
        assert (out_f == -1.0).all(), t   # nothing launched
    for im in ([[0, 0, 8, 17]], [[1, 0, 8, 16]], [[0, 2, 8, 16]], [[0, 1, 9, 16]]):
        with pytest.raises(RuntimeError, match="vis_tiles"):
            K.vis_tiles(store, 4, None, 0, 3, 8, good[:1], np.array(im, np.int64), tables, out_f, out_u8)
    with pytest.raises(RuntimeError, match="vis_tiles"):
        K.vis_tiles(store, 4, None, 0, 2, 8, good, images, tables, out_f, out_u8)
