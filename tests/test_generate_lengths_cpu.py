"""generate_lengths' row planner and checks (p2pvg_b200/gen_engine.py) and generate_video's tile table
(p2pvg_b200/generate.py), without a GPU: the tiles, gathered with NumPy, give the reference generate.py's pictures bit for
bit (tests/golden/generate_ref.pt)."""
import hashlib
import os
import types

import numpy as np
import pytest
import torch

from p2pvg_b200 import gen_engine, generate
from tests.generate_ref import stub_samples

FIX = os.path.join(os.path.dirname(__file__), "golden", "generate_ref.pt")


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def test_plan_lengths_groups_rows_and_counters():
    lens, T, n_past, gr = [4, 9, 2, 9, 6], 6, 2, 6
    rs = np.random.RandomState(0)
    probs = [rs.uniform(0, 1, L - 1) for L in lens]
    order, active, fl = gen_engine.plan_lengths(lens, T, probs, 0.5, n_past, gr)
    assert order == [1, 3, 4, 0, 2]                  # longest first, ties in caller order
    assert active == [gr * n for n in (5, 4, 4, 3, 3, 2, 2, 2)]
    nG, S = len(lens), max(lens) - 1
    assert len(fl) == 2 * S * nG
    tab = torch.tensor(fl, dtype=torch.float64).float().view(2, S, nG)
    for g, k in enumerate(order):
        sl = gen_engine.plan_slots(lens[k], T, probs[k], 0.5, n_past, False, lens[k] - 1)
        assert len(sl) == lens[k] - 1
        for s in range(S):
            want = (sl[s][1], sl[s][2]) if s < len(sl) else (0.0, 0.0)
            assert tab[0, s, g].item() == np.float32(want[0]) and tab[1, s, g].item() == np.float32(want[1]), (g, s)


def test_single_length_plan_is_the_plain_call():
    probs = [np.random.RandomState(1).uniform(0, 1, 7)]
    order, active, fl = gen_engine.plan_lengths([8], 5, probs, 0.3, 1, 4)
    _, _, ref = gen_engine.plan_segments([(0, 5, 8, 7)], 5, probs, 0.3, 1, False, "full")
    assert order == [0] and active == [4] * 7 and fl == ref


@pytest.mark.parametrize("bad", [[], None, [1, 5], [5, "a"], [2.5], [True, 4], 7])
def test_check_lengths_rejects(bad):
    with pytest.raises(ValueError):
        gen_engine.check_lengths(bad, 10, 1)


def test_check_lengths_needs_the_teacher_forced_frames():
    assert gen_engine.check_lengths([3, 2], 3, 3) == [3, 2]
    assert gen_engine.check_lengths([2], 2, 3) == [2]
    with pytest.raises(ValueError):
        gen_engine.check_lengths([4], 2, 3)


def test_rejections_before_any_draw():
    """A model the graphed engine does not take, or malformed lengths, raise before NumPy or torch draws anything."""
    from p2pvg_b200.models import dcgan_64
    from p2pvg_b200.models.p2p_model import P2PModel
    opt = types.SimpleNamespace(dataset="mnist", backbone_net=dcgan_64, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0,
                                weight_align=0.5, skip_prob=0.5, n_past=1, last_frame_skip=False, batch_size=1)
    model = P2PModel(1, 1, 128, 10, 256, 1, 1, 2, opt=opt).eval()
    x = torch.rand(5, 1, 1, 64, 64)
    for lens in ([], [1], ["x"]):
        st, rng = np.random.get_state(), torch.get_rng_state()
        with pytest.raises(ValueError):
            model.p2p_generate_lengths(x, lens)
        assert np.array_equal(np.random.get_state()[1], st[1]) and np.random.get_state()[2] == st[2]
        assert torch.equal(torch.get_rng_state(), rng)
    with pytest.raises(ValueError):
        generate.check_generate(model, x.unsqueeze(1)[:, :, 0], (10,), 5, 5)   # not on a CUDA device
    with pytest.raises(ValueError):
        generate.generate_video(model, x, "OUT", nsamples=2, ndisplays=3)


def gather(store0, store1, plan, C, H):
    """The kernel's gather, restated with NumPy: the pictures of every length."""
    images, tiles, layout, n_f, n_u8 = plan
    out_f, out_u8 = np.zeros(n_f, np.float32), np.zeros(n_u8, np.uint8)
    bc = {1: np.array([1.0, 165.0 / 255.0, 0.0], np.float32), 2: np.array([1.0, 0.0, 0.0], np.float32)}
    edge = np.ones((H, H), bool)
    edge[3:H - 3, 3:H - 3] = False
    for st, f, border, img, y, x in tiles:
        src = (store0, store1)[st]
        v = np.zeros((3, H, H), np.float32) if f < 0 else np.repeat(src[f], 3 // C, 0)
        if border:
            v = np.where(edge[None], bc[border][:, None, None], v)
        off, kind, h, w = images[img]
        if kind == 0:
            out_f[off:off + 3 * h * w].reshape(3, h, w)[:, y:y + H, x:x + H] = v
        else:
            out_u8[off:off + 3 * h * w].reshape(h, w, 3)[y:y + H, x:x + H] = (v * np.float32(255)).astype(np.uint8).transpose(1, 2, 0)
    return [tuple((out_f if len(shape) == 3 else out_u8)[o:o + int(np.prod(shape))].reshape(shape) for o, shape in lay)
            for lay in layout]


@pytest.mark.parametrize("case", range(2))
def test_tile_table_gives_the_reference_pictures(case):
    c = torch.load(FIX, weights_only=False)["composition"][case]
    seq, samples = stub_samples(c)
    lens, ns, C, H = c["lens"], c["nsamples"], c["C"], c["H"]
    store1 = np.concatenate([samples[L].reshape(-1, C, H, H).numpy() for L in lens])
    base = np.cumsum([0] + [ns * L for L in lens])
    plan = generate.plan_video(len(seq), lens, c["idxs"], H, lambda t: (0, t), lambda k, s, t: (1, int(base[k]) + s * lens[k] + t))
    got = {}
    for L, idx, (gt, block, gif) in zip(lens, c["idxs"], gather(seq.reshape(-1, C, H, H).numpy(), store1, plan, C, H)):
        names = generate.file_names("OUT", L, len(idx))
        vals = [sha(gt)] + [sha(block[:, ix * H:(ix + 1) * H]) for ix in range(len(idx))] + [sha(block)] + \
            [[sha(f[:, ix * H:(ix + 1) * H]) for f in gif] for ix in range(len(idx))] + [[sha(f) for f in gif]]
        got.update(zip(names, vals))
    assert list(got) == [n for n, _ in c["files"]]
    for n, d in c["files"]:
        assert got[n] == d, n


def test_file_names_are_generate_py_s():
    names = generate.file_names("out", 10, 2)
    assert names == ["out/len_10-gt.png", "out/len_10-gen_000.png", "out/len_10-gen_001.png", "out/len_10-gen_full.png",
                     "out/len_10-gen_000.gif", "out/len_10-gen_001.gif", "out/len_10-gen_full.gif"]


def test_backbone_of_rejects_h36m():
    with pytest.raises(ValueError, match="h36m"):
        generate.backbone_of(types.SimpleNamespace(dataset="h36m", backbone="mlp", image_width=64))
    assert generate.backbone_of(types.SimpleNamespace(dataset="mnist", backbone="vgg", image_width=128)).__name__.endswith("vgg_128")


@pytest.mark.parametrize("case", range(2))
def test_torch_restatement_gives_the_reference_pictures(case):
    """tests/generate_ref.generate_ref (the benchmark's eager baseline) writes generate.py's files bit for bit on the
    composition cases' stub samples."""
    from tests.generate_ref import generate_ref, stub_frames
    c = torch.load(FIX, weights_only=False)["composition"][case]
    seq, _ = stub_samples(c)
    calls = {}

    class Stub:
        def p2p_generate(self, x, L, cp, model_mode="full"):
            np.random.uniform(0, 1, L - 1)
            s = calls[L] = calls.get(L, -1) + 1
            return list(stub_frames(c, L, s))

    files = []
    np.random.set_state(c["np_before"])
    generate_ref(Stub(), seq, "OUT", lambda t, name: files.append((name, sha(t.numpy()))),
                 lambda name, frames: files.append((name, [sha(f) for f in frames])))
    assert files == c["files"]
    after = np.random.get_state()
    assert after[2] == c["np_after"][2] and np.array_equal(after[1], c["np_after"][1])


def test_read_video_as_generate_py(monkeypatch):
    import sys
    frames = [np.random.RandomState(k).randint(0, 256, size=(8, 8, 3)).astype(np.uint8) for k in range(4)]
    monkeypatch.setitem(sys.modules, "imageio", types.SimpleNamespace(get_reader=lambda name: iter(frames)))
    v = generate.read_video("clip.mp4")
    assert v.shape == (4, 1, 3, 8, 8) and v.dtype == torch.float32
    assert torch.equal(v[2, 0], torch.from_numpy((frames[2] / 255.).astype(np.float32)).permute(2, 0, 1))
    monkeypatch.setitem(sys.modules, "imageio", None)   # not installed
    with pytest.raises(RuntimeError, match="imageio"):
        generate.read_video("clip.mp4")


def test_cli_rejects_h36m_checkpoints_before_building_a_model():
    ckpt = os.path.join(os.path.dirname(__file__), "golden", "ckpt_ref_small.pth")   # a reference-written h36m checkpoint
    with pytest.raises(ValueError, match="h36m"):
        generate.main(["--ckpt", ckpt, "--video", "clip.mp4"])
    with pytest.raises(SystemExit):
        generate.main(["--ckpt", ckpt])   # generate.py's --video is needed (its image branch is not provided)
