"""p2pvg_video_windows / p2pvg_b200.data.ClipBatches: Weizmann and BAIR batches cut on the device from uint8 clips.

tests/golden/video_ref.json was written by the unmodified reference loaders (make_golden_video.py) on the seeded trees of
tests/video_tree.py; the same trees are regenerated here, and the kernel fed the same entries and draws must reproduce every
sequence bit for bit."""
import ctypes
import hashlib
import json
import os
import sys
import types

import numpy as np
import pytest
import torch
from scipy import stats

from tests import video_tree

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "video_ref.json")


@pytest.fixture(scope="module")
def ref():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("video"))
    video_tree.write_weizmann_tree(root)
    video_tree.write_bair_tree(root)
    return root


def kernels():
    from p2pvg_b200._lib import kernels_for
    return kernels_for("cuda")


def sha(x):
    return hashlib.sha256(x.contiguous().cpu().numpy().tobytes()).hexdigest()


def windows(clips, entries, draws, T):
    B = len(entries)
    out = torch.full((T, B) + tuple(clips.frames.shape[1:]), float("nan"), device="cuda")
    d = None if draws is None else torch.tensor(draws, dtype=torch.int64).to(torch.int32).cuda()
    kernels().video_windows(clips.frames, clips.clip_first, clips.clip_len, torch.tensor(entries, dtype=torch.int32).cuda(), d,
                            clips.paired_flips, clips.max_seq_len, out)
    return out


def expected_window(clips, e, r, T):
    """The host copy of entry e's window: frames as stored, mirrored for an odd paired entry, / 255 in fp32."""
    k = e >> 1 if clips.paired_flips else e
    first, n = int(clips.clip_first[k]), int(clips.clip_len[k])
    start = 0 if r is None else (r % 2 ** 32) % (n - clips.max_seq_len + 1)
    x = clips.frames[first + start:first + start + T].cpu().float().div(255)
    return x.flip(-1) if clips.paired_flips and e & 1 else x


def check_hashes(clips, entries, draws, T, want, label):
    out = windows(clips, entries, draws, T)
    bad = [b for b in range(len(entries)) if sha(out[:, b]) != want[b]]
    detail = ""
    if bad:
        b = bad[0]
        diff = (out[:, b].cpu() - expected_window(clips, entries[b], None if draws is None else draws[b], T)).abs().max()
        detail = f"; row {b} max |diff| to the host window {diff.item()}"
    assert not bad, f"{label} T={T}: rows {bad} differ from the reference{detail}"


@pytest.mark.parametrize("train", [True, False], ids=["train", "test"])
def test_weizmann_sequences_bit_identical(ref, tree, train):
    from p2pvg_b200.data import load_weizmann_clips
    case = ref["weizmann_train" if train else "weizmann_test"]
    clips = load_weizmann_clips(tree, train, case["max_seq_len"], video_tree.SIZE)
    # the reference's entry i -> ours, through the clip names (its identity order is the filesystem's)
    ours = [2 * clips.names.index(c["name"]) + f for c in case["clips"] for f in (0, 1)]
    entries = [ours[i] for i in case["index"]]
    assert any(e & 1 for e in entries) and any(not e & 1 for e in entries)
    for T, key in ((case["max_seq_len"], "sha256_full"), (case["t_short"], "sha256_short")):
        check_hashes(clips, entries, case["draws"], T, case[key], f"weizmann train={train}")


def test_bair_sequences_bit_identical(ref, tree):
    from p2pvg_b200.data import load_bair_clips
    case = ref["bair_train"]
    clips = load_bair_clips(tree, True, case["max_seq_len"], video_tree.SIZE)
    entries = [clips.names.index(n) for n in case["names"]]
    for T, key in ((case["max_seq_len"], "sha256_full"), (case["t_short"], "sha256_short")):
        check_hashes(clips, entries, None, T, case[key], "bair train")
    case = ref["bair_test"]
    clips = load_bair_clips(tree, False, case["max_seq_len"], video_tree.SIZE)
    entries = [clips.names.index(n) for b in case["batches"] for n in b]
    check_hashes(clips, entries, None, case["max_seq_len"], case["sha256_full"], "bair test")


def to_u8(x):
    return (x * 255).round().to(torch.uint8)


def first_frame_ids(clips, x):
    """For each row of a batch: (entry, window start) found by matching its first frame against the store."""
    store = clips.frames
    ids = []
    for b in range(x.shape[1]):
        f = to_u8(x[0, b])
        hit = None
        for k in range(len(clips.names)):
            a, n = int(clips.clip_first[k]), int(clips.clip_len[k])
            for flip in ((0, 1) if clips.paired_flips else (0,)):
                cand = store[a:a + n].flip(-1) if flip else store[a:a + n]
                m = (cand == f).flatten(1).all(1).nonzero()
                if len(m):
                    hit = ((2 * k + flip) if clips.paired_flips else k, int(m[0]))
        ids.append(hit)
    return ids


def test_permutation_epochs_starts_and_flips(tree):
    from p2pvg_b200.data import ClipBatches, load_weizmann_clips
    clips = load_weizmann_clips(tree, True, video_tree.TRAIN_LEN, video_tree.SIZE)
    n, B = len(clips), 3
    it = ClipBatches(clips, B, "permutation", seq_len=(10, 18), generator=torch.Generator("cuda").manual_seed(4))
    np.random.seed(0)
    epochs, starts, flips = [], {k: [] for k in range(len(clips.names))}, []
    for _ in range(120):
        epoch = []
        for _ in range(n // B):
            x = next(it)
            assert x.dtype == torch.float32 and tuple(x.shape[1:]) == (B, 3, 64, 64) and 10 <= len(x) <= 18
            for e, s in first_frame_ids(clips, x):
                epoch.append(e)
                starts[e >> 1].append(s)
                flips.append(e & 1)
        epochs.append(epoch)
    for epoch in epochs:
        assert len(set(epoch)) == len(epoch) == n // B * B   # drop_last: a permutation's first n // B * B entries
    for k, s in starts.items():
        span = int(clips.clip_len[k]) - video_tree.TRAIN_LEN + 1
        assert min(s) >= 0 and max(s) < span
        if span > 1:
            assert stats.chisquare(np.bincount(s, minlength=span)).pvalue > 1e-3, clips.names[k]
    assert stats.chisquare(np.bincount(flips, minlength=2)).pvalue > 1e-3
    with pytest.raises(ValueError):
        ClipBatches(clips, n + 1, "permutation", seq_len=(10, 18))


def test_uniform_and_ordered_bair_sampling(tree):
    from p2pvg_b200.data import ClipBatches, load_bair_clips
    clips = load_bair_clips(tree, True, video_tree.BAIR_LEN, video_tree.SIZE)
    it = ClipBatches(clips, 64, "uniform", seq_len=(20, 30), generator=torch.Generator("cuda").manual_seed(1))
    got = [e for _ in range(4) for e, s in first_frame_ids(clips, next(it))]
    assert all(s == 0 for _, s in first_frame_ids(clips, next(it)))
    assert set(got) == set(range(len(clips.names)))
    assert stats.chisquare(np.bincount(got, minlength=len(clips.names))).pvalue > 1e-3

    test = load_bair_clips(tree, False, video_tree.BAIR_LEN, video_tree.SIZE)
    B = 3000   # 10000 // 3000 = 3 batches per epoch
    it = ClipBatches(test, B, "ordered", seq_len=(1, 1))
    n = len(test.names)
    for i in range(7):
        x = next(it)
        k = i % 3
        want = torch.tensor([(k * B + j) % n for j in range(B)])
        firsts = test.frames[test.clip_first.long()]       # frame 0 of every trajectory
        match = (to_u8(x[0]).unsqueeze(1) == firsts.unsqueeze(0)).flatten(2).all(2).float().argmax(1).cpu()
        assert torch.equal(match, want), i


def test_sequence_lengths_follow_numpy_and_seeds_repeat(tree):
    from p2pvg_b200.data import ClipBatches, load_weizmann_clips
    clips = load_weizmann_clips(tree, False, video_tree.TEST_LEN, video_tree.SIZE)
    runs = []
    for _ in range(2):
        np.random.seed(11)
        it = ClipBatches(clips, 2, "permutation", seq_len=(6, 10), generator=torch.Generator("cuda").manual_seed(3))
        runs.append([next(it) for _ in range(20)])
    np.random.seed(11)
    want = [np.random.randint(6, 11) for _ in range(20)]
    assert [len(x) for x in runs[0]] == want and len(set(want)) > 2
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    assert any(not torch.equal(a[:6], b[:6]) for a, b in zip(runs[0], runs[0][1:]))


def vgg_model(B):
    from p2pvg_b200.models import vgg_64
    from p2pvg_b200.models.p2p_model import P2PModel
    opt = types.SimpleNamespace(dataset="weizmann", backbone_net=vgg_64, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0,
                                weight_align=0.5, skip_prob=0.0, n_past=1, last_frame_skip=False, batch_size=B)
    torch.manual_seed(1)
    return P2PModel(B, 3, 128, 10, 256, 1, 1, 2, opt=opt).cuda()


def test_vgg64_steps_from_clip_batches_equal_host_frames(tree, monkeypatch):
    from p2pvg_b200.data import ClipBatches, load_weizmann_clips
    monkeypatch.setenv("P2PVG_GRAPH", "0")
    monkeypatch.setenv("P2PVG_PRECISION", "bf16")
    B = 8
    clips = load_weizmann_clips(tree, True, video_tree.TRAIN_LEN, video_tree.SIZE)
    runs, frames = [], []
    for fed in ("device", "host"):
        model = vgg_model(B)
        model.train()
        it = ClipBatches(clips, B, "permutation", seq_len=(10, 18), generator=torch.Generator("cuda").manual_seed(2))
        np.random.seed(0)
        losses = []
        for i in range(2):
            if fed == "device":
                x = next(it)
                frames.append(x.cpu())
            else:
                np.random.randint(10, 19)   # the draw ClipBatches makes, so that forward sees the same NumPy stream
                x = frames[i].pin_memory().cuda(non_blocking=True)
            torch.manual_seed(100 + i)
            losses.append(np.array(model(x, 0, len(x) - 1), dtype=np.float64))
        runs.append(losses)
        del model
        torch.cuda.empty_cache()
    for a, b in zip(*runs):
        assert np.all(np.isfinite(a))
        np.testing.assert_allclose(a, b, rtol=1e-5, atol=0)


@pytest.mark.parametrize("dataset", ["weizmann", "bair"])
def test_dropin_generators(tree, monkeypatch, dataset):
    monkeypatch.setenv("P2PVG_REF", "")
    monkeypatch.syspath_prepend(os.path.join(ROOT, "dropin"))
    for m in ("data", "data.data_utils"):
        monkeypatch.delitem(sys.modules, m, raising=False)
    import data.data_utils as du
    try:
        opt = types.SimpleNamespace(dataset=dataset, data_root=tree, max_seq_len=30, delta_len=5, image_width=64, channels=3,
                                    batch_size=3)
        train, test = du.load_dataset(opt)
        if dataset == "weizmann":
            assert len(train) == 8 and len(test) == 6 and (train.max_seq_len, test.max_seq_len) == (18, 10)
            bounds = ((10, 18), (6, 10))
        else:
            assert len(train) == len(test) == 10000 and train.max_seq_len == 30
            bounds = ((20, 30), (20, 30))
        for ds, is_train, (lo, hi) in ((train, True, bounds[0]), (test, False, bounds[1])):
            gen = du.get_data_generator(ds, train=is_train, opt=opt)
            for _ in range(4):
                x = next(gen)
                assert x.is_cuda and x.dtype == torch.float32 and lo <= len(x) <= hi
                assert tuple(x.shape[1:]) == (3, 3, 64, 64) and 0 <= float(x.min()) and float(x.max()) <= 1
        with pytest.raises(AssertionError):
            du.load_dataset(types.SimpleNamespace(**dict(vars(opt), channels=1)))
    finally:
        for m in ("data", "data.data_utils"):
            sys.modules.pop(m, None)


def test_kernel_rejects_bad_arguments():
    from p2pvg_b200._lib import load_library
    lib = load_library()
    B, L, T, C, H, W = 2, 4, 3, 3, 16, 32
    frames = torch.zeros(8, C, H, W, dtype=torch.uint8, device="cuda")
    first = torch.tensor([0, 4], dtype=torch.int64, device="cuda")
    lens = torch.tensor([4, 4], dtype=torch.int32, device="cuda")
    entries = torch.tensor([0, 3], dtype=torch.int32, device="cuda")
    draws = torch.zeros(B, dtype=torch.int32, device="cuda")
    out = torch.empty(T, B, C, H, W, device="cuda")
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = ctypes.c_void_p

    def call(fr=frames.data_ptr(), cf=first.data_ptr(), cl=lens.data_ptr(), n_clips=2, en=entries.data_ptr(),
             dr=draws.data_ptr(), B=B, L=L, T=T, C=C, H=H, W=W, o=out.data_ptr()):
        return lib.p2pvg_video_windows(P(fr), P(cf), P(cl), n_clips, P(en), P(dr), 1, B, L, T, C, H, W, P(o), stream)

    assert call() == 0
    assert call(dr=None) == 0
    torch.cuda.synchronize()
    for kw in (dict(fr=None), dict(cf=None), dict(cl=None), dict(en=None), dict(o=None), dict(fr=frames.data_ptr() + 2),
               dict(o=out.data_ptr() + 8), dict(T=L + 1), dict(T=-1), dict(B=-1), dict(L=0), dict(C=0), dict(H=0), dict(W=18),
               dict(W=2), dict(W=0), dict(n_clips=0)):
        assert call(**kw) == -1, kw


def test_every_level_converts_like_totensor_and_mirrors():
    """All 256 uint8 levels, plain and mirrored, against torch's CPU u / 255 (what ToTensor computes)."""
    from p2pvg_b200.data import VideoClips
    lv = torch.arange(256, dtype=torch.uint8).reshape(1, 1, 4, 64).repeat(2, 3, 1, 1)
    lv[1] = lv[1].flip(0)
    clips = VideoClips(lv.cuda(), torch.tensor([0], device="cuda"), torch.tensor([2], dtype=torch.int32, device="cuda"), ["lv"],
                       True, 2)
    out = windows(clips, [0, 1], [0, 1], 2)
    want = lv.float().div(255)
    assert torch.equal(out[:, 0].cpu(), want) and torch.equal(out[:, 1].cpu(), want.flip(-1))
