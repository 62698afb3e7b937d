"""Weizmann and BAIR clip loaders, host side (no GPU): split, filtering, name order and flip pairing against the entry map the
unmodified reference loaders produced (tests/golden/video_ref.json, make_golden_video.py), frame decoding, rejection of bad
frames, and the ``ordered`` sampling schedule."""
import json
import os

import numpy as np
import pytest
import torch
from PIL import Image

from p2pvg_b200.data import ClipBatches, load_bair_clips, load_weizmann_clips, ordered_schedule
from tests import video_tree

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "video_ref.json")


@pytest.fixture(scope="module")
def ref():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    root = tmp_path_factory.mktemp("video")
    return str(root), video_tree.write_weizmann_tree(str(root)), video_tree.write_bair_tree(str(root))


def chw(a):
    return np.broadcast_to(a, (3,) + a.shape) if a.ndim == 2 else a.transpose(2, 0, 1)


@pytest.mark.parametrize("train", [True, False])
def test_weizmann_clips_split_filter_and_order(ref, tree, train):
    root, arrays, _ = tree
    case = ref["weizmann_train" if train else "weizmann_test"]
    clips = load_weizmann_clips(root, train, case["max_seq_len"], video_tree.SIZE, device="cpu")
    # the same clips as the reference kept (its identity order is the filesystem's; ours is sorted)
    assert clips.names == sorted(c["name"] for c in case["clips"])
    assert len(clips) == 2 * len(case["clips"]) and clips.paired_flips
    assert clips.frames.dtype == torch.uint8 and tuple(clips.frames.shape[1:]) == (3, 64, 64)
    by_name = {c["name"]: c["files"] for c in case["clips"]}
    for k, name in enumerate(clips.names):
        files = by_name[name]
        first, n = int(clips.clip_first[k]), int(clips.clip_len[k])
        assert n == len(files) >= case["max_seq_len"]
        # frame files in the reference's lexicographic order, each decoded to the seeded pixels
        for j, f in enumerate(files):
            want = arrays[name][video_tree.frame_number(f)]
            assert np.array_equal(clips.frames[first + j].numpy(), chw(want)), (name, f)
        assert clips.entry(2 * k) == (name, False) and clips.entry(2 * k + 1) == (name, True)
    # lexicographic, not numeric, frame order, and the exact-length and too-short clips
    if train:
        assert by_name["ido/walk"][:3] == ["0.png", "1.png", "10.png"]
        assert len(by_name["ido/run"]) == 18
    assert "daria/jump" not in by_name and "moshe/skip" not in by_name and ("ido/run" in by_name) == train


@pytest.mark.parametrize("train", [True, False])
def test_bair_clips_follow_sorted_trajectories(ref, tree, train):
    root, _, arrays = tree
    split = "train" if train else "test"
    clips = load_bair_clips(root, train, video_tree.BAIR_LEN, video_tree.SIZE, device="cpu")
    want = sorted(n.split("/", 1)[1] for n in arrays if n.startswith(split + "/"))
    assert clips.names == sorted(want, key=lambda d: d.split("/"))
    assert len(clips) == len(want) and not clips.paired_flips
    names = ref["bair_train"]["names"] if train else [n for b in ref["bair_test"]["batches"] for n in b]
    assert set(names) <= set(clips.names)
    for k, name in enumerate(clips.names):
        assert clips.entry(k) == (name, False)
        first = int(clips.clip_first[k])
        for j in (0, video_tree.BAIR_LEN - 1):
            assert np.array_equal(clips.frames[first + j].numpy(), chw(arrays[f"{split}/{name}"][j]))


def test_ordered_schedule_matches_the_reference_walk(ref, tree):
    root = tree[0]
    case = ref["bair_test"]
    clips = load_bair_clips(root, False, video_tree.BAIR_LEN, video_tree.SIZE, device="cpu")
    B = case["batch_size"]
    sched = ordered_schedule(len(clips), B, epoch_items=case["epoch_items"])
    per_epoch = case["epoch_items"] // B
    assert len(sched) == per_epoch * B
    # the reference walks its own (filesystem-ordered) listing; its first pass reveals that order
    listing = list(dict.fromkeys(n for b in case["batches"] for n in b))
    assert sorted(listing) == sorted(clips.names)
    for i, batch in enumerate(case["batches"]):
        k = i % per_epoch
        assert [listing[int(e)] for e in sched[k * B:(k + 1) * B]] == batch, i
    # the restart is visible: without it the second epoch would continue the walk
    assert case["batches"][per_epoch] != [listing[(per_epoch * B + j) % len(clips)] for j in range(B)]
    assert len(ordered_schedule(5, 256)) == (10000 // 256) * 256


def write_clip(root, frames, mode):
    d = os.path.join(root, "weizmann", "a", "walk")
    os.makedirs(d, exist_ok=True)
    for i, a in enumerate(frames):
        Image.fromarray(a, mode).save(os.path.join(d, f"{i:02d}.png"))
    return d


@pytest.mark.parametrize("mode,shape", [("RGBA", (64, 64, 4)), ("RGB", (64, 48, 3)), ("RGB", (32, 32, 3))])
def test_bad_frames_raise_naming_the_file(tmp_path, mode, shape):
    frames = [np.zeros(shape, np.uint8)] * 20
    d = write_clip(str(tmp_path), frames, mode)
    with pytest.raises(ValueError, match=os.path.join(d, "00.png")):
        load_weizmann_clips(str(tmp_path), True, 10, 64, device="cpu")


def test_grayscale_frames_are_replicated(tmp_path):
    rs = np.random.RandomState(0)
    frames = [rs.randint(0, 256, (64, 64)).astype(np.uint8) for _ in range(15)]
    write_clip(str(tmp_path), frames, "L")
    clips = load_weizmann_clips(str(tmp_path), True, 10, 64, device="cpu")
    assert clips.names == ["a/walk"] and int(clips.clip_len[0]) == 10
    for j in range(10):
        assert np.array_equal(clips.frames[j].numpy(), np.stack([frames[j]] * 3))


def test_no_clip_long_enough_raises(tmp_path):
    write_clip(str(tmp_path), [np.zeros((64, 64, 3), np.uint8)] * 12, "RGB")
    with pytest.raises(ValueError, match="max_seq_len"):
        load_weizmann_clips(str(tmp_path), True, 10, 64, device="cpu")


def test_batch_larger_than_the_dataset_raises(ref, tree):
    clips = load_weizmann_clips(tree[0], False, video_tree.TEST_LEN, video_tree.SIZE, device="cpu")
    with pytest.raises(ValueError, match="exceeds"):
        ClipBatches(clips, len(clips) + 1, "permutation", seq_len=(6, 10))
    with pytest.raises(ValueError, match="seq_len"):
        ClipBatches(clips, 2, "permutation", seq_len=(6, 11))
    with pytest.raises(ValueError, match="sampling"):
        ClipBatches(clips, 2, "shuffle", seq_len=(6, 10))
