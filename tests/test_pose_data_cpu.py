"""Human3.6M pose windows, host side (no GPU): the draw -> frame mapping of p2pvg_pose_windows restated in NumPy against the
hashes the unmodified reference ``Human36mDataset`` produced (tests/golden/pose_data_ref.pt, make_golden_pose_data.py), the
``PoseClips`` store, every ValueError of ``PoseClips`` / ``PoseBatches``, and the drop-in ``h36m`` branches."""
import hashlib
import importlib
import os
import sys
import types

import numpy as np
import pytest
import torch

from p2pvg_b200.data import PoseBatches, PoseClips
from tests import pose_tree

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "pose_data_ref.pt")


@pytest.fixture(scope="module")
def fix():
    return torch.load(GOLDEN, weights_only=False)


def lists(fix, case):
    split = fix["train" if case.startswith("train") else "test"]
    return [a.numpy() for a in split["pose_2d"]], [a.numpy() for a in split["pose_3d"]], split["camera_view"]


def sha(x):
    return hashlib.sha256(np.ascontiguousarray(x.astype(np.float32)).tobytes()).hexdigest()


@pytest.mark.parametrize("case", ["train", "test", "train_speeds"])
def test_numpy_mapping_reproduces_the_reference_windows(fix, case):
    L, t_short = fix["max_seq_len"], fix["t_short"]
    lo, hi = fix[case]["speed_range"]
    rec = fix[case]["records"]
    p2, p3, _ = lists(fix, case)
    draws = pose_tree.r_values(rec, (lo, hi), np.random.RandomState(0)).view(np.uint32).astype(np.int64)
    assert (draws[0] >= 2 ** 31).any() and (draws[0] < 2 ** 31).any()      # r taken as unsigned is exercised
    for k, e in enumerate(rec["index"]):
        n = len(p3[e])
        assert rec["start_high"][k] == n - hi * L + 1
        start = draws[0, k] % (n - hi * L + 1)
        speed = lo + draws[1, k] % (hi - lo + 1)
        frames = start + np.arange(L) * speed
        for pose, key in ((p2, "sha_2d"), (p3, "sha_3d")):
            assert sha(pose[e][frames]) == rec[key][k], (case, k)
            assert sha(pose[e][frames[:t_short]]) == rec[key + "_short"][k], (case, k)
    # the fixture covers the 180-frame entry (one start at speed 6) and both ends of every entry's start range
    highs = {(e, h) for e, h in zip(rec["index"], rec["start_high"])}
    if case == "train":
        assert (0, 1) in highs
    assert {(e, 0) for e in set(rec["index"])} <= set(zip(rec["index"], rec["start"]))
    assert {(e, h - 1) for e, h in highs} <= set(zip(rec["index"], rec["start"]))
    assert len(set(rec["speed"])) == hi - lo + 1


@pytest.mark.parametrize("split", ["train", "test"])
def test_pose_clips_store(fix, split):
    p2, p3, cv = lists(fix, split)
    L, speed_hi = fix["max_seq_len"], fix[split]["speed_range"][1]
    clips = PoseClips(p2, p3, cv, L, speed_hi, device="cpu")
    assert len(clips) == fix[split]["len"] == len(p2) and clips.lengths == [len(a) for a in p2]
    assert clips.pose_2d.dtype == clips.pose_3d.dtype == torch.float32
    assert torch.equal(clips.pose_2d, torch.cat([torch.from_numpy(a).float() for a in p2]))
    assert torch.equal(clips.pose_3d, torch.cat([torch.from_numpy(a).float() for a in p3]))
    assert clips.seq_first.dtype == torch.int64 and clips.seq_len.dtype == torch.int32
    assert clips.seq_first.tolist() == np.concatenate([[0], np.cumsum(clips.lengths)[:-1]]).tolist()
    assert clips.seq_len.tolist() == clips.lengths
    # the unfiltered camera-view list, as the dataset holds it: longer than the entries
    assert clips.camera_view.dtype == torch.int64 and clips.camera_view.tolist() == cv and len(cv) > len(clips)
    moved = clips.to("cpu")
    assert moved.lengths == clips.lengths and moved.max_seq_len == L and torch.equal(moved.pose_3d, clips.pose_3d)


def synthetic(lengths, J=17):
    rs = np.random.RandomState(0)
    return [rs.randn(n, J, 2) for n in lengths], [rs.randn(n, J, 3) for n in lengths], [0, 1, 2, 3] * len(lengths)


def test_pose_clips_reject_bad_entries():
    p2, p3, cv = synthetic([70, 35, 80])
    with pytest.raises(ValueError, match="entry 1: 35 frames, fewer than speed_hi \\* max_seq_len = 60"):
        PoseClips(p2, p3, cv, 30, speed_hi=2, device="cpu")
    PoseClips(p2, p3, cv, 30, speed_hi=1, device="cpu")
    bad = list(p3)
    bad[2] = bad[2][:-1]
    with pytest.raises(ValueError, match="entry 2: 80 2d frames but 79 3d frames"):
        PoseClips(p2, bad, cv, 30, device="cpu")
    for k, a in ((0, np.zeros((70, 17, 3))), (1, np.zeros((35, 16, 2))), (2, np.zeros((80, 34)))):
        bad = list(p2)
        bad[k] = a
        with pytest.raises(ValueError, match=f"entry {k}: pose arrays"):
            PoseClips(bad, p3, cv, 30, device="cpu")
    bad = list(p3)
    bad[1] = np.zeros((35, 17, 2))
    with pytest.raises(ValueError, match="entry 1: pose arrays"):
        PoseClips(p2, bad, cv, 30, device="cpu")
    with pytest.raises(ValueError, match="3 2d entries but 2 3d entries"):
        PoseClips(p2, p3[:2], cv, 30, device="cpu")
    with pytest.raises(ValueError, match="no pose entries"):
        PoseClips([], [], [], 30, device="cpu")
    with pytest.raises(ValueError, match="2 camera views for 3 entries"):
        PoseClips(p2, p3, [0, 1], 30, device="cpu")


def test_pose_batches_reject_bad_arguments():
    clips = PoseClips(*synthetic([180, 200, 190]), 30, speed_hi=6, device="cpu")
    with pytest.raises(ValueError, match="exceeds the 3 items"):
        PoseBatches(clips, 4, (20, 30), (6, 6))
    with pytest.raises(ValueError, match="batch_size = 0"):
        PoseBatches(clips, 0, (20, 30), (6, 6))
    for bounds in ((0, 30), (20, 31), (25, 20)):
        with pytest.raises(ValueError, match="seq_len"):
            PoseBatches(clips, 2, bounds, (6, 6))
    for speeds in ((0, 6), (6, 5), (0, 0)):
        with pytest.raises(ValueError, match="speed_range"):
            PoseBatches(clips, 2, (20, 30), speeds)
    with pytest.raises(ValueError, match="entry 0: 180 frames"):
        PoseBatches(clips, 2, (20, 30), (6, 7))


@pytest.fixture
def dropin(monkeypatch):
    """The drop-in ``data.data_utils``, imported fresh with ``PoseClips`` kept on the host; yields (module, reference path or
    None)."""
    ref = os.environ.get("P2PVG_REF", "")
    ref = ref if os.path.isfile(os.path.join(ref, "data", "human36m", "human36m.py")) else None
    monkeypatch.setenv("P2PVG_REF", ref or "")
    monkeypatch.syspath_prepend(os.path.join(ROOT, "dropin"))
    if ref:
        for name, mod in pose_tree.stub_modules().items():
            monkeypatch.setitem(sys.modules, name, mod)
        monkeypatch.syspath_prepend(os.path.join(ref, "data", "human36m"))   # where train.py's working directory puts it
    fresh = ("data", "data.data_utils", "data._reference_data_utils", "human36m", "skeleton")
    for m in fresh:
        monkeypatch.delitem(sys.modules, m, raising=False)
    try:
        du = importlib.import_module("data.data_utils")
        monkeypatch.setattr(du, "PoseClips", lambda *a, device=None, **k: PoseClips(*a, device="cpu", **k))
        yield du, ref
    finally:
        for m in fresh:
            sys.modules.pop(m, None)


def test_dropin_pose_set_without_the_reference(fix, dropin):
    du, _ = dropin
    ds = pose_tree.fixture_dataset(fix, "train")
    pose = du.PoseSet(ds)
    assert len(pose) == fix["train"]["len"] and pose.skeleton is ds.skeleton and pose.speed_range == [6, 6]
    np.random.seed(3)
    got = [pose.get_seq_len() for _ in range(200)]
    assert min(got) == 20 and max(got) == 30
    with pytest.raises(NotImplementedError, match="n_breakpoints"):
        du.PoseSet(pose_tree.fixture_dataset(fix, "train", n_breakpoints=2))
    with pytest.raises(NotImplementedError):
        du.get_data_generator(pose, train=True, dynamic_length=False, opt=types.SimpleNamespace(dataset="h36m", batch_size=2))


def test_dropin_load_dataset_matches_the_reference(fix, dropin, tmp_path):
    du, ref = dropin
    if ref is None:
        pytest.skip("P2PVG_REF does not name a reference checkout")
    root = pose_tree.write_tree(str(tmp_path))
    opt = types.SimpleNamespace(dataset="h36m", data_root=root, delta_len=pose_tree.DELTA_LEN, batch_size=2)
    train, test = du.load_dataset(opt)
    assert isinstance(train, du.PoseSet) and isinstance(test, du.PoseSet)
    assert opt.data_root == os.path.join(root, pose_tree.SUBDIR)       # the reference's own load_dataset ran
    h36m = importlib.import_module("human36m")
    for ours, split, speeds in ((train, "train", [6, 6]), (test, "test", [1, 1])):
        theirs = h36m.Human36mDataset(data_root=opt.data_root, max_seq_len=30, delta_len=opt.delta_len, speed_range=speeds,
                                      n_breakpoints=0, acc_range=[0, 0], mode=split)
        assert len(ours) == len(theirs) == fix[split]["len"]
        assert ours.clips.camera_view.tolist() == list(theirs.data["camera_view"]) == fix[split]["camera_view"]
        assert np.array_equal(ours.skeleton.parents(), theirs.skeleton.parents())
        assert list(ours.skeleton.parents()) == fix[split]["parents"]
        assert (ours.max_seq_len, ours.delta_len, ours.speed_range) == (theirs.max_seq_len, theirs.delta_len, speeds)
        for seed in (0, 1):
            np.random.seed(seed)
            a = [ours.get_seq_len() for _ in range(100)]
            np.random.seed(seed)
            assert a == [theirs.get_seq_len() for _ in range(100)] and min(a) == 20 and max(a) == 30
        assert torch.equal(ours.clips.pose_3d, torch.cat([torch.from_numpy(x).float() for x in theirs.data["pose"]["3d"]]))
        assert torch.equal(ours.clips.pose_2d, torch.cat([torch.from_numpy(x).float() for x in theirs.data["pose"]["2d"]]))
