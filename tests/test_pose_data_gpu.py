"""p2pvg_pose_windows / p2pvg_b200.data.PoseBatches: Human3.6M batches gathered on the device from resident pose stores.

tests/golden/pose_data_ref.pt was written by the unmodified reference ``Human36mDataset`` (make_golden_pose_data.py): its
normalised lists, and per ``__getitem__`` the start and speed it drew and the hashes of the fp32 windows.  The kernel, fed the
same draws as r values, must reproduce every window bit for bit."""
import ctypes
import hashlib
import os
import sys
import types

import numpy as np
import pytest
import torch

from tests import pose_tree

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "pose_data_ref.pt")


@pytest.fixture(scope="module")
def fix():
    return torch.load(GOLDEN, weights_only=False)


def clips_of(fix, split, speed_hi):
    from p2pvg_b200.data import PoseClips
    s = fix[split]
    return PoseClips([a.numpy() for a in s["pose_2d"]], [a.numpy() for a in s["pose_3d"]], s["camera_view"], fix["max_seq_len"],
                     speed_hi)


def sha(x):
    return hashlib.sha256(x.contiguous().cpu().numpy().tobytes()).hexdigest()


@pytest.mark.parametrize("case", ["train", "test", "train_speeds"])
def test_windows_bit_identical_to_the_reference(fix, case):
    from p2pvg_b200._lib import kernels_for
    speeds = tuple(fix[case]["speed_range"])
    rec = fix[case]["records"]
    clips = clips_of(fix, "test" if case == "test" else "train", speeds[1])
    entries = torch.tensor(rec["index"], dtype=torch.int32, device="cuda")
    draws = torch.from_numpy(pose_tree.r_values(rec, speeds, np.random.RandomState(1))).cuda()
    B, J = len(entries), clips.pose_2d.shape[1]
    for T, suffix in ((fix["max_seq_len"], ""), (fix["t_short"], "_short")):
        out_2d = torch.full((T, B, J, 2), float("nan"), device="cuda")
        out_3d = torch.full((T, B, J, 3), float("nan"), device="cuda")
        kernels_for("cuda").pose_windows(clips.pose_2d, clips.pose_3d, clips.seq_first, clips.seq_len, entries, draws, speeds,
                                         fix["max_seq_len"], out_2d, out_3d)
        for out, key in ((out_2d, "sha_2d"), (out_3d, "sha_3d")):
            bad = [b for b in range(B) if sha(out[:, b]) != rec[key + suffix][b]]
            assert not bad, f"{case} {key} T={T}: rows {bad} (entries {[rec['index'][b] for b in bad]}) differ from the reference"


def row_windows(clips, x2, x3):
    """For each row of a batch: (entry, start, speed), found by matching its frames against the store; and a check that
    the row is exactly that window of both stores."""
    first, lengths = clips.seq_first.tolist(), clips.lengths
    ids = []
    for b in range(x3.shape[1]):
        hits = (clips.pose_3d == x3[0, b]).flatten(1).all(1).nonzero().flatten().tolist()
        assert len(hits) == 1, b
        f0 = hits[0]
        e = max(k for k in range(len(first)) if first[k] <= f0)
        nxt = (clips.pose_3d[f0:first[e] + lengths[e]] == x3[1, b]).flatten(1).all(1).nonzero().flatten().tolist()
        speed = nxt[0]
        frames = f0 + speed * torch.arange(len(x3), device=x3.device)
        assert torch.equal(clips.pose_3d[frames], x3[:, b]) and torch.equal(clips.pose_2d[frames], x2[:, b]), b
        ids.append((e, f0 - first[e], speed))
    return ids


@pytest.mark.parametrize("split,speeds,B", [("test", (1, 1), 3), ("train", (1, 3), 1), ("train", (6, 6), 2)])
def test_pose_batches_epochs_lengths_and_camera_views(fix, split, speeds, B):
    from p2pvg_b200.data import PoseBatches
    clips = clips_of(fix, split, speeds[1])
    n, L = len(clips), fix["max_seq_len"]
    torch.manual_seed(5)
    np.random.seed(7)
    it = PoseBatches(clips, B, (L - 2 * fix["delta_len"], L), speeds, generator=torch.Generator("cuda").manual_seed(3))
    epochs, lengths, seen_speeds = [], [], set()
    for _ in range(10):
        epoch = []
        for _ in range(n // B):
            x2, x3, cv = next(it)
            T = len(x3)
            lengths.append(T)
            assert x2.is_cuda and x3.is_cuda and x2.dtype == x3.dtype == torch.float32
            assert x2.shape == (T, B, 17, 2) and x3.shape == (T, B, 17, 3) and x2.is_contiguous() and x3.is_contiguous()
            assert cv.device.type == "cpu" and cv.dtype == torch.int64 and cv.shape == (B,)
            ids = row_windows(clips, x2, x3)
            for (e, start, speed), v in zip(ids, cv.tolist()):
                assert 0 <= start <= clips.lengths[e] - speeds[1] * L and speeds[0] <= speed <= speeds[1]
                assert v == fix[split]["camera_view"][e]
                seen_speeds.add(speed)
                epoch.append(e)
        epochs.append(epoch)
    for epoch in epochs:
        assert len(set(epoch)) == len(epoch) == n // B * B     # drop_last: a permutation's first n // B * B entries
    assert len({tuple(e) for e in epochs}) > 1
    assert seen_speeds == set(range(speeds[0], speeds[1] + 1))
    np.random.seed(7)
    assert lengths == [np.random.randint(L - 2 * fix["delta_len"], L + 1) for _ in lengths]


def test_next_does_not_synchronise(fix):
    from p2pvg_b200.data import PoseBatches
    clips = clips_of(fix, "test", 1)
    it = PoseBatches(clips, 3, (20, 30), (1, 1))
    next(it)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(7):       # crosses two epoch boundaries: a new permutation uploaded each time
            next(it)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def test_seeds_repeat(fix):
    from p2pvg_b200.data import PoseBatches
    clips = clips_of(fix, "train", 3)
    runs = []
    for _ in range(2):
        torch.manual_seed(2)
        np.random.seed(4)
        it = PoseBatches(clips, 1, (20, 30), (1, 3), generator=torch.Generator("cuda").manual_seed(9))
        runs.append([next(it) for _ in range(6)])
    for a, b in zip(*runs):
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])


def test_h36m_mlp_steps_on_pose_batches(fix, monkeypatch):
    from p2pvg_b200.data import PoseBatches
    from p2pvg_b200.models import h36m_mlp
    from p2pvg_b200.models.p2p_model import P2PModel
    monkeypatch.setenv("P2PVG_PRECISION", "fp32")
    monkeypatch.setenv("P2PVG_GRAPH", "0")
    B = 10
    opt = types.SimpleNamespace(dataset="h36m", backbone_net=h36m_mlp, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0,
                                weight_align=0.5, skip_prob=0.5, n_past=1, last_frame_skip=False, batch_size=B)
    torch.manual_seed(1)
    model = P2PModel(B, 1, 128, 10, 512, 1, 1, 2, opt=opt).cuda()
    model.train()
    np.random.seed(0)
    it = PoseBatches(clips_of(fix, "test", 1), B, (20, 30), (1, 1), generator=torch.Generator("cuda").manual_seed(0))
    for _ in range(3):
        x = next(it)
        losses = model(x, 0, len(x[1]) - 1)
        assert len(losses) == 4 and all(np.isfinite(float(v)) for v in losses)


def test_dropin_generators(fix, monkeypatch):
    monkeypatch.setenv("P2PVG_REF", "")
    monkeypatch.syspath_prepend(os.path.join(ROOT, "dropin"))
    for m in ("data", "data.data_utils"):
        monkeypatch.delitem(sys.modules, m, raising=False)
    import data.data_utils as du
    try:
        opt = types.SimpleNamespace(dataset="h36m", batch_size=2)
        train, test = (du.PoseSet(pose_tree.fixture_dataset(fix, s)) for s in ("train", "test"))
        assert train.clips.pose_3d.is_cuda and len(train) == fix["train"]["len"] and len(test) == fix["test"]["len"]
        assert list(train.skeleton.parents()) == fix["train"]["parents"]
        for ds, is_train, B in ((train, True, 2), (test, False, 10)):
            gen = du.get_data_generator(ds, train=is_train, opt=opt)
            for _ in range(3):
                x2, x3, cv = next(gen)
                assert x3.is_cuda and x3.shape[1:] == (B, 17, 3) and x2.shape == x3.shape[:3] + (2,) and 20 <= len(x3) <= 30
                assert cv.shape == (B,)
        # the reference's test loader draws batches of 10: a split with fewer entries is refused, not looped on forever
        small = du.PoseSet(pose_tree.fixture_dataset(fix, "train"))
        with pytest.raises(ValueError, match="exceeds"):
            du.get_data_generator(small, train=False, opt=opt)
    finally:
        for m in ("data", "data.data_utils"):
            sys.modules.pop(m, None)


def test_kernel_rejects_bad_arguments():
    from p2pvg_b200._lib import load_library
    lib = load_library()
    B, L, T, J = 2, 4, 3, 5
    p2 = torch.zeros(20, J, 2, device="cuda")
    p3 = torch.zeros(20, J, 3, device="cuda")
    first = torch.tensor([0, 8], dtype=torch.int64, device="cuda")
    lens = torch.tensor([8, 12], dtype=torch.int32, device="cuda")
    entries = torch.tensor([0, 1], dtype=torch.int32, device="cuda")
    draws = torch.zeros(2, B, dtype=torch.int32, device="cuda")
    o2 = torch.empty(T, B, J, 2, device="cuda")
    o3 = torch.empty(T, B, J, 3, device="cuda")
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = ctypes.c_void_p

    def call(a=p2.data_ptr(), c=p3.data_ptr(), J=J, sf=first.data_ptr(), sl=lens.data_ptr(), n_seq=2, en=entries.data_ptr(),
             dr=draws.data_ptr(), B=B, lo=1, hi=2, L=L, T=T, x=o2.data_ptr(), y=o3.data_ptr()):
        return lib.p2pvg_pose_windows(P(a), P(c), J, P(sf), P(sl), n_seq, P(en), P(dr), B, lo, hi, L, T, P(x), P(y), stream)

    assert call() == 0
    assert call(T=0) == 0 and call(B=0) == 0
    torch.cuda.synchronize()
    for kw in (dict(a=None), dict(c=None), dict(sf=None), dict(sl=None), dict(en=None), dict(dr=None), dict(x=None), dict(y=None),
               dict(a=p2.data_ptr() + 2), dict(c=p3.data_ptr() + 1), dict(sf=first.data_ptr() + 4), dict(sl=lens.data_ptr() + 2),
               dict(en=entries.data_ptr() + 2), dict(dr=draws.data_ptr() + 1), dict(x=o2.data_ptr() + 2),
               dict(y=o3.data_ptr() + 3), dict(T=L + 1), dict(T=-1), dict(B=-1), dict(L=0), dict(J=0), dict(n_seq=0),
               dict(lo=0), dict(lo=3, hi=2)):
        assert call(**kw) == -1, kw
    for kw in (dict(hi=2 ** 30), dict(J=2 ** 28)):
        assert call(**kw) == -2, kw
