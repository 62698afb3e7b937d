#!/usr/bin/env python
"""Write tests/golden/pose_data_ref.pt by running the UNMODIFIED reference ``Human36mDataset`` on the seeded synthetic tree of
tests/pose_tree.py.

Needs the reference checkout ($P2PVG_REF, read-only; nothing is copied from it), like make_golden.py.  Its
``data/human36m/human36m.py`` is imported as-is, with ``h5py``, ``matplotlib`` and ``mpl_toolkits`` stubbed through
``sys.modules`` (pose_tree.stub_modules: the ``h5py.File`` stub serves the tree's seeded annotations).  ``__init__`` runs for
real: reading, reformatting, the length filter, the joint removal and the normalisation.  ``np.random.randint`` is wrapped to
record what each ``__getitem__`` draws, and for some calls to force the window start to its lowest or highest value.

Recorded per case, as load_dataset builds the datasets (max_seq_len 30, delta_len 5, no breakpoints):
  train         speed_range [6, 6]; test: [1, 1]
  train_speeds  the train split with speed_range [1, 3], so that the speed draw has a range (its lists equal train's)
For train and test: the normalised float64 lists ``data['pose']['2d' | '3d']``, ``data['camera_view']``, ``len`` and the skeleton
parents.  For every case, per ``__getitem__``: the index, the start and speed drawn, the start's randint ``high``, and the
SHA-256 of ``torch.from_numpy(pose).float()`` for 2d and 3d, over all L frames and over the first ``t_short`` = 20.

    python tests/golden/make_golden_pose_data.py
"""
import hashlib
import importlib
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests import pose_tree  # noqa: E402

REF = os.environ.get("P2PVG_REF", "/root/reference")
ROUNDS = 4      # every entry is drawn this many times with NumPy's own draws
T_SHORT = pose_tree.L - 2 * pose_tree.DELTA_LEN


def sha(x):
    return hashlib.sha256(torch.from_numpy(x).float().numpy().tobytes()).hexdigest()


class Recorder:
    """Wraps np.random.randint: records (low, high, value) of every call; ``force`` holds values to return instead of a
    draw, None meaning "draw"."""

    def __init__(self):
        self.calls, self.force = [], []

    def __enter__(self):
        self.orig = np.random.randint

        def randint(low, high=None, size=None, dtype=int):
            assert size is None
            v = self.force.pop(0) if self.force else None
            v = self.orig(low, high) if v is None else v
            self.calls.append((int(low), int(high), int(v)))
            return v
        np.random.randint = randint
        return self

    def __exit__(self, *exc):
        np.random.randint = self.orig


def record(ds, seed):
    n = len(ds)
    rs = np.random.RandomState(seed)
    index = [int(i) for _ in range(ROUNDS) for i in rs.permutation(n)]
    forced = [None] * len(index)
    for e in range(n):          # each entry once at its lowest and once at its highest window start
        span = ds.data["pose"]["3d"][e].shape[0] - ds.speed_range[1] * ds.max_seq_len + 1
        index += [e, e]
        forced += [0, span - 1]
    np.random.seed(seed)
    rec = {k: [] for k in ("index", "start", "speed", "start_high", "sha_2d", "sha_3d", "sha_2d_short", "sha_3d_short")}
    with Recorder() as r:
        for i, f in zip(index, forced):
            r.force = [f, None]
            k = len(r.calls)
            item = ds[i]
            (lo0, hi0, start), (lo1, hi1, speed) = r.calls[k:]
            assert lo0 == 0 and (lo1, hi1) == (ds.speed_range[0], ds.speed_range[1] + 1) and item["speed"] == speed
            assert item["pose_2d"].shape[0] == item["pose_3d"].shape[0] == ds.max_seq_len
            for key, v in (("index", i), ("start", start), ("speed", speed), ("start_high", hi0),
                           ("sha_2d", sha(item["pose_2d"])), ("sha_3d", sha(item["pose_3d"])),
                           ("sha_2d_short", sha(item["pose_2d"][:T_SHORT])), ("sha_3d_short", sha(item["pose_3d"][:T_SHORT]))):
                rec[key].append(v)
    return rec


def dataset_fields(ds):
    return dict(pose_2d=[torch.from_numpy(a) for a in ds.data["pose"]["2d"]],
                pose_3d=[torch.from_numpy(a) for a in ds.data["pose"]["3d"]],
                camera_view=[int(v) for v in ds.data["camera_view"]], len=len(ds),
                parents=[int(p) for p in ds.skeleton.parents()])


def main():
    if not os.path.isdir(REF):
        raise SystemExit(f"reference checkout not found at {REF}")
    sys.modules.update(pose_tree.stub_modules())
    sys.path.insert(0, os.path.join(REF, "data", "human36m"))     # human36m.py imports `skeleton` by its bare name
    h36m = importlib.import_module("human36m")
    out = dict(max_seq_len=pose_tree.L, delta_len=pose_tree.DELTA_LEN, t_short=T_SHORT)
    with tempfile.TemporaryDirectory() as root:
        data_root = os.path.join(pose_tree.write_tree(root), pose_tree.SUBDIR)

        def dataset(mode, speed_range):
            return h36m.Human36mDataset(data_root=data_root, max_seq_len=pose_tree.L, delta_len=pose_tree.DELTA_LEN,
                                        speed_range=speed_range, n_breakpoints=0, acc_range=[0, 0], mode=mode)
        for name, mode, speeds, seed in (("train", "train", [6, 6], 1), ("test", "test", [1, 1], 2),
                                         ("train_speeds", "train", [1, 3], 3)):
            ds = dataset(mode, speeds)
            case = dict(speed_range=speeds, records=record(ds, seed))
            if name == "train_speeds":
                assert all(np.array_equal(a, b.numpy()) for a, b in zip(ds.data["pose"]["3d"], out["train"]["pose_3d"]))
            else:
                case.update(dataset_fields(ds))
            out[name] = case
    path = os.path.join(HERE, "pose_data_ref.pt")
    torch.save(out, path)
    print(f"pose_data_ref.pt ok: {os.path.getsize(path)} bytes, train {out['train']['len']} entries, test {out['test']['len']}")


if __name__ == "__main__":
    main()
