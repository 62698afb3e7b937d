#!/usr/bin/env python
"""Write tests/golden/video_ref.json by running the UNMODIFIED reference Weizmann and BAIR loaders on the seeded synthetic trees
of tests/video_tree.py.

Needs the reference checkout ($P2PVG_REF, read-only; nothing is copied from it), like make_golden.py.  Its ``data/weizmann.py``
and ``data/bair.py`` are imported as-is with these substitutions:

  1. stub modules for ``matplotlib.pyplot`` (imported, unused, by weizmann.py) and for ``scipy.misc.imresize`` / ``imread``
     (imported, unused, by bair.py; gone from SciPy);
  2. ``np.random.randint(low, high)`` -> ``low + r % (high - low)`` with r the next value of a seeded draws table, which is the
     contract of p2pvg_video_windows (include/p2pvg_b200.h) for a window start;
  3. ``Image.open`` wrapped to record which frame files each clip / sequence is read from (the reference keeps no names).

Recorded per case, with hashes only so the fixture stays small:
  weizmann_{train,test}  the clips in the reference's append order (name, frame files), and for each draw: the dataset index,
                         r, and the SHA-256 of the fp32 sequence ``__getitem__`` returns (all L frames, and the first t_short)
  bair_train             for each draw: r, the trajectory ``get_seq`` picked (``randint(len(dirs))``) and the sequence hashes
  bair_test              the ordered walk through DataLoader(batch_size=3, shuffle=True, drop_last=True, num_workers=1) over two
                         epochs, with ``__len__`` cut to 10 items so an epoch is 3 batches: trajectory names per batch row
                         and hashes
The writer asserts that every odd Weizmann entry is the left-right mirror of the entry before it.

    python tests/golden/make_golden_video.py
"""
import hashlib
import importlib.util
import json
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests import video_tree  # noqa: E402

REF = os.environ.get("P2PVG_REF", "/root/reference")
WEIZMANN_ROUNDS = 3     # every Weizmann entry is drawn this many times
BAIR_DRAWS = 12
BAIR_DELTA = 5
ORDERED_B, ORDERED_ITEMS, ORDERED_EPOCHS = 3, 10, 2


def sha(x):
    return hashlib.sha256(np.ascontiguousarray(x.numpy()).tobytes()).hexdigest()


def install_stubs():
    plt = types.ModuleType("matplotlib.pyplot")
    mpl = types.ModuleType("matplotlib")
    mpl.pyplot = plt
    misc = types.ModuleType("scipy.misc")

    def unavailable(*a, **k):
        raise RuntimeError("scipy.misc stub: not used by the loaders")
    misc.imresize = misc.imread = unavailable
    sys.modules.update({"matplotlib": mpl, "matplotlib.pyplot": plt, "scipy.misc": misc})


def load_ref(name):
    spec = importlib.util.spec_from_file_location(f"ref_{name}", os.path.join(REF, "data", f"{name}.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class OpenRecorder:
    """Wraps the module's ``Image.open`` and records the path of every frame read, relative to ``base``."""

    def __init__(self, mod, base):
        self.mod, self.base, self.paths = mod, base, []
        self.orig = mod.Image.open

    def __enter__(self):
        def record(path, *a, **k):
            self.paths.append(os.path.relpath(path, self.base))
            return self.orig(path, *a, **k)
        self.mod.Image.open = record
        return self

    def __exit__(self, *exc):
        self.mod.Image.open = self.orig


class DrawTable:
    """np.random.randint(low, high) -> low + r % (high - low), r the next draw of the table."""

    def __init__(self, draws):
        self.draws, self.k = draws, 0

    def __enter__(self):
        self.orig = np.random.randint

        def randint(low, high=None, size=None, dtype=int):
            assert size is None
            if high is None:
                low, high = 0, low
            r = int(self.draws[self.k])
            self.k += 1
            return low + r % (high - low)
        np.random.randint = randint
        return self

    def __exit__(self, *exc):
        np.random.randint = self.orig


def weizmann_case(wz, root, train):
    L = video_tree.TRAIN_LEN if train else video_tree.TEST_LEN
    t_short = 10 if train else 6   # the shortest T get_seq_len() draws
    base = os.path.join(root, "weizmann")
    with OpenRecorder(wz, base) as rec:
        ds = wz.WeizmannDataset(data_root=root, train=train, max_seq_len=L, image_size=video_tree.SIZE)
    # each clip reads its frames in one run: group the recorded paths by clip directory
    clips = []
    for p in rec.paths:
        name = os.path.dirname(p)
        if not clips or clips[-1]["name"] != name:
            clips.append({"name": name, "files": []})
        clips[-1]["files"].append(os.path.basename(p))
    assert len(ds.data) == 2 * len(clips)
    for k, c in enumerate(clips):
        a, b = ds.data[2 * k], ds.data[2 * k + 1]
        assert a["n_frames"] == b["n_frames"] == len(c["files"])
        assert torch.equal(b["seq"], a["seq"].flip(-1)), c["name"]
    rs = np.random.RandomState(7 if train else 8)
    index = np.concatenate([rs.permutation(len(ds)) for _ in range(WEIZMANN_ROUNDS)]).astype(np.int64)
    draws = rs.randint(0, 2 ** 31 - 1, size=len(index)).astype(np.int64)
    full, short = [], []
    with DrawTable(draws) as dt:
        for i in index:
            seq = ds[int(i)]
            full.append(sha(seq))
            short.append(sha(seq[:t_short]))
        assert dt.k == len(draws)
    return dict(max_seq_len=L, t_short=t_short, clips=clips, index=index.tolist(), draws=draws.tolist(), sha256_full=full,
                sha256_short=short)


def bair_train_case(bair, root):
    base = os.path.join(root, "bair", "processed_data", "train")
    ds = bair.BairRobotPush(root, train=True, max_seq_len=video_tree.BAIR_LEN, delta_len=BAIR_DELTA, image_size=video_tree.SIZE)
    draws = np.random.RandomState(9).randint(0, 2 ** 31 - 1, size=BAIR_DRAWS).astype(np.int64)
    names, full, short = [], [], []
    t_short = video_tree.BAIR_LEN - 2 * BAIR_DELTA
    with DrawTable(draws) as dt, OpenRecorder(bair, base) as rec:
        for _ in range(BAIR_DRAWS):
            n0 = len(rec.paths)
            seq = ds.get_seq()
            dirs = {os.path.dirname(p) for p in rec.paths[n0:]}
            assert len(dirs) == 1 and len(rec.paths) - n0 == video_tree.BAIR_LEN
            names.append(dirs.pop())
            full.append(sha(seq))
            short.append(sha(seq[:t_short]))
        assert dt.k == BAIR_DRAWS
    return dict(max_seq_len=video_tree.BAIR_LEN, t_short=t_short, draws=draws.tolist(), names=names, sha256_full=full,
                sha256_short=short)


def bair_test_case(bair, root, arrays):
    from torch.utils.data import DataLoader

    class Short(bair.BairRobotPush):
        def __len__(self):
            return ORDERED_ITEMS

    ds = Short(root, train=False, max_seq_len=video_tree.BAIR_LEN, delta_len=BAIR_DELTA, image_size=video_tree.SIZE)
    # the worker process reads the frames, so each returned sequence is named by its first frame, matched to the tree's arrays
    first = {a[0].tobytes(): name.split("/", 1)[1] for name, a in arrays.items() if name.startswith("test/")}
    loader = DataLoader(ds, batch_size=ORDERED_B, shuffle=True, drop_last=True, num_workers=1)
    batches, full = [], []
    for _ in range(ORDERED_EPOCHS):
        for x in loader:
            batches.append([first[(s[0] * 255).round().to(torch.uint8).permute(1, 2, 0).numpy().tobytes()] for s in x])
            full.extend(sha(s) for s in x)
    t_short = video_tree.BAIR_LEN - 2 * BAIR_DELTA
    return dict(max_seq_len=video_tree.BAIR_LEN, t_short=t_short, batch_size=ORDERED_B, epoch_items=ORDERED_ITEMS,
                batches=batches, sha256_full=full)


def main():
    if not os.path.isdir(REF):
        raise SystemExit(f"reference checkout not found at {REF}")
    install_stubs()
    wz, bair = load_ref("weizmann"), load_ref("bair")
    with tempfile.TemporaryDirectory() as root:
        video_tree.write_weizmann_tree(root)
        arrays = video_tree.write_bair_tree(root)
        rec = dict(size=video_tree.SIZE, weizmann_seed=video_tree.WEIZMANN_SEED, bair_seed=video_tree.BAIR_SEED,
                   weizmann_train=weizmann_case(wz, root, True), weizmann_test=weizmann_case(wz, root, False),
                   bair_train=bair_train_case(bair, root), bair_test=bair_test_case(bair, root, arrays))
    with open(os.path.join(HERE, "video_ref.json"), "w") as f:
        json.dump(rec, f, indent=1)
    print("video_ref.json ok")


if __name__ == "__main__":
    main()
