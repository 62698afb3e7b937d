"""A seeded synthetic Human3.6M tree, laid out the way the reference's ``Human36mDataset`` reads it, and the module stubs that
let its unmodified ``data/human36m/human36m.py`` run without ``h5py`` or ``matplotlib``.

``<root>/processed/h36m-fetch/processed/<subject>/<action>/annot.h5`` (the path ``load_dataset`` builds from ``--data_root``):
the files are empty placeholders, and the ``h5py.File`` stub serves seeded ``pose/2d`` [4n, 32, 2] and ``pose/3d``
[4n, 32, 3] arrays (four camera views of n frames each, as h36m-fetch stores them) plus a ``frame`` dataset for each one.
Per split, with windows of ``L = 30`` frames:
  * one sequence shorter than L (dropped by the length filter);
  * one of exactly 180 frames: at the train split's speed 6 its only window start is 0;
  * longer ones, and in the test split one of exactly L frames, ten entries in all (the reference's test batch is 10);
  * a subject of neither split (``S2``), which the reference skips."""
import os
import types

import numpy as np

SUBDIR = os.path.join("processed", "h36m-fetch", "processed")
SEED = 36
L, DELTA_LEN = 30, 5
# subject -> {action: frames per view}
TREE = {
    "S1": {"Directions": 12, "Eating": 180, "Walking": 193},
    "S2": {"Waiting": 200},
    "S5": {"Greeting": 214},
    "S9": {"Phoning": 17, "Photo": 33, "Posing": 30, "Purchases": 52, "SittingDown": 38, "Waiting": 31},
    "S11": {"Discussion": 35, "Greeting": 44, "Sitting": 180, "Smoking": 41, "Walking": 36},
}


def annotation(subject, action):
    """The seeded arrays of one annot.h5: 2d poses around an image centre in pixels, 3d poses in millimetres."""
    n = TREE[subject][action]
    rs = np.random.RandomState(SEED + sorted((s, a) for s in TREE for a in TREE[s]).index((subject, action)))
    pose_2d = 500 + 120 * rs.randn(4 * n, 32, 2)
    pose_3d = np.array([0, 0, 4500]) + 400 * rs.randn(4 * n, 32, 3)
    return {"pose": {"2d": pose_2d, "3d": pose_3d}, "frame": np.arange(4 * n)}


def write_tree(root):
    """Placeholder annot.h5 files under ``root``; returns ``root``, the ``--data_root`` to pass to ``load_dataset``."""
    for subject, actions in TREE.items():
        for action in actions:
            d = os.path.join(root, SUBDIR, subject, action)
            os.makedirs(d, exist_ok=True)
            open(os.path.join(d, "annot.h5"), "wb").close()
    return root


def stub_modules():
    """{name: module} for ``sys.modules``: ``h5py`` serving ``annotation()`` for any ``<subject>/<action>/annot.h5`` path, and
    empty ``matplotlib`` / ``mpl_toolkits`` modules (imported by human36m.py for its visualiser only)."""
    h5py = types.ModuleType("h5py")

    class Group(dict):
        pass

    class File(Group):
        def __init__(self, path, mode="r"):
            action_dir = os.path.dirname(os.path.abspath(path))
            a = annotation(os.path.basename(os.path.dirname(action_dir)), os.path.basename(action_dir))
            super().__init__(pose=Group(a["pose"]), frame=a["frame"])

    h5py.Group, h5py.File = Group, File
    plt = types.ModuleType("matplotlib.pyplot")
    mpl = types.ModuleType("matplotlib")
    mpl.pyplot = plt
    mplot3d = types.ModuleType("mpl_toolkits.mplot3d")
    mplot3d.Axes3D = None
    toolkits = types.ModuleType("mpl_toolkits")
    toolkits.mplot3d = mplot3d
    return {"h5py": h5py, "matplotlib": mpl, "matplotlib.pyplot": plt, "mpl_toolkits": toolkits, "mpl_toolkits.mplot3d": mplot3d}


def r_values(records, speed_range, rs):
    """Draws [2, K] int32 that the p2pvg_pose_windows mapping turns into the recorded starts and speeds: each is the recorded
    value plus a random multiple of its range, spread over all of uint32 and stored as int32 (two's complement)."""
    lo, hi = speed_range

    def spread(value, span):
        return value + span * np.array([rs.randint(0, 2 ** 32 // int(s)) for s in span], dtype=np.uint64)
    start = np.asarray(records["start"], dtype=np.uint64)
    r0 = spread(start, np.asarray(records["start_high"], dtype=np.uint64))
    r1 = spread(np.asarray(records["speed"], dtype=np.uint64) - np.uint64(lo), np.full(len(start), hi - lo + 1, dtype=np.uint64))
    return np.stack([r0, r1]).astype(np.uint32).view(np.int32)


class FixtureDataset(types.SimpleNamespace):
    """Stands in for a ``Human36mDataset`` with the attributes the drop-in reads, filled from pose_data_ref.pt."""

    def __len__(self):
        return len(self.data["pose"]["2d"])


def fixture_dataset(fix, split, **kw):
    s = fix[split]
    attrs = dict(data={"pose": {"2d": [a.numpy() for a in s["pose_2d"]], "3d": [a.numpy() for a in s["pose_3d"]]},
                       "camera_view": s["camera_view"]},
                 max_seq_len=fix["max_seq_len"], delta_len=fix["delta_len"], speed_range=s["speed_range"], n_breakpoints=0,
                 skeleton=types.SimpleNamespace(parents=lambda: np.array(s["parents"])))
    attrs.update(kw)
    return FixtureDataset(**attrs)
