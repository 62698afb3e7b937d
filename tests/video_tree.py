"""Seeded synthetic Weizmann and BAIR directory trees, laid out the way the reference's loaders read them.

Every frame is a PNG of random uint8 pixels (all 256 levels occur, left and right halves differ), so PNG's lossless round trip
gives back exactly the seeded arrays and a mirrored or misplaced frame cannot pass for the right one.

Weizmann (``<root>/weizmann/<identity>/<action>/<frame>.png``), with ``TRAIN_LEN = 18`` and ``TEST_LEN = 10`` windows:
  * a stray file at the root (not an identity);
  * ``daria/jump``: 20 frames, too short for either split; ``moshe/skip``: 14 frames, likewise;
  * ``ido/run``: 27 frames, exactly 18 train frames, and 9 test frames (too short for the test split);
  * ``daria/bend`` (40), ``moshe/side`` (31) and ``ido/walk`` (44, grayscale): long enough for both splits;
  * unpadded frame numbers (``1.png``, ``10.png``, ``2.png``) in ``daria/bend`` and ``ido/walk``, so that the lexicographic
    order the reference sorts by differs from the numeric one; zero-padded names elsewhere.
BAIR (``<root>/bair/processed_data/{train,test}/<d1>/<d2>/{0..29}.png``): two d1 directories per split, trajectory names whose
lexicographic order differs from the numeric one."""
import os

import numpy as np
from PIL import Image

SIZE = 64
TRAIN_LEN, TEST_LEN = 18, 10
BAIR_LEN = 30
WEIZMANN_SEED, BAIR_SEED = 2024, 2025
# (identity, action, frames, grayscale, unpadded names)
WEIZMANN_CLIPS = [
    ("daria", "bend", 40, False, True),
    ("daria", "jump", 20, False, False),
    ("ido", "run", 27, False, False),
    ("ido", "walk", 44, True, True),
    ("moshe", "side", 31, False, False),
    ("moshe", "skip", 14, False, False),
]
BAIR_TRAJ = {"train": {"traj_0_to_255": ["9", "10", "11"], "traj_256_to_511": ["256", "300"]},
             "test": {"traj_0_to_255": ["2", "10"], "traj_256_to_511": ["7", "30"]}}


def random_frame(rs, gray, size=SIZE):
    shape = (size, size) if gray else (size, size, 3)
    a = rs.randint(0, 256, shape).astype(np.uint8)
    a.reshape(-1)[:256] = rs.permutation(256)
    assert not np.array_equal(a, a[:, ::-1])
    return a


def weizmann_frame_name(i, unpadded):
    return f"{i}.png" if unpadded else f"frame_{i:04d}.png"


def frame_number(name):
    """The frame index in a Weizmann frame file name written here."""
    return int("".join(ch for ch in name if ch.isdigit()))


def write_weizmann_tree(root, seed=WEIZMANN_SEED, size=SIZE):
    """Writes ``<root>/weizmann``; returns {"identity/action": [uint8 frame, ...] in frame-number order}."""
    rs = np.random.RandomState(seed)
    base = os.path.join(root, "weizmann")
    os.makedirs(base, exist_ok=True)
    with open(os.path.join(base, "README.txt"), "w") as f:
        f.write("not an identity\n")
    clips = {}
    for ident, act, n, gray, unpadded in WEIZMANN_CLIPS:
        d = os.path.join(base, ident, act)
        os.makedirs(d, exist_ok=True)
        frames = [random_frame(rs, gray, size) for _ in range(n)]
        for i, a in enumerate(frames):
            Image.fromarray(a, "L" if gray else "RGB").save(os.path.join(d, weizmann_frame_name(i, unpadded)))
        clips[f"{ident}/{act}"] = frames
    return clips


def write_bair_tree(root, seed=BAIR_SEED, size=SIZE, length=BAIR_LEN):
    """Writes ``<root>/bair/processed_data``; returns {"split/d1/d2": [uint8 frame, ...]}."""
    rs = np.random.RandomState(seed)
    clips = {}
    for split, d1s in BAIR_TRAJ.items():
        for d1, d2s in d1s.items():
            for d2 in d2s:
                d = os.path.join(root, "bair", "processed_data", split, d1, d2)
                os.makedirs(d, exist_ok=True)
                frames = [random_frame(rs, False, size) for _ in range(length)]
                for i, a in enumerate(frames):
                    Image.fromarray(a, "RGB").save(os.path.join(d, f"{i}.png"))
                clips[f"{split}/{d1}/{d2}"] = frames
    return clips
