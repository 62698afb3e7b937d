#!/usr/bin/env python
"""Write the Moving MNIST fixtures (tests/golden/mmnist_*.pt) by running the UNMODIFIED reference renderer.

Needs the reference checkout ($P2PVG_REF, read-only; nothing is copied from it), like make_golden.py.  Its
``data/moving_mnist.py`` is imported as-is with three substitutions:

  1. ``datasets.MNIST`` -> an in-memory fake of 40 synthetic uint8 32x32 digits, returned through the transform like
     the real dataset returns them.  The real dataset is never constructed (``download=True`` would go to the network).
  2. an explicit ``transform=transforms.ToTensor()`` (the default ``transforms.Scale`` is gone from torchvision).
  3. ``np.random.randint(low, high)`` -> ``low + r % (high - low)`` with r popped from a seeded draws table row per
     (sequence, digit), which is exactly the contract of p2pvg_moving_mnist (include/p2pvg_b200.h).

The writer traces the reference's own locals to assert that every wall bounce of both rules occurs in every case and that
digit overlaps hit the final clip wherever two or more digits are drawn.

Outputs: mmnist_digits.pt (the digits) and one mmnist_det<0|1>_nd<n>_s<S>.pt per case: the draws, the SHA-256 of every
rendered fp32 sequence (all MAX_SEQ_LEN frames, and its first T_SHORT frames), and the first sequence's first T_SHORT
frames at S = 64 for diagnostics.

    python tests/golden/make_golden_mnist.py
"""
import hashlib
import importlib.util
import linecache
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("P2PVG_REF", "/root/reference")
N_DIGITS = 40
N_SEQ = 24
MAX_SEQ_LEN = 30
T_SHORT = 17
CASES = [(det, nd, S) for det in (False, True) for nd in (1, 2, 3) for S in (64, 128)]


def case_name(det, nd, S):
    return f"mmnist_det{int(det)}_nd{nd}_s{S}.pt"


def synthetic_digits():
    """Bright blobs with a saturated core and noisy rim: every uint8 level occurs, and two overlapping digits exceed 1."""
    rs = np.random.RandomState(2024)
    yy, xx = np.mgrid[0:32, 0:32]
    out = np.zeros((N_DIGITS, 32, 32), dtype=np.uint8)
    for i in range(N_DIGITS):
        cy, cx = rs.uniform(10, 22, 2)
        ry, rx = rs.uniform(6, 15, 2)
        r = ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2
        img = np.where(r < 1, rs.randint(0, 256, (32, 32)), 0)
        img[r < 0.35] = 255
        out[i] = img
    return out


def sha(x):
    return hashlib.sha256(np.ascontiguousarray(x.numpy()).tobytes()).hexdigest()


def load_reference_renderer(digits):
    from PIL import Image
    from torchvision import transforms
    spec = importlib.util.spec_from_file_location("ref_moving_mnist", os.path.join(REF, "data", "moving_mnist.py"))
    mm = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mm)

    class FakeMNIST:
        def __init__(self, root, train=True, download=False, transform=None):
            self.transform = transform

        def __len__(self):
            return len(digits)

        def __getitem__(self, i):
            return self.transform(Image.fromarray(digits[i])), 0

    mm.datasets.MNIST = FakeMNIST  # the module's own `datasets` namespace: the real class is never reached
    return mm, transforms.ToTensor()


def render_case(mm, transform, det, nd, S, draws):
    ds = mm.DynamicLengthMovingMNIST(data_root="unused", train=True, transform=transform, max_seq_len=MAX_SEQ_LEN, delta_len=0,
                                     image_size=S, num_digits=nd, deterministic=det)
    getitem = ds.__getitem__.__func__.__code__
    seen, clip_hit, cursor = set(), [False], {}
    lim = S - 32

    def randint(low, high=None, size=None, dtype=int):
        fr = sys._getframe(1)
        assert fr.f_code is getitem and size is None, "randint called outside __getitem__"
        if high is None:
            low, high = 0, low
        key = (fr.f_locals["index"], fr.f_locals["n"])
        k = cursor.get(key, 0)
        cursor[key] = k + 1
        return low + int(draws[key[0], key[1], k]) % (high - low)

    def local_trace(frame, event, arg):
        if event == "line":
            src = linecache.getline(frame.f_code.co_filename, frame.f_lineno).strip()
            L = frame.f_locals
            if src == "if sy < 0:":
                seen.add("sy<0" if L["sy"] < 0 else "sy>=" if L["sy"] >= lim else None)
            elif src == "if sx < 0:":
                seen.add("sx<0" if L["sx"] < 0 else "sx>=" if L["sx"] >= lim else None)
            elif src.startswith("x[t, 0, sy:sy+32, sx:sx+32]"):
                assert 0 <= L["sy"] <= S - 33 and 0 <= L["sx"] <= S - 33
            elif src.startswith("x[x>1]"):
                clip_hit[0] |= bool((L["x"] > 1).any())
        return local_trace

    def global_trace(frame, event, arg):
        return local_trace if frame.f_code is getitem else None

    orig = mm.np.random.randint
    mm.np.random.randint = randint
    sys.settrace(global_trace)
    try:
        seqs = [ds[b] for b in range(len(draws))]
    finally:
        sys.settrace(None)
        mm.np.random.randint = orig
    seen.discard(None)
    assert seen == {"sy<0", "sy>=", "sx<0", "sx>="}, (det, nd, S, seen)
    assert clip_hit[0] or nd == 1, (det, nd, S, "no digit overlap reached the clip")
    return seqs


def main():
    if not os.path.isdir(REF):
        raise SystemExit(f"reference checkout not found at {REF}")
    digits = synthetic_digits()
    mm, transform = load_reference_renderer(digits)
    torch.save({"digits": torch.from_numpy(digits)}, os.path.join(HERE, "mmnist_digits.pt"))
    for ci, (det, nd, S) in enumerate(CASES):
        stride = 5 + 4 * MAX_SEQ_LEN
        draws = np.random.RandomState(100 + ci).randint(0, 2 ** 31 - 1, size=(N_SEQ, nd, stride)).astype(np.int32)
        seqs = render_case(mm, transform, det, nd, S, draws)
        rec = dict(deterministic=det, num_digits=nd, image_size=S, max_seq_len=MAX_SEQ_LEN, t_short=T_SHORT,
                   draws=torch.from_numpy(draws), sha256_full=[sha(x) for x in seqs], sha256_short=[sha(x[:T_SHORT]) for x in seqs])
        if S == 64:
            rec["frames"] = seqs[0][:T_SHORT].clone()
        torch.save(rec, os.path.join(HERE, case_name(det, nd, S)))
        print(case_name(det, nd, S), "ok")


if __name__ == "__main__":
    main()
