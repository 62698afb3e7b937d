#!/usr/bin/env python
"""The reference's generate.py workload: one clip of T = 30 frames at batch 1, lengths 10, 20 and 30, 5 samples each, on
randomly initialised weights in eval mode (the default P2PVG_PRECISION), for dcgan_64, vgg_64 and dcgan_128 with 3 channels:
  eager     15 eager p2p_generate calls and the torch composition of generate.py (tests/generate_ref.generate_ref)
  looped    3 p2p_generate_graphed(nsample=5) calls, one per length
  lengths   one p2p_generate_lengths call
  video     generate_video end to end, writing into a temporary directory
  write     the file writing of generate_video alone (generate.write_files on its pictures: 21 PNGs, 18 GIFs)
and one batched API case (dcgan_64, B = 32, nsample 5): looped against lengths.  Every time is a host clock around a call
that ends in a device synchronise, after one warm-up call of each variant (graph capture); the variants alternate and the
median and the spread (min..max) of --reps are reported.  PNGs go through torchvision's save_image, GIFs through imageio when
it is installed, else a stand-in that only takes the frames.  Prints the card name, power limit and SM clocks, then one JSON
line per row."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from p2pvg_b200 import generate  # noqa: E402
from p2pvg_b200.models import dcgan_64, dcgan_128, vgg_64  # noqa: E402
from p2pvg_b200.models.p2p_model import P2PModel  # noqa: E402
from tests.generate_ref import generate_ref  # noqa: E402

LENS = [10, 20, 30]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def make(net, B, W):
    opt = types.SimpleNamespace(dataset="mnist", backbone_net=net, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0,
                                weight_align=0.5, skip_prob=0.5, n_past=1, last_frame_skip=False, batch_size=B)
    torch.manual_seed(1)
    model = P2PModel(B, 3, 128, 10, 256, 1, 1, 2, opt=opt).cuda().eval()
    x = torch.rand(30, B, 3, W, W, generator=torch.Generator().manual_seed(2)).cuda()
    return model, x


def host_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    print("card:", card(), flush=True)
    if "imageio" not in sys.modules:
        try:
            import imageio  # noqa: F401
        except ImportError:
            sys.modules["imageio"] = types.SimpleNamespace(mimsave=lambda name, frames: [np.asarray(f) for f in frames])
    import imageio
    import torchvision.utils as vutils
    with tempfile.TemporaryDirectory() as tmp:
        cases = [("dcgan_64", dcgan_64, 64, 1, 1), ("vgg_64", vgg_64, 64, 1, 1), ("dcgan_128", dcgan_128, 128, 1, 1),
                 ("dcgan_64 B=32", dcgan_64, 64, 32, 0)]
        for name, net, W, B, full in cases:
            model, x = make(net, B, W)
            variants = {
                "looped": lambda: [model.p2p_generate_graphed(x, L, L - 1, nsample=5) for L in LENS],
                "lengths": lambda: model.p2p_generate_lengths(x, LENS, nsample=5),
            }
            if full:
                pics = generate.generate_video(model, x, tmp)
                variants = dict(eager=lambda: generate_ref(model, x, tmp, vutils.save_image, imageio.mimsave), **variants,
                                video=lambda: generate.generate_video(model, x, tmp),
                                write=lambda: generate.write_files(tmp, LENS, pics, 5, imageio))
            for fn in variants.values():
                fn()
            ts = {k: [] for k in variants}
            for _ in range(args.reps):
                for k, fn in variants.items():
                    ts[k].append(host_ms(fn))
            row = {"workload": name, "T": 30, "B": B, "len_outputs": LENS, "nsample": 5, "reps": args.reps}
            for k, v in ts.items():
                row[k] = {"median_ms": round(statistics.median(v), 3), "min_ms": round(min(v), 3), "max_ms": round(max(v), 3)}
            for k in ("eager", "looped"):
                if k in ts:
                    row[f"lengths_speedup_vs_{k}"] = round(statistics.median(ts[k]) / statistics.median(ts["lengths"]), 2)
            if full:
                row["video_speedup_vs_eager"] = round(statistics.median(ts["eager"]) / statistics.median(ts["video"]), 2)
            print(json.dumps(row), flush=True)
            del model, x
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
