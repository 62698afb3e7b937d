#!/usr/bin/env python
"""One ``vis_seq`` call (misc/visualize.py) as train.py makes it: the reference's, restated over the eager p2p_generate
(tests/vis_ref.vis_seq_ref: 20 calls on the whole test batch, the composition in torch), against p2pvg_b200.visualize.vis_seq
(the n_block displayed rows, all samples in one graph replay, one p2pvg_vis_canvas launch).  Workloads of
tools/bench_generate.py, bf16, randomly initialised weights, eval mode, skip_frame=False, nsample 20:

  (b) dcgan_64, C=1, B=100, 30 input frames, output_len 10 and 30
  (g) vgg_64,   C=3, B=128, 30 input frames, output_len 10 and 30

Both write through a no-op writer and a fake imageio into a temporary directory; save_image is torchvision's own when it is
installed (so the PNG encoding is timed), else the same conversion and PIL encoding.  Each time is a host clock around a call
that ends in a device synchronise; the two paths alternate, and the median and the spread (min..max) of --reps are reported.
The composition alone: the p2pvg_vis_canvas launch against the torch composition it replaces (tests/vis_ref.compose_ref on
the device), CUDA events, median of --reps.  Prints the card name, power limit and SM clocks, then one JSON line per row."""
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
from p2pvg_b200 import visualize as V  # noqa: E402
from p2pvg_b200.models import dcgan_64, vgg_64  # noqa: E402
from p2pvg_b200.models.p2p_model import P2PModel  # noqa: E402
from tests.vis_ref import Recorder, compose_ref, vis_seq_ref  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def save_image_pil(t, name):
    from PIL import Image
    a = t.mul(255).add_(0.5).clamp_(0, 255).permute(1, 2, 0).to("cpu", torch.uint8).numpy()
    Image.fromarray(a).save(name)


class NoWriter:
    def add_image(self, *a, **k):
        pass

    def add_video(self, *a, **k):
        pass


def install_io(rec):
    rec.imageio.mimsave = lambda name, frames: None
    sys.modules["imageio"] = rec.imageio
    try:
        import torchvision.utils as vutils
        rec.vutils.save_image = vutils.save_image
    except ImportError:
        tv = types.ModuleType("torchvision")
        tv.utils = types.SimpleNamespace(save_image=save_image_pil)
        sys.modules["torchvision"], sys.modules["torchvision.utils"] = tv, tv.utils
        rec.vutils.save_image = save_image_pil


def make(kind, B, ns, log_dir):
    net, C = (dcgan_64, 1) if kind == "dcgan64" else (vgg_64, 3)
    opt = types.SimpleNamespace(dataset="mnist", backbone_net=net, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0,
                                weight_align=0.5, skip_prob=0.5, n_past=1, last_frame_skip=False, batch_size=B, nsample=ns,
                                log_dir=log_dir)
    torch.manual_seed(1)
    return P2PModel(B, C, 128, 10, 256, 1, 1, 2, opt=opt).cuda().eval(), C


def host_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def event_ms(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts), min(ts), max(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only", default="bg")
    args = ap.parse_args()
    print("card:", card(), flush=True)
    rec = Recorder()
    install_io(rec)
    w = NoWriter()
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "gen_vis"))
        for tag, kind, B in (("b", "dcgan64", 100), ("g", "vgg64", 128)):
            if tag not in args.only:
                continue
            model, C = make(kind, B, 20, tmp)
            x = torch.rand(30, B, C, 64, 64, generator=torch.Generator().manual_seed(5)).cuda()
            for L in (10, 30):
                def ref():
                    vis_seq_ref(model, x, 0, L, model_mode="full", recon_mode=None, skip_frame=False, writer=w, opt=model.opt,
                                rec=rec)

                def new():
                    V.vis_seq(model, x, 0, L, model_mode="full", recon_mode=None, skip_frame=False, writer=w, opt=model.opt)
                ref()
                new()
                t = {"reference": [], "vis_seq": []}
                for _ in range(args.reps):
                    t["reference"].append(host_ms(ref))
                    t["vis_seq"].append(host_ms(new))
                # the composition alone, on the frames of one call: kernel against the torch composition it replaces
                nb, ns, r_len = 10, 20, max(30, L)
                g = torch.Generator(device="cuda").manual_seed(7)
                gt = torch.rand(30, nb, C, 64, 64, device="cuda", generator=g)
                smp = torch.rand(ns, L, nb, C, 64, 64, device="cuda", generator=g)
                np.random.seed(0)
                tiles = V.plan_tiles(30, L, nb, ns, lambda f: (0, f * nb), lambda s, f: (1, (s * L + f) * nb))
                s0, s1 = gt.reshape(-1, C, 64, 64), smp.reshape(-1, C, 64, 64)
                s_lists = [[1] + list(np.random.randint(ns, size=4)) for _ in range(nb)]
                k = event_ms(lambda: V.compose(s0, s1, tiles, C, 64), args.reps * 4)
                tc = event_ms(lambda: compose_ref(gt, smp, 30, L, s_lists)[:2], args.reps * 4)
                out = dict(workload=tag, backbone=kind, B=B, nsample=20, seq_len=30, output_len=L, r_len=r_len,
                           **{f"{k_}_ms": round(statistics.median(v), 2) for k_, v in t.items()},
                           **{f"{k_}_spread_ms": [round(min(v), 2), round(max(v), 2)] for k_, v in t.items()},
                           speedup=round(statistics.median(t["reference"]) / statistics.median(t["vis_seq"]), 2),
                           compose_kernel_ms=[round(v, 3) for v in k], compose_torch_ms=[round(v, 3) for v in tc],
                           out_bytes=3 * nb * 6 * r_len * 64 * 64 * (4 + 4 + 1))
                print(json.dumps(out), flush=True)
            del model
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
