#!/usr/bin/env python
"""PNG encoding on the GPU (p2pvg_b200.png) against the host encoders it replaces in train.py's vis_seq calls.

  (a) torchvision.utils.save_image against p2pvg_b200.png.save_image of a CUDA picture, on the three pictures train.py
      writes most: the dcgan_64 Moving MNIST vis_seq canvas and the vgg_64 colour canvas (3 x 3840 x 1920 each: 10 blocks of
      6 rows, 30 frames of 64 px; tests/png_ref.py draws them), and the dcgan_128 gen_full picture (3 x 640 x 3840).  Host
      clock around the call, which ends with the file written; file sizes of both.
  (b) one vis_seq call end to end as train.py makes it (dcgan_64, B=100, nsample 20, output_len 30, skip_frame=False, bf16),
      through the drop-in (dropin/misc/visualize.py and dropin/tensorboardX's writer) against p2pvg_b200.visualize.vis_seq
      with torchvision's save_image and the stock torch.utils.tensorboard writer, both writing real files and event records
      in a temporary directory (flushed inside the timed call).  imageio and moviepy are stubbed for both: GIFs and videos
      are not part of this measurement.  Also timed: the call with the PNG file and the image record skipped (generation,
      composition and the GIF frames' copy), the canvas' device-to-host copy alone, the drop-in writer's add_image of the host
      canvas alone, and the event-file write of a ready image record alone.
  (c) the kernels alone: torch.profiler device times of one encode_png of each canvas, in a run of its own; and CUDA events
      around encode_png (launches, the size read-back and the pinned copy).

The variants alternate, after warm-up; median and [min..max] of --reps.  Prints the card name, power limit and SM clocks,
then one JSON line per row."""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torchvision.utils as vutils  # noqa: E402

from bench_vis_seq import NoWriter, card, make  # noqa: E402
from p2pvg_b200 import png  # noqa: E402
from p2pvg_b200 import visualize as V  # noqa: E402
from tests.png_ref import mnist_canvas, rgb_canvas  # noqa: E402

PICTURES = {
    "dcgan64_vis_seq_mnist": lambda: mnist_canvas(seed=1),
    "vgg64_vis_seq_rgb": lambda: rgb_canvas(seed=1),
    "dcgan128_gen_full": lambda: mnist_canvas(rows=5, cols=30, size=128, seed=2),
}


def host_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def stats(ts):
    return {"median_ms": round(statistics.median(ts), 3), "min_ms": round(min(ts), 3), "max_ms": round(max(ts), 3)}


def alternate(fns, reps, warmup=2):
    for _ in range(warmup):
        for fn in fns.values():
            fn()
    ts = {k: [] for k in fns}
    for _ in range(reps):
        for k, fn in fns.items():
            ts[k].append(host_ms(fn))
    return {k: stats(v) for k, v in ts.items()}


def part_a(reps, d):
    for name, make_pic in PICTURES.items():
        t = make_pic().cuda()
        paths = {"torchvision": os.path.join(d, name + "_tv.png"), "gpu": os.path.join(d, name + "_gpu.png")}
        res = alternate({"torchvision": lambda: vutils.save_image(t, paths["torchvision"]),
                         "gpu": lambda: png.save_image(t, paths["gpu"])}, reps)
        sizes = {k: os.path.getsize(p) for k, p in paths.items()}
        print(json.dumps({"part": "a", "picture": name, "shape": list(t.shape), **{k: {**res[k], "bytes": sizes[k]}
                                                                                    for k in res},
                          "speedup": round(res["torchvision"]["median_ms"] / res["gpu"]["median_ms"], 1),
                          "size_ratio": round(sizes["gpu"] / sizes["torchvision"], 3)}), flush=True)


def part_b(reps, d):
    from torch.utils.tensorboard import SummaryWriter as Stock
    sys.path.insert(0, os.path.join(ROOT, "dropin"))
    import misc.visualize as dropin_vis
    from tensorboardX import SummaryWriter as DropinWriter
    sys.modules["imageio"] = types.SimpleNamespace(mimsave=lambda name, frames: None)
    B, ns, L = 100, 20, 30
    os.environ["P2PVG_PRECISION"] = "bf16"
    model, C = make("dcgan64", B, ns, d)
    os.makedirs(os.path.join(d, "gen_vis"), exist_ok=True)
    x = torch.rand(30, B, C, 64, 64, generator=torch.Generator().manual_seed(3)).cuda()
    writers = {"stock": Stock(os.path.join(d, "tb_stock")), "dropin": DropinWriter(os.path.join(d, "tb_dropin"))}
    for w in writers.values():
        w.add_video = lambda *a, **k: None
    canvas = [None]

    def stock():
        canvas[0] = V.vis_seq(model, x, 0, L, skip_frame=False, writer=writers["stock"], opt=model.opt)[0]
        writers["stock"].flush()

    def dropin():
        dropin_vis.vis_seq(model, x, 0, L, skip_frame=False, writer=writers["dropin"], opt=model.opt)
        writers["dropin"].flush()

    def no_png():
        V.vis_seq(model, x, 0, L, skip_frame=False, writer=NoWriter(), opt=model.opt, save_png=lambda t, name: None)

    with torch.no_grad():
        res = alternate({"stock": stock, "dropin": dropin, "without_png_and_image": no_png}, reps)
        res["canvas_to_host"] = stats([host_ms(lambda: canvas[0].cpu().numpy()) for _ in range(reps)])
        host = canvas[0].cpu().numpy()
        w = writers["dropin"]

        def add_image():
            w.add_image("x", host, 0)
            w.flush()
        res["dropin_add_image_alone"] = stats([host_ms(add_image) for _ in range(reps)])
        from tensorboard.compat.proto.summary_pb2 import Summary
        data, = png.encode_png([canvas[0].contiguous()], "tensorboard")
        rec = Summary(value=[Summary.Value(tag="x", image=Summary.Image(height=host.shape[1], width=host.shape[2],
                                                                        colorspace=3, encoded_image_string=data))])

        def event_write():
            w._get_file_writer().add_summary(rec, 0, None)
            w.flush()
        res["event_write_alone"] = stats([host_ms(event_write) for _ in range(reps)])
        res["event_record_bytes"] = len(data)
    print(json.dumps({"part": "b", "workload": f"dcgan_64 B={B} nsample={ns} output_len={L} bf16", **res,
                      "speedup": round(res["stock"]["median_ms"] / res["dropin"]["median_ms"], 2)}), flush=True)


def part_c(reps):
    pics = {k: f().cuda() for k, f in PICTURES.items()}
    for k, t in pics.items():
        png.encode_png([t])
        ts = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            png.encode_png([t])
            b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        print(json.dumps({"part": "c", "picture": k, "encode_png_events": stats(ts)}), flush=True)
    from torch.profiler import ProfilerActivity, profile
    for k, t in pics.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            png.encode_png([t])
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            if e.device_type.name == "CUDA" and e.device_time_total > 0:
                kern[e.key[:60]] = round(e.device_time_total / 1e3, 3)
        print(json.dumps({"part": "c", "picture": k, "profiler_device_ms": kern}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--parts", default="abc")
    a = ap.parse_args()
    print("card:", card(), flush=True)
    with tempfile.TemporaryDirectory() as d:
        if "a" in a.parts:
            part_a(a.reps, d)
        if "b" in a.parts:
            part_b(a.reps, d)
    if "c" in a.parts:
        part_c(a.reps)


if __name__ == "__main__":
    main()
