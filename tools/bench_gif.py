#!/usr/bin/env python
"""GIF encoding on the GPU (p2pvg_b200.gif) and the native event-record checksum, against the host code they replace in
train.py's vis_seq calls.

  (a) 30-frame animations of the vis_seq GIF's shape [30, n_block * H, 6 * H, 3]: 640 x 384 grey digits with the orange and
      red borders, 640 x 384 colour, 1280 x 768 colour (the 128-pixel backbones).  p2pvg_b200.gif.save_gif of the CUDA
      frames against Pillow's save_all GIF writer (and imageio.mimsave when installed) of the host frames; host clock around
      the call, which ends with the file written.  File sizes, and the MSE of each file's decoded frames against the source.
  (b) one event record holding the dcgan_64 vis_seq PNG (tests/png_ref.mnist_canvas): tensorboard's RecordWriter.write
      (pure-Python masked CRC-32C) against the drop-in writer's native one, into memory.
  (c) one vis_seq call end to end as train.py makes it (B=100, nsample 20, output_len 30, skip_frame=False, bf16) for
      dcgan_64 and vgg_64, writing real files and event records in a temporary directory: the stock stack
      (p2pvg_b200.visualize.vis_seq with torchvision's save_image, imageio.mimsave -- Pillow's save_all writer when imageio is
      not installed -- and the stock torch.utils.tensorboard writer, whose add_video writes an empty value without moviepy)
      against the drop-ins (dropin/misc/visualize.py and dropin/tensorboardX's writer).

The variants alternate, after warm-up; median and [min..max] of the repetitions.  Prints the card name, power limit and SM
clocks, then one JSON line per row."""
import argparse
import io
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_png import alternate, host_ms, stats  # noqa: E402
from bench_vis_seq import card, make  # noqa: E402
from p2pvg_b200 import gif  # noqa: E402
from p2pvg_b200 import visualize as V  # noqa: E402
from tests.test_gif_gpu import grey_digits, smooth_colour, with_borders  # noqa: E402

ANIMATIONS = {
    "grey_640x384": lambda: with_borders(grey_digits(30, 640, 384, 1)),
    "colour_640x384": lambda: smooth_colour(30, 640, 384, 2),
    "colour_1280x768": lambda: smooth_colour(30, 1280, 768, 3),
}


def pil_save(name, frames):
    ims = [Image.fromarray(f) for f in frames]
    ims[0].save(name, format="GIF", save_all=True, append_images=ims[1:], duration=100, loop=0)


def decoded_mse(path, frames):
    im = Image.open(path)
    err = 0.0
    for k in range(len(frames)):
        im.seek(k)
        err += float(((np.asarray(im.convert("RGB")).astype(np.float64) - frames[k]) ** 2).mean())
    return err / len(frames)


def part_a(reps, d):
    try:
        import imageio
    except ImportError:
        imageio = None
    for name, make_frames in ANIMATIONS.items():
        host = make_frames()
        dev = torch.from_numpy(host).cuda()
        frames = list(host)
        paths = {k: os.path.join(d, f"{name}_{k}.gif") for k in ("gpu", "pillow", "imageio")}
        gpu = alternate({"gpu": lambda: gif.save_gif(paths["gpu"], dev)}, reps)["gpu"]
        res = {"gpu": gpu, "pillow": stats([host_ms(lambda: pil_save(paths["pillow"], frames)) for _ in range(2)])}
        if imageio is not None:
            res["imageio"] = stats([host_ms(lambda: imageio.mimsave(paths["imageio"], frames)) for _ in range(2)])
        for k in res:
            res[k]["bytes"] = os.path.getsize(paths[k])
            res[k]["mse"] = round(decoded_mse(paths[k], host), 3)
        print(json.dumps({"part": "a", "animation": name, "shape": list(host.shape), **res,
                          "speedup_vs_pillow": round(res["pillow"]["median_ms"] / gpu["median_ms"], 1),
                          "size_ratio_vs_pillow": round(res["gpu"]["bytes"] / res["pillow"]["bytes"], 3)}), flush=True)


def part_b(reps):
    from tensorboard.compat.proto.summary_pb2 import Summary
    from tensorboard.compat.proto.event_pb2 import Event
    from tensorboard.summary.writer.record_writer import RecordWriter
    from p2pvg_b200 import png, tboard
    from tests.png_ref import mnist_canvas
    canvas = mnist_canvas(seed=1).cuda()
    data, = png.encode_png([canvas], "tensorboard")
    ev = Event(wall_time=0.0, step=0, summary=Summary(value=[Summary.Value(tag="x", image=Summary.Image(
        height=canvas.shape[1], width=canvas.shape[2], colorspace=3, encoded_image_string=data))])).SerializeToString()
    stock, native = RecordWriter(io.BytesIO()), RecordWriter(io.BytesIO())

    class _FW:
        pass
    fw = _FW()
    fw.event_writer = _FW()
    fw.event_writer._async_writer = _FW()
    fw.event_writer._async_writer._writer = native
    tboard.native_record_crc(fw)
    res = {}
    for k, w in (("python", stock), ("native", native)):
        ts = []
        for _ in range(reps + 2):
            t0 = time.perf_counter()
            w.write(ev)
            ts.append((time.perf_counter() - t0) * 1e3)
        res[k] = stats(ts[2:])
    assert stock._writer.getvalue() == native._writer.getvalue()
    print(json.dumps({"part": "b", "record_bytes": len(ev), **res,
                      "speedup": round(res["python"]["median_ms"] / res["native"]["median_ms"], 1)}), flush=True)


def part_c(reps, d):
    from torch.utils.tensorboard import SummaryWriter as Stock
    sys.path.insert(0, os.path.join(ROOT, "dropin"))
    import misc.visualize as dropin_vis
    from tensorboardX import SummaryWriter as DropinWriter
    try:
        import imageio  # noqa: F401
        gif_writer = "imageio.mimsave"
    except ImportError:
        import types
        sys.modules["imageio"] = types.SimpleNamespace(mimsave=pil_save)
        gif_writer = "Pillow save_all (imageio not installed)"
    B, ns, L = 100, 20, 30
    os.environ["P2PVG_PRECISION"] = "bf16"
    for kind in ("dcgan64", "vgg64"):
        kd = os.path.join(d, kind)
        model, C = make(kind, B, ns, kd)
        os.makedirs(os.path.join(kd, "gen_vis"), exist_ok=True)
        x = torch.rand(30, B, C, 64, 64, generator=torch.Generator().manual_seed(3)).cuda()
        writers = {"stock": Stock(os.path.join(kd, "tb_stock")), "dropin": DropinWriter(os.path.join(kd, "tb_dropin"))}

        def stock():
            V.vis_seq(model, x, 0, L, skip_frame=False, writer=writers["stock"], opt=model.opt)
            writers["stock"].flush()

        def dropin():
            dropin_vis.vis_seq(model, x, 0, L, skip_frame=False, writer=writers["dropin"], opt=model.opt)
            writers["dropin"].flush()

        with torch.no_grad():
            res = alternate({"stock": stock, "dropin": dropin}, reps, warmup=1)
        sizes = {k: os.path.getsize(os.path.join(kd, "gen_vis", "gen-model_full-len-30-epoch_0.gif")) for k in ("dropin",)}
        for w in writers.values():
            w.close()
        print(json.dumps({"part": "c", "workload": f"{kind} B={B} nsample={ns} output_len={L} bf16", "stock_gif": gif_writer,
                          **res, "dropin_gif_bytes": sizes["dropin"],
                          "speedup": round(res["stock"]["median_ms"] / res["dropin"]["median_ms"], 2)}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--parts", default="abc")
    args = ap.parse_args()
    print(card(), flush=True)
    with tempfile.TemporaryDirectory() as d:
        if "a" in args.parts:
            part_a(args.reps, d)
        if "b" in args.parts:
            part_b(args.reps * 20)
        if "c" in args.parts:
            part_c(args.reps, d)


if __name__ == "__main__":
    main()
