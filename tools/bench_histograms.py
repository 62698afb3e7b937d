#!/usr/bin/env python
"""The reference's train.py histogram block (train.py:225-233: every parameter and gradient through add_histogram, every 50
iterations) for the dcgan_64 (C2: B=256, T=30) and vgg_64 (C3: B=128, T=30) parameter sets after one bf16 training step
with bench.py's options, three ways:

  (a) the stock block, param.data.cpu().numpy() into torch.utils.tensorboard's add_histogram (np.histogram on the host)
  (b) the same block through the drop-in writer (dropin/tensorboardX: the same host arrays, uploaded, counted on the GPU)
  (c) p2pvg_b200.tboard.add_param_histograms (one launch, one device-to-host copy, no per-tensor copies)

Each is a host clock around the whole block, ending with writer.flush() (the event file written, CRC32C included) and a
device synchronise; the three alternate, and the median and spread (min..max) of --reps are reported.  Reported apart:
one launch (CUDA events over --launches launches: table upload, counts memset and kernel), the kernel alone (torch.profiler
device time, in a profiler run of its own; GB/s against the bytes read), and the event-file write alone
(add_histogram_raw of precomputed fields + flush, the share of (c) that holds the CRC32C floor).  Prints the card name,
power limit and SM clocks, then one JSON line per configuration."""
import argparse
import importlib
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
from p2pvg_b200 import tboard  # noqa: E402
from p2pvg_b200.models.p2p_model import P2PModel  # noqa: E402

CONFIGS = {"C2": ("dcgan_64", "mnist", 1, 256), "C3": ("vgg_64", "weizmann", 3, 128)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def trained_model(name, T=30):
    backbone, dataset, C, B = CONFIGS[name]
    os.environ["P2PVG_PRECISION"], os.environ["P2PVG_GRAPH"] = "bf16", "1"
    torch.manual_seed(1)
    np.random.seed(0)
    opt = types.SimpleNamespace(dataset=dataset, backbone_net=importlib.import_module(f"p2pvg_b200.models.{backbone}"), lr=1e-3,
                                beta1=0.9, beta=1e-4, weight_cpc=100.0, weight_align=0.5, skip_prob=0.0, n_past=1,
                                last_frame_skip=False, batch_size=B)
    model = P2PModel(B, C, 128, 10, 256, 1, 1, 2, opt=opt).cuda().train()
    x = torch.rand(T, B, C, 64, 64, generator=torch.Generator().manual_seed(1234)).cuda()
    model(x, 0, T - 1)
    torch.cuda.synchronize()
    return model


def stock_block(writer, model, step):
    for name, param in model.named_parameters():
        if param.requires_grad:
            name = name.replace('.', '/')
            writer.add_histogram(name, param.data.cpu().numpy(), step)
            try:
                writer.add_histogram(name + '/grad', param.grad.data.cpu().numpy(), step)
            except Exception:
                pass


def host_s(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def summary(xs):
    return dict(median=statistics.median(xs), min=min(xs), max=max(xs))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C2,C3")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--launches", type=int, default=50)
    args = ap.parse_args()
    print("card:", card(), flush=True)
    from torch.utils.tensorboard import SummaryWriter
    sys.path.insert(1, os.path.join(ROOT, "dropin"))
    DropIn = importlib.import_module("tensorboardX").SummaryWriter
    for name in args.configs.split(","):
        model = trained_model(name)
        tags, tensors = tboard.param_tensors(model)
        n_values = sum(t.numel() for t in tensors)
        n_bytes = sum(t.numel() * t.element_size() for t in tensors)
        with tempfile.TemporaryDirectory() as d:
            ws = {k: cls(log_dir=os.path.join(d, k)) for k, cls in (("a", SummaryWriter), ("b", DropIn), ("c", SummaryWriter),
                                                                    ("w", SummaryWriter))}
            paths = {"a": lambda s: (stock_block(ws["a"], model, s), ws["a"].flush()),
                     "b": lambda s: (stock_block(ws["b"], model, s), ws["b"].flush()),
                     "c": lambda s: (tboard.add_param_histograms(ws["c"], model, s), ws["c"].flush())}
            for k, fn in paths.items():   # warm-up: module loads, allocator, first file writes
                fn(0)
            times = {k: [] for k in paths}
            for r in range(args.reps):
                for k, fn in paths.items():
                    times[k].append(host_s(lambda: fn(r + 1)))
            # the event-file write alone: add_histogram_raw of precomputed fields, then flush
            fields = [tboard.histogram_fields(c, s, tboard.DEFAULT_BINS) for c, s in tboard.histograms(tensors)]

            def write(s):
                for tag, f in zip(tags, fields):
                    ws["w"].add_histogram_raw(tag, **f, global_step=s)
                ws["w"].flush()
            write(0)
            t_write = [host_s(lambda: write(r + 1)) for r in range(args.reps)]
            for w in ws.values():
                w.close()
        # one launch: table upload, counts memset and kernel, as seen by the stream
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(3):
            tboard.histograms_device(tensors)
        kern = []
        for _ in range(args.launches):
            e0.record()
            tboard.histograms_device(tensors)
            e1.record()
            e1.synchronize()
            kern.append(e0.elapsed_time(e1) * 1e-3)
        # the kernel's own device time, from a profiler run of its own (the event window above also holds the host's
        # enqueue: the table upload, the counts memset and the ctypes call)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(20):
                tboard.histograms_device(tensors)
            torch.cuda.synchronize()
        ev = [e for e in prof.key_averages() if "histogram_kernel" in e.key][0]
        k_dev = ev.device_time_total / ev.count * 1e-6
        row = dict(config=name, backbone=CONFIGS[name][0], histograms=len(tensors), values=n_values, bytes_read=n_bytes,
                   stock_s=summary(times["a"]), dropin_s=summary(times["b"]), direct_s=summary(times["c"]),
                   event_write_s=summary(t_write), launch_s=summary(kern), kernel_s=k_dev, kernel_GBps=n_bytes / k_dev / 1e9,
                   speedup_dropin=statistics.median(times["a"]) / statistics.median(times["b"]),
                   speedup_direct=statistics.median(times["a"]) / statistics.median(times["c"]),
                   event_write_share_of_direct=statistics.median(t_write) / statistics.median(times["c"]))
        print(json.dumps(row), flush=True)
        del model
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
