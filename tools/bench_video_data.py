#!/usr/bin/env python
"""Weizmann / BAIR input path: batches cut on the GPU from device-resident uint8 clips (p2pvg_video_windows) against the
reference's CPU loaders.

    python tools/bench_video_data.py gpu [--launches 300] [--steps 10] [--rounds 3] [--load-trajectories 256]
    python tools/bench_video_data.py cpu-reference --ref /path/to/p2pvg [--batches 3]

gpu: prints the card name, power limit and SM clock, then one JSON line each for
  kernel  p2pvg_video_windows at the Weizmann C3 batch (B = 128, T = 18) and the BAIR batch (B = 256, T = 30), 64x64x3:
          CUDA events around --launches launches after warm-up, and the fp32 bytes written per launch over that time; plus the
          host-clocked cost of one ClipBatches next() (T draw + randint + allocation + launch, ending in a synchronise)
  e2e     the C3 train step (vgg_64, 3 channels, B = 128, bf16, CUDA graph) fed by ClipBatches (`x = next(it); model(x, 0,
          T - 1)`) and the same loop on one resident batch, alternated --rounds times (median per loop); host clock around
          --steps steps ending in a synchronise
  load    the one-time decode of a synthetic BAIR tree of --load-trajectories trajectories x 30 PNG frames (written first to a
          temporary directory) by load_bair_clips, host clock
  The clip store for the kernel and e2e lines is synthetic: 93 Weizmann-sized clips (40..80 frames) and 1024 BAIR trajectories.
cpu-reference: the reference's own WeizmannDataset and BairRobotPush (train splits) through DataLoader(num_workers=1), as
  data/data_utils.py builds them but with a random sampler long enough for the timed batches, on synthetic trees written to a temporary directory (Weizmann:
  9 identities x 10 actions x 48 frames; BAIR: 64 trajectories x 30 frames); first batch (worker start) excluded.  Prints the
  host's CPU model and core count with the rate."""
import argparse
import importlib.util
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
S = 64
SHAPES = {"weizmann_c3": dict(B=128, T=18, L=18, paired=True), "bair": dict(B=256, T=30, L=30, paired=False)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def cpu_model():
    try:
        with open("/proc/cpuinfo") as f:
            return next(l.split(":", 1)[1].strip() for l in f if l.startswith("model name"))
    except (OSError, StopIteration):
        return "unknown"


def synthetic_clips(lens, L, paired, device):
    from p2pvg_b200.data import VideoClips
    lens = torch.tensor(lens, dtype=torch.int32)
    first = torch.cumsum(lens.long(), 0) - lens.long()
    frames = torch.randint(0, 256, (int(lens.sum()), 3, S, S), dtype=torch.uint8, generator=torch.Generator().manual_seed(0))
    return VideoClips(frames.to(device), first.to(device), lens.to(device), [str(i) for i in range(len(lens))], paired, L)


def time_kernel(K, clips, B, T, launches, gen):
    n = len(clips)
    entries = torch.randint(0, n, (B,), dtype=torch.int32, device="cuda", generator=gen)
    draws = torch.randint(0, 2 ** 31 - 1, (B,), dtype=torch.int32, device="cuda", generator=gen) if clips.paired_flips else None
    out = torch.empty(T, B, 3, S, S, device="cuda")

    def launch():
        K.video_windows(clips.frames, clips.clip_first, clips.clip_len, entries, draws, clips.paired_flips, clips.max_seq_len, out)
    for _ in range(20):
        launch()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(launches):
        launch()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / launches * 1e3, out.numel() * 4


def time_next(it, n=50):
    for _ in range(5):
        next(it)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        next(it)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n * 1e6


def run_gpu(args):
    from p2pvg_b200._lib import kernels_for
    from p2pvg_b200.data import ClipBatches, load_bair_clips
    from p2pvg_b200.models import vgg_64
    from p2pvg_b200.models.p2p_model import P2PModel
    from tests import video_tree
    if not torch.cuda.is_available():
        raise SystemExit("gpu mode needs a CUDA device")
    print("card:", card(), flush=True)
    K = kernels_for("cuda")
    gen = torch.Generator("cuda").manual_seed(0)
    rs = np.random.RandomState(0)
    weizmann = synthetic_clips(rs.randint(40, 81, 93).tolist(), 18, True, "cuda")
    bair = synthetic_clips([30] * 1024, 30, False, "cuda")
    stores = {"weizmann_c3": (weizmann, "permutation", (18, 18)), "bair": (bair, "uniform", (30, 30))}
    for name, shp in SHAPES.items():
        clips, sampling, seq_len = stores[name]
        us, nbytes = time_kernel(K, clips, shp["B"], shp["T"], args.launches, gen)
        next_us = time_next(ClipBatches(clips, shp["B"], sampling, seq_len, generator=gen))
        print(json.dumps(dict(metric="video_windows_kernel", shape=name, B=shp["B"], T=shp["T"], C=3, H=S, W=S,
                              kernel_us=round(us, 2), write_bytes=nbytes, write_GBps=round(nbytes / (us * 1e-6) / 1e9, 1),
                              clipbatches_next_us=round(next_us, 1))), flush=True)

    os.environ["P2PVG_PRECISION"] = "bf16"
    os.environ["P2PVG_GRAPH"] = "1"
    B = 128
    opt = types.SimpleNamespace(dataset="weizmann", backbone_net=vgg_64, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0,
                                weight_align=0.5, skip_prob=0.0, n_past=1, last_frame_skip=False, batch_size=B)
    torch.manual_seed(1)
    np.random.seed(0)
    model = P2PModel(B, 3, 128, 10, 256, 1, 1, 2, opt=opt).cuda()
    model.train()
    it = ClipBatches(weizmann, B, "permutation", seq_len=(18, 18), generator=gen)   # T fixed: one graph, comparable steps
    resident = next(it)

    def loop(fed, n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n):
            x = next(it) if fed else resident
            model(x, 0, len(x) - 1)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    loop(True, 4)
    loop(False, 4)
    res = {True: [], False: []}
    for _ in range(args.rounds):
        for fed in (True, False):
            res[fed].append(18 * B * args.steps / loop(fed, args.steps))
    fps = {k: statistics.median(v) for k, v in res.items()}
    print(json.dumps(dict(metric="video_e2e_c3", T=18, B=B, steps=args.steps, rounds=args.rounds,
                          frames_per_s_clipbatches=round(fps[True]), frames_per_s_resident=round(fps[False]),
                          ms_per_step_clipbatches=round(18 * B / fps[True] * 1e3, 2),
                          ms_per_step_resident=round(18 * B / fps[False] * 1e3, 2),
                          all_clipbatches=[round(v) for v in res[True]], all_resident=[round(v) for v in res[False]])), flush=True)
    del model
    torch.cuda.empty_cache()

    with tempfile.TemporaryDirectory() as root:
        write_bair(root, args.load_trajectories)
        t0 = time.perf_counter()
        clips = load_bair_clips(root, True, 30, S)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
    print(json.dumps(dict(metric="bair_load", trajectories=len(clips.names), frames=clips.frames.shape[0], seconds=round(dt, 2),
                          frames_per_s=round(clips.frames.shape[0] / dt), store_bytes=clips.frames.numel(),
                          cpu=cpu_model(), usable_cores=len(os.sched_getaffinity(0)))), flush=True)


def write_bair(root, n_traj, length=30):
    from tests import video_tree
    from PIL import Image
    rs = np.random.RandomState(1)
    for t in range(n_traj):
        d = os.path.join(root, "bair", "processed_data", "train", f"traj_{t // 256 * 256}_to_{t // 256 * 256 + 255}", str(t))
        os.makedirs(d)
        for i in range(length):
            Image.fromarray(video_tree.random_frame(rs, False)).save(os.path.join(d, f"{i}.png"))


def write_weizmann(root, ids=9, acts=10, frames=48):
    from PIL import Image
    from tests import video_tree
    rs = np.random.RandomState(2)
    for a in range(ids):
        for b in range(acts):
            d = os.path.join(root, "weizmann", f"id{a}", f"act{b}")
            os.makedirs(d)
            for i in range(frames):
                Image.fromarray(video_tree.random_frame(rs, False)).save(os.path.join(d, f"{i:03d}.png"))


def run_cpu_reference(args):
    from torch.utils.data import DataLoader, RandomSampler
    plt = types.ModuleType("matplotlib.pyplot")
    mpl = types.ModuleType("matplotlib")
    mpl.pyplot = plt
    misc = types.ModuleType("scipy.misc")
    misc.imresize = misc.imread = None     # imported, unused, by bair.py; gone from SciPy
    sys.modules.update({"matplotlib": mpl, "matplotlib.pyplot": plt, "scipy.misc": misc})

    def load(name):
        spec = importlib.util.spec_from_file_location(f"ref_{name}", os.path.join(args.ref, "data", f"{name}.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        return mod

    with tempfile.TemporaryDirectory() as root:
        write_weizmann(root)
        write_bair(root, 64)
        cases = [("weizmann_c3", 128, 18, lambda: load("weizmann").WeizmannDataset(data_root=root, train=True, max_seq_len=18,
                                                                                     image_size=S)),
                 ("bair", 256, 30, lambda: load("bair").BairRobotPush(root, train=True, max_seq_len=30, image_size=S))]
        for name, B, T, make in cases:
            t0 = time.perf_counter()
            ds = make()
            init_s = time.perf_counter() - t0
            # the loader of data_utils.py:135, except that the shuffled epoch is long enough for the timed batches (the
            # synthetic Weizmann tree has 180 entries); each item costs the same __getitem__ either way
            sampler = RandomSampler(ds, replacement=True, num_samples=B * (args.batches + 1))
            it = iter(DataLoader(ds, batch_size=B, sampler=sampler, drop_last=True, num_workers=1))
            next(it)
            t0 = time.perf_counter()
            for _ in range(args.batches):
                x = next(it)
            dt = (time.perf_counter() - t0) / args.batches
            assert tuple(x.shape) == (B, T, 3, S, S)
            print(json.dumps(dict(metric="reference_cpu_loader", dataset=name, B=B, T=T, batches=args.batches,
                                  dataset_init_s=round(init_s, 1), ms_per_batch=round(dt * 1e3, 1), frames_per_s=round(T * B / dt),
                                  cpu=cpu_model(), cores=os.cpu_count(), usable_cores=len(os.sched_getaffinity(0)),
                                  torch_threads=torch.get_num_threads())), flush=True)


def main():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="mode", required=True)
    g = sub.add_parser("gpu")
    g.add_argument("--launches", type=int, default=300)
    g.add_argument("--steps", type=int, default=10)
    g.add_argument("--rounds", type=int, default=3)
    g.add_argument("--load-trajectories", type=int, default=256)
    c = sub.add_parser("cpu-reference")
    c.add_argument("--ref", default=os.environ.get("P2PVG_REF", ""))
    c.add_argument("--batches", type=int, default=3)
    args = ap.parse_args()
    if args.mode == "gpu":
        run_gpu(args)
    else:
        if not os.path.isfile(os.path.join(args.ref, "data", "weizmann.py")):
            raise SystemExit("--ref must name the reference checkout")
        run_cpu_reference(args)


if __name__ == "__main__":
    main()
