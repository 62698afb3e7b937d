#!/usr/bin/env python
"""Moving MNIST input path: GPU-rendered batches (p2pvg_moving_mnist) against the reference's CPU loader.

    python tools/bench_moving_mnist.py gpu [--launches 300] [--steps 20] [--rounds 3]
    python tools/bench_moving_mnist.py cpu-reference --ref /path/to/p2pvg [--batches 4]

gpu: prints the card name, power limit and SM clock, then one JSON line each for
  kernel  p2pvg_moving_mnist at the C2 batch (T = 30, B = 256, 64x64, 2 digits): CUDA events around --launches launches after
          warm-up, and the frame bytes it writes per launch over that time; plus the host-clocked cost of one MovingMNIST batch
          (draws + allocation + launch, ending in a synchronise)
  e2e     train-step frames/s of the C2 step (dcgan_64, bf16, CUDA graph) fed by MovingMNIST (`x = next(mm); model(x, 0, T-1)`)
          and the same loop on one resident batch, alternated --rounds times (median per loop); host clock around --steps
          steps ending in a synchronise.
cpu-reference: the reference's own DynamicLengthMovingMNIST.__getitem__ through DataLoader(batch_size=256, num_workers=1), as
  data/data_utils.py:135 builds it, with MNIST faked in memory (28x28 uint8 digits, transform Resize(32) + ToTensor, i.e. the
  PIL resize per digit the reference's Scale(32) does); first batch (worker start) excluded.  Prints the host's CPU model and
  core count with the rate."""
import argparse
import importlib.util
import json
import os
import statistics
import subprocess
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
T, B, S, ND = 30, 256, 64, 2


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def synthetic_digits(n=60000):
    return torch.randint(0, 256, (n, 32, 32), dtype=torch.uint8, generator=torch.Generator().manual_seed(0))


def run_gpu(args):
    from p2pvg_b200._lib import kernels_for
    from p2pvg_b200.data import MovingMNIST
    from p2pvg_b200.models import dcgan_64
    from p2pvg_b200.models.p2p_model import P2PModel
    if not torch.cuda.is_available():
        raise SystemExit("gpu mode needs a CUDA device")
    print("card:", card(), flush=True)
    K = kernels_for("cuda")
    digits = synthetic_digits().cuda()
    gen = torch.Generator("cuda").manual_seed(0)
    draws = torch.randint(0, 2 ** 31 - 1, (B, ND, 5 + 4 * T), dtype=torch.int32, device="cuda", generator=gen)
    out = torch.empty(T, B, 1, S, S, device="cuda")
    for _ in range(20):
        K.moving_mnist(digits, draws, out, T, B, S, ND, False)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(args.launches):
        K.moving_mnist(digits, draws, out, T, B, S, ND, False)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) / args.launches * 1e3
    nbytes = out.numel() * 4   # the frames; draws and digits read are < 0.3% of it
    mm = MovingMNIST(digits, B, T, 0, image_size=S, num_digits=ND, generator=gen)
    for _ in range(5):
        next(mm)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(50):
        next(mm)
    torch.cuda.synchronize()
    batch_us = (time.perf_counter() - t0) / 50 * 1e6
    print(json.dumps(dict(metric="moving_mnist_kernel", T=T, B=B, S=S, num_digits=ND, kernel_us=round(us, 2),
                          write_bytes=nbytes, write_GBps=round(nbytes / (us * 1e-6) / 1e9, 1),
                          movingmnist_batch_us=round(batch_us, 1))), flush=True)

    os.environ["P2PVG_PRECISION"] = "bf16"
    os.environ["P2PVG_GRAPH"] = "1"
    opt = types.SimpleNamespace(dataset="mnist", backbone_net=dcgan_64, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0,
                                weight_align=0.5, skip_prob=0.0, n_past=1, last_frame_skip=False, batch_size=B)
    torch.manual_seed(1)
    np.random.seed(0)
    model = P2PModel(B, 1, 128, 10, 256, 1, 1, 2, opt=opt).cuda()
    model.train()
    resident = next(mm)

    def loop(rendered, n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n):
            x = next(mm) if rendered else resident
            model(x, 0, len(x) - 1)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    loop(True, 4)
    loop(False, 4)
    res = {True: [], False: []}
    for _ in range(args.rounds):
        for rendered in (True, False):
            res[rendered].append(T * B * args.steps / loop(rendered, args.steps))
    fps = {k: statistics.median(v) for k, v in res.items()}
    print(json.dumps(dict(metric="moving_mnist_e2e", T=T, B=B, steps=args.steps, rounds=args.rounds,
                          frames_per_s_rendered=round(fps[True]), frames_per_s_resident=round(fps[False]),
                          ms_per_step_rendered=round(T * B / fps[True] * 1e3, 2), ms_per_step_resident=round(T * B / fps[False] * 1e3, 2),
                          all_rendered=[round(v) for v in res[True]], all_resident=[round(v) for v in res[False]])), flush=True)


def cpu_model():
    try:
        with open("/proc/cpuinfo") as f:
            return next(l.split(":", 1)[1].strip() for l in f if l.startswith("model name"))
    except (OSError, StopIteration):
        return "unknown"


def run_cpu_reference(args):
    from PIL import Image
    from torch.utils.data import DataLoader
    from torchvision import transforms
    spec = importlib.util.spec_from_file_location("ref_moving_mnist", os.path.join(args.ref, "data", "moving_mnist.py"))
    mm = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mm)
    raw = np.random.RandomState(0).randint(0, 256, (1000, 28, 28)).astype(np.uint8)

    class FakeMNIST:   # in memory; the real dataset (download=True) is never constructed
        def __init__(self, root, train=True, download=False, transform=None):
            self.transform = transform

        def __len__(self):
            return 60000

        def __getitem__(self, i):
            return self.transform(Image.fromarray(raw[i % len(raw)])), 0

    mm.datasets.MNIST = FakeMNIST
    ds = mm.DynamicLengthMovingMNIST(data_root="unused", train=True, max_seq_len=T, delta_len=5, image_size=S, num_digits=ND,
                                     deterministic=False, transform=transforms.Compose([transforms.Resize(32), transforms.ToTensor()]))
    loader = DataLoader(ds, batch_size=B, shuffle=True, drop_last=True, num_workers=1)
    it = iter(loader)
    next(it)
    t0 = time.perf_counter()
    for _ in range(args.batches):
        x = next(it)
    dt = (time.perf_counter() - t0) / args.batches
    assert tuple(x.shape) == (B, T, 1, S, S)
    print(json.dumps(dict(metric="reference_cpu_loader", T=T, B=B, S=S, num_digits=ND, batches=args.batches,
                          ms_per_batch=round(dt * 1e3, 1), sequences_per_s=round(B / dt, 1), frames_per_s=round(T * B / dt),
                          cpu=cpu_model(), cores=os.cpu_count(), usable_cores=len(os.sched_getaffinity(0)),
                          torch_threads=torch.get_num_threads())), flush=True)


def main():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="mode", required=True)
    g = sub.add_parser("gpu")
    g.add_argument("--launches", type=int, default=300)
    g.add_argument("--steps", type=int, default=20)
    g.add_argument("--rounds", type=int, default=3)
    c = sub.add_parser("cpu-reference")
    c.add_argument("--ref", default=os.environ.get("P2PVG_REF", ""))
    c.add_argument("--batches", type=int, default=4)
    args = ap.parse_args()
    if args.mode == "gpu":
        run_gpu(args)
    else:
        if not os.path.isfile(os.path.join(args.ref, "data", "moving_mnist.py")):
            raise SystemExit("--ref must name the reference checkout")
        run_cpu_reference(args)


if __name__ == "__main__":
    main()
