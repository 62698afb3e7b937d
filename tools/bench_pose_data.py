#!/usr/bin/env python
"""Human3.6M input path: batches gathered on the GPU from device-resident pose stores (p2pvg_pose_windows) against the
reference's CPU loader.

    python tools/bench_pose_data.py gpu [--launches 300] [--steps 20] [--rounds 3]
    python tools/bench_pose_data.py cpu-reference --ref /path/to/p2pvg [--epochs 3]

gpu: prints the card name, power limit and SM clock, then one JSON line each for
  kernel  p2pvg_pose_windows at B = 256 and B = 22 (T = 30, J = 17, train speed 6): CUDA events around one CUDA-graph replay
          of --launches launches (after 20 eager warm-up launches), and the fp32 bytes written per launch over that time;
          the same events around --launches eager launches, which the Python call paces; the host-clocked cost of one
          PoseBatches next() (T draw, draws, two allocations, launch; a permutation upload per epoch), ending in a synchronise
  e2e     a C5-shaped train step (h36m_mlp, rnn_size 512, B = 256, T = 30, bf16, CUDA graph) fed by PoseBatches
          (`x = next(it); model(x, 0, len(x[1]) - 1)`) and the same loop on one resident batch, alternated --rounds times
          (median per loop); host clock around --steps steps ending in a synchronise
  The store is synthetic: 1200 sequences of 200..400 frames.
cpu-reference: the reference's unmodified Human36mDataset.__getitem__ through DataLoader(shuffle=True, drop_last=True,
  num_workers=1) as data/data_utils.py builds it, iterated epoch after epoch as get_h36m_generator does (a new worker each
  epoch, included), with its main-process .permute(1, 0, 2, 3).float() of both pose tensors (not .cuda(): the host has no
  GPU).  The dataset holds synthetic normalised float64 sequences of 1000..3000 frames, set directly instead of through
  __init__ (which only reads annot.h5 and normalises): 150 entries at B = 22, 1200 at B = 256.  h5py and matplotlib are
  stubbed, since only __init__ and the visualiser use them.  Prints the host's CPU model and core count with the rate."""
import argparse
import importlib
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
J, L, SPEED = 17, 30, 6


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


def synthetic_clips(n, device):
    from p2pvg_b200.data import PoseClips
    g = torch.Generator().manual_seed(0)
    lens = torch.randint(200, 401, (n,), generator=g).tolist()
    p2 = [3 * torch.randn(k, J, 2, generator=g).numpy() for k in lens]
    p3 = [3 * torch.randn(k, J, 3, generator=g).numpy() for k in lens]
    return PoseClips(p2, p3, [0, 1, 2, 3] * n, L, SPEED, device=device)


def time_kernel(K, clips, B, T, launches, gen):
    entries = torch.randint(0, len(clips), (B,), dtype=torch.int32, device="cuda", generator=gen)
    draws = torch.randint(0, 2 ** 31 - 1, (2, B), dtype=torch.int32, device="cuda", generator=gen)
    out_2d = torch.empty(T, B, J, 2, device="cuda")
    out_3d = torch.empty(T, B, J, 3, device="cuda")

    def launch():
        K.pose_windows(clips.pose_2d, clips.pose_3d, clips.seq_first, clips.seq_len, entries, draws, (SPEED, SPEED), L, out_2d,
                       out_3d)
    for _ in range(20):
        launch()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(launches):
        launch()
    e1.record()
    torch.cuda.synchronize()
    eager_us = e0.elapsed_time(e1) / launches * 1e3
    # the eager loop is paced by the Python call (argument checks + ctypes), not by the kernel: replay the same launches
    # from a CUDA graph to time the kernel itself
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(launches):
            launch()
    graph.replay()
    torch.cuda.synchronize()
    e0.record()
    graph.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / launches * 1e3, eager_us, (out_2d.numel() + out_3d.numel()) * 4


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
    from p2pvg_b200.data import PoseBatches
    from p2pvg_b200.models import h36m_mlp
    from p2pvg_b200.models.p2p_model import P2PModel
    if not torch.cuda.is_available():
        raise SystemExit("gpu mode needs a CUDA device")
    print("card:", card(), flush=True)
    K = kernels_for("cuda")
    gen = torch.Generator("cuda").manual_seed(0)
    clips = synthetic_clips(1200, "cuda")
    for B in (256, 22):
        us, eager_us, nbytes = time_kernel(K, clips, B, L, args.launches, gen)
        next_us = time_next(PoseBatches(clips, B, (L, L), (SPEED, SPEED), generator=gen))
        print(json.dumps(dict(metric="pose_windows_kernel", B=B, T=L, J=J, speed=SPEED, kernel_us=round(us, 2), write_bytes=nbytes,
                              write_GBps=round(nbytes / (us * 1e-6) / 1e9, 1), eager_launch_us=round(eager_us, 2),
                              posebatches_next_us=round(next_us, 1))), flush=True)

    os.environ["P2PVG_PRECISION"] = "bf16"
    os.environ["P2PVG_GRAPH"] = "1"
    B = 256
    opt = types.SimpleNamespace(dataset="h36m", backbone_net=h36m_mlp, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0,
                                weight_align=0.5, skip_prob=0.0, n_past=1, last_frame_skip=False, batch_size=B)
    torch.manual_seed(1)
    np.random.seed(0)
    model = P2PModel(B, 1, 128, 10, 512, 1, 1, 2, opt=opt).cuda()
    model.train()
    it = PoseBatches(clips, B, (L, L), (SPEED, SPEED), generator=gen)   # T fixed: one graph, comparable steps
    resident = next(it)

    def loop(fed, n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n):
            x = next(it) if fed else resident
            model(x, 0, len(x[1]) - 1)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    loop(True, 4)
    loop(False, 4)
    res = {True: [], False: []}
    for _ in range(args.rounds):
        for fed in (True, False):
            res[fed].append(args.steps / loop(fed, args.steps))
    sps = {k: statistics.median(v) for k, v in res.items()}
    print(json.dumps(dict(metric="pose_e2e_c5_shape", T=L, B=B, rnn_size=512, steps=args.steps, rounds=args.rounds,
                          ms_per_step_posebatches=round(1e3 / sps[True], 3), ms_per_step_resident=round(1e3 / sps[False], 3),
                          all_ms_posebatches=[round(1e3 / v, 3) for v in res[True]],
                          all_ms_resident=[round(1e3 / v, 3) for v in res[False]])), flush=True)


def run_cpu_reference(args):
    from torch.utils.data import DataLoader
    from tests import pose_tree
    sys.modules.update(pose_tree.stub_modules())
    sys.path.insert(0, os.path.join(args.ref, "data", "human36m"))
    h36m = importlib.import_module("human36m")
    for B, n in ((22, 150), (256, 1200)):
        rs = np.random.RandomState(0)
        lens = rs.randint(1000, 3001, n)
        ds = h36m.Human36mDataset.__new__(h36m.Human36mDataset)
        ds.max_seq_len, ds.delta_len, ds.speed_range, ds.n_breakpoints, ds.acc_range = L, 5, [SPEED, SPEED], 0, [0, 0]
        ds.data = {"pose": {"2d": [3 * rs.randn(k, J, 2) for k in lens], "3d": [3 * rs.randn(k, J, 3) for k in lens]},
                   "camera_view": [0, 1, 2, 3] * n}
        loader = DataLoader(ds, batch_size=B, shuffle=True, drop_last=True, num_workers=1)
        batches = 0
        t0 = time.perf_counter()
        for _ in range(args.epochs):
            for data in loader:
                ds.get_seq_len()
                x2 = data["pose_2d"].permute(1, 0, 2, 3).float()
                x3 = data["pose_3d"].permute(1, 0, 2, 3).float()
                batches += 1
        dt = (time.perf_counter() - t0) / batches
        assert tuple(x3.shape) == (L, B, J, 3) and tuple(x2.shape) == (L, B, J, 2)
        print(json.dumps(dict(metric="reference_cpu_loader", B=B, entries=n, epochs=args.epochs, batches=batches,
                              ms_per_batch=round(dt * 1e3, 1), cpu=cpu_model(), cores=os.cpu_count(),
                              usable_cores=len(os.sched_getaffinity(0)), torch_threads=torch.get_num_threads())), flush=True)


def main():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="mode", required=True)
    g = sub.add_parser("gpu")
    g.add_argument("--launches", type=int, default=300)
    g.add_argument("--steps", type=int, default=20)
    g.add_argument("--rounds", type=int, default=3)
    c = sub.add_parser("cpu-reference")
    c.add_argument("--ref", default=os.environ.get("P2PVG_REF", ""))
    c.add_argument("--epochs", type=int, default=3)
    args = ap.parse_args()
    if args.mode == "gpu":
        run_gpu(args)
    else:
        if not os.path.isfile(os.path.join(args.ref, "data", "human36m", "human36m.py")):
            raise SystemExit("--ref must name the reference checkout")
        run_cpu_reference(args)


if __name__ == "__main__":
    main()
