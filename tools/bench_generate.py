#!/usr/bin/env python
"""Eager p2p_generate / p2p_generate_samples against the graph-replayed p2p_generate_graphed on the calls the reference's
callers make (dcgan backbones, eval-mode BatchNorm, randomly initialised weights, skip_frame=False):

  (a) generate.py:115-116      dcgan_64,  C=1, B=1,   30 frames, 5 samples   eager: 5 looped calls     graphed: nsample=5
  (b) misc/visualize.py:135    dcgan_64,  C=1, B=100, 30 frames, 20 samples  eager: 20 looped calls and p2p_generate_samples
                                                                             graphed: 20 looped calls and nsample=20
  (c)                          dcgan_128, C=3, B=64,  30 frames, 1 sample
  (d) misc/visualize.py:135    h36m_mlp, rnn_size 512, B=10, 30 frames, 20 samples   (as (b))
  (e) generate.py:115-116      h36m_mlp, rnn_size 512, B=1,  30 frames, 5 samples    (as (a))
  (f) generate.py:115-116      vgg_64,   C=3, B=1,   30 frames, 5 samples   (as (a))
  (g) misc/visualize.py:135    vgg_64,   C=3, B=128, 30 frames, 20 samples  (as (b); the C3 training batch)
  (h)                          vgg_128,  C=3, B=16,  30 frames, 1 sample

The pose workloads (d) / (e) run exact fp32 in both P2PVG_PRECISION modes and use the fp32 parity bound.  Each JSON line also gives the graph buffers' device memory (GenerateEngine.memory_bytes()) of
one looped call's and one nsample call's signature, each cached alone.

Eager and graphed calls alternate; every time is a host clock around calls that end in a device synchronise (median of
--reps).  Before timing, each pair of paths is fed the same eps draws and compared at the timed size.  Prints the card
name, power limit and SM clock, then one JSON line per workload."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from p2pvg_b200.infer import eps_stream  # noqa: E402
from p2pvg_b200.models import dcgan_64, dcgan_128, h36m_mlp, vgg_64, vgg_128  # noqa: E402
from p2pvg_b200.models.p2p_model import P2PModel  # noqa: E402

TOL = {"fp32": (2e-4, 2e-5), "bf16": (4e-2, 6e-3), "pose": (3e-4, 3e-5)}
WORKLOADS = (("a_generate_py", 64, 1, 1, 5), ("b_vis_seq", 64, 1, 100, 20), ("c_d128_rgb", 128, 3, 64, 1),
             ("d_pose_vis_seq", "pose", 0, 10, 20), ("e_pose_generate_py", "pose", 0, 1, 5),
             ("f_vgg64_generate_py", "vgg64", 3, 1, 5), ("g_vgg64_vis_seq", "vgg64", 3, 128, 20), ("h_vgg128_rgb", "vgg128", 3, 16, 1))
SIDE = {"vgg64": 64, "vgg128": 128}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def make_model(width, C, B):
    pose = width == "pose"
    net = h36m_mlp if pose else {64: dcgan_64, 128: dcgan_128, "vgg64": vgg_64, "vgg128": vgg_128}[width]
    opt = types.SimpleNamespace(dataset="h36m" if pose else "mnist", backbone_net=net, lr=1e-3, beta1=0.9, beta=1e-4,
                                weight_cpc=100.0, weight_align=0.5, skip_prob=0.5, n_past=1, last_frame_skip=False, batch_size=B)
    torch.manual_seed(1)
    return P2PModel(B, max(C, 1), 128, 10, 512 if pose else 256, 1, 1, 2, opt=opt).cuda().eval()


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


def flat(res):
    if isinstance(res[0], list):
        return [f for s in res for f in s]
    return res


def check(eager, graphed, rows, n_steps, prec):
    """Both paths fed the same draws (the eager samples path and nsample>1 consume [nsample*B, z] per draw)."""
    g = torch.Generator().manual_seed(7)
    draws = [torch.randn(rows, 10, generator=g) for _ in range(2 * n_steps)]
    out = []
    for fn in (eager, graphed):
        np.random.seed(3)
        with eps_stream(list(draws)):
            out.append([f.float().cpu() for f in flat(fn())])
    tmax, tmean = TOL[prec]
    worst = max((a - b).abs().max().item() for a, b in zip(*out))
    mean = max((a - b).abs().mean().item() for a, b in zip(*out))
    return dict(max_err=worst, mean_err=mean, within_tol=bool(worst <= tmax and mean <= tmean))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    ap.add_argument("--only", default="abcde", help="workload letters to run")
    args = ap.parse_args()
    prec = os.environ.get("P2PVG_PRECISION", "bf16")
    info = card()
    print("card (name, power limit, SM clock, max SM clock):", info, "| precision", prec, flush=True)
    T = L = 30
    cp = L - 1
    lines = []
    for name, width, C, B, ns in WORKLOADS:
        if name[0] not in args.only:
            continue
        model = make_model(width, C, B)
        gen = torch.Generator(device="cuda").manual_seed(2)
        if width == "pose":   # poses standardised to std 3 (the h36m loader)
            x = 3 * torch.randn(T, B, 17, 3, device="cuda", generator=gen)
        else:
            side = SIDE.get(width, width)
            x = torch.rand(T, B, C, side, side, device="cuda", generator=gen)
        tol = "pose" if width == "pose" else prec
        xs = list(x)
        steps = L - 1   # skip_frame=False: every step executes
        variants = {
            "eager_looped": lambda: [model.p2p_generate(xs, L, cp) for _ in range(ns)],
            "graphed_looped": lambda: [model.p2p_generate_graphed(xs, L, cp) for _ in range(ns)],
        }
        if ns > 1:
            variants["eager_samples"] = lambda: model.p2p_generate_samples(xs, ns, L, cp)
            variants["graphed_nsample"] = lambda: model.p2p_generate_graphed(xs, L, cp, nsample=ns)
        parity = {"looped_call": check(lambda: model.p2p_generate(xs, L, cp), lambda: model.p2p_generate_graphed(xs, L, cp),
                                       B, steps, tol)}
        if ns > 1:
            parity["nsample"] = check(lambda: model.p2p_generate_samples(xs, ns, L, cp),
                                      lambda: model.p2p_generate_graphed(xs, L, cp, nsample=ns), ns * B, steps, tol)
        for fn in variants.values():   # warm-up: module loads, graph capture
            fn()
        times = {k: [] for k in variants}
        for _ in range(args.reps):     # alternate the paths
            for k, fn in variants.items():
                times[k].append(timed(fn, 1))
        eng = model._gen_engine
        memory = {}
        for k, fn in (("looped_call", lambda: model.p2p_generate_graphed(xs, L, cp)),
                      ("nsample", lambda: model.p2p_generate_graphed(xs, L, cp, nsample=ns))):
            if k == "nsample" and ns == 1:
                continue
            eng.clear()
            fn()
            memory[k] = eng.memory_bytes()
        frames = ns * B * (L - 1)
        res = dict(workload=name, image_width=width, channels=C, B=B, samples=ns, len_output=L, precision=prec, card=info,
                   parity=parity, graph_memory_bytes=memory)
        for k, ts in times.items():
            ms = statistics.median(ts)
            calls = ns if k.endswith("looped") else 1
            res[k] = dict(ms_per_workload=round(ms, 3), ms_per_call=round(ms / calls, 3), frames_per_s=round(frames / ms * 1e3, 1),
                          ms_per_step=round(ms / calls / steps, 4), spread_ms=round(max(ts) - min(ts), 3))
        line = json.dumps(res)
        print(line, flush=True)
        lines.append(line)
        del model
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
