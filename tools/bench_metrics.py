#!/usr/bin/env python
"""Scoring generated videos on the GPU (p2pvg_frame_metrics, P2PModel.p2p_evaluate) at the scoring shapes of
tools/bench_generate.py:

  (b) misc/visualize.py:135    dcgan_64, C=1, B=100, 30 frames, 20 samples: 58,000 scored 64x64x1 pairs
  (g) misc/visualize.py:135    vgg_64,   C=3, B=128, 30 frames, 20 samples: 74,240 scored 64x64x3 pairs

  kernel    CUDA events around --launches back-to-back launches on the pairs p2p_evaluate scores (metrics.plan_pairs, the
            samples of one ground-truth frame adjacent), after warm-up; median and spread of --reps windows.  Achieved
            bytes/s under two byte models -- every pair reads both its frames (pred + gt per pair), and every byte is read
            from HBM once (pred + distinct gt) -- against the 3.35 TB/s HBM3 data-sheet rate.
  evaluate  p2p_evaluate against p2p_generate_graphed with the same arguments (bf16, randomly initialised weights), alternated,
            host clock around calls that end in a device synchronise, median of --reps; the difference is the scoring's
            cost per call.  p2p_generate_graphed also copies its frames out of graph memory, which p2p_evaluate does not,
            so the kernel time over the generate call is given beside the difference.

Prints the card name, power limit and maximum SM clock, then one JSON line per workload."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_generate import make_model  # noqa: E402
from p2pvg_b200 import metrics  # noqa: E402

HBM_TBS = 3.35
WORKLOADS = (("b_vis_seq", 64, 1, 100, 20), ("g_vgg64_vis_seq", "vgg64", 3, 128, 20))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def kernel_ms(pred, gt, pairs, launches, reps):
    shape = tuple(pred.shape[1:])
    for _ in range(5):
        metrics.launch_frame_metrics(pred, gt, pairs, shape, 1.0)
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(launches):
            metrics.launch_frame_metrics(pred, gt, pairs, shape, 1.0)
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) / launches)
    return ts


def host_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    info = card()
    print("card (name, power limit, max SM clock):", info, flush=True)
    T = L = 30
    lines = []
    for name, width, C, B, ns in WORKLOADS:
        side = 64
        n_past = 1
        frames, pairs = metrics.plan_pairs(L, T, n_past, ns, B)
        pairs = pairs.cuda()
        gen = torch.Generator(device="cuda").manual_seed(1)
        fbytes = C * side * side * 4
        pred = torch.rand((L - n_past) * ns * B, C, side, side, device="cuda", generator=gen)
        gt = torch.rand(T * B, C, side, side, device="cuda", generator=gen)
        ts = kernel_ms(pred, gt, pairs, args.launches, args.reps)
        ms = statistics.median(ts)
        n = len(pairs)
        per_pair = 2 * n * fbytes
        distinct = pred.numel() * 4 + len(frames) * B * fbytes
        floor_ms = distinct / (HBM_TBS * 1e12) * 1e3
        res = dict(workload=name, channels=C, side=side, B=B, samples=ns, pairs=n, card=info,
                   kernel=dict(ms=round(ms, 4), spread_ms=round(max(ts) - min(ts), 4), launches_per_window=args.launches,
                               bytes_pred_plus_gt_per_pair=per_pair, tbs_pred_plus_gt_per_pair=round(per_pair / ms / 1e9, 3),
                               bytes_pred_plus_distinct_gt=distinct, tbs_pred_plus_distinct_gt=round(distinct / ms / 1e9, 3),
                               hbm_floor_ms=round(floor_ms, 4), share_of_hbm_bound=round(floor_ms / ms, 3)))
        del pred, gt
        torch.cuda.empty_cache()
        # p2p_evaluate against p2p_generate_graphed, same arguments, alternated
        model = make_model(width, C, B)
        x = torch.rand(T, B, C, side, side, device="cuda", generator=gen)
        xs = list(x)
        ev = lambda: model.p2p_evaluate(xs, nsample=ns)                    # noqa: E731
        gr = lambda: model.p2p_generate_graphed(xs, L, L - 1, nsample=ns)  # noqa: E731
        for fn in (ev, gr, ev, gr):   # warm-up: capture, module loads
            fn()
        te, tg = [], []
        for _ in range(args.reps):
            te.append(host_ms(ev))
            tg.append(host_ms(gr))
        me, mg = statistics.median(te), statistics.median(tg)
        res["evaluate"] = dict(p2p_evaluate_ms=round(me, 3), p2p_generate_graphed_ms=round(mg, 3), scoring_ms=round(me - mg, 3),
                               scoring_share=round((me - mg) / mg, 4),
                               kernel_share_of_generate=round(ms / mg, 4), spread_evaluate_ms=round(max(te) - min(te), 3),
                               spread_generate_ms=round(max(tg) - min(tg), 3))
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
