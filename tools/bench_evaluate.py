#!/usr/bin/env python
"""Split-level evaluation (p2pvg_b200.evaluate.evaluate_split) against the per-batch alternatives, on randomly initialised
weights in eval mode (the default P2PVG_PRECISION), T = 30, lengths 10, 20 and 30, nsample 20:
  split     one evaluate_split step: one p2p_evaluate_lengths replay, one metrics launch, one p2pvg_metrics_fold launch,
            and the report's read-back
  looped    p2p_evaluate(x, 20, len_output=L) for each length: one replay and one metrics launch per length
  eager     the reference's way: p2p_generate per sample and length (60 eager calls) scored on the host by the float64
            NumPy restatement tests/metrics_ref.py, best sample per row chosen on the host
Workloads: dcgan_64 with 1 channel (Moving MNIST shape) at B = 100, vgg_64 with 3 channels at B = 128.  The eager loop
scores 60 * B * 30 frame pairs one by one on the host (about 5 ms per 1-channel and 13 ms per 3-channel 64 x 64 pair), so it
is timed once, at B = 4, beside split and looped at the same B = 4.  Also: the wall time of a 50-batch split (dcgan_64,
B = 100; five distinct batches cycled) and the device time of p2pvg_metrics_fold from torch.profiler in a run of its own.
Every time is a host clock around work that ends in a device synchronise, after one warm-up call of each variant (graph
capture); variants alternate, and the median and spread (min..max) of --reps are reported.  Prints the card name, power
limit and SM clocks, then one JSON line per row."""
import argparse
import itertools
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
from p2pvg_b200 import evaluate  # noqa: E402
from p2pvg_b200.models import dcgan_64, vgg_64  # noqa: E402
from p2pvg_b200.models.p2p_model import P2PModel  # noqa: E402
from tests import metrics_ref as R  # noqa: E402

LENS, NS, T = [10, 20, 30], 20, 30


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def make(net, C, B, seed=2):
    opt = types.SimpleNamespace(dataset="mnist", backbone_net=net, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0,
                                weight_align=0.5, skip_prob=0.5, n_past=1, last_frame_skip=False, batch_size=B)
    torch.manual_seed(1)
    model = P2PModel(B, C, 128, 10, 256, 1, 1, 2, opt=opt).cuda().eval()
    return model, clip(C, B, seed)


def clip(C, B, seed):
    return torch.rand(T, B, C, 64, 64, generator=torch.Generator().manual_seed(seed)).cuda()


def host_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def eager(model, x):
    """The reference's loop: one eager p2p_generate per sample and length, scored pair by pair on the host."""
    n_past = int(model.opt.n_past)
    out = []
    for L in LENS:
        seqs = [model.p2p_generate(x, L, L - 1) for _ in range(NS)]
        frames = list(range(n_past, L)) if L == len(x) else [L - 1]
        gts = frames if L == len(x) else [len(x) - 1]
        xs = x.double().cpu().numpy()
        sc = np.array([[[R.frame_scores(seqs[s][f][b].double().cpu().numpy(), xs[t][b]) for b in range(x.shape[1])]
                        for f, t in zip(frames, gts)] for s in range(NS)])            # [NS, F, B, 3]
        best = sc.mean(1).argmax(0)                                                  # per row and metric (mse lower below)
        best[:, 0] = sc[..., 0].mean(1).argmin(0)
        out.append((sc, best))
    return out


def timed(variants, reps):
    for fn in variants.values():
        fn()
    ts = {k: [] for k in variants}
    for _ in range(reps):
        for k, fn in variants.items():
            ts[k].append(host_ms(fn))
    return {k: {"median_ms": round(statistics.median(v), 3), "min_ms": round(min(v), 3), "max_ms": round(max(v), 3)}
            for k, v in ts.items()}


def fold_device_us(model, x, n=50):
    """Device time of one p2pvg_metrics_fold launch on the workload's scores, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    (frames, offsets, B), scores, names = model._graphed_engine().score_lengths(x, LENS, NS)
    tot = evaluate.SplitTotals(names, x.device)
    tot.fold(scores, LENS, T, frames, offsets, B, NS)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            tot.fold(scores, LENS, T, frames, offsets, B, NS)
        torch.cuda.synchronize()
    ev = [e for e in prof.key_averages() if "metrics_fold" in e.key]
    total = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) for e in ev)
    count = sum(e.count for e in ev)
    return round(total / max(count, 1), 2), count, int(scores.shape[0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--skip_eager", action="store_true")
    args = ap.parse_args()
    print("card:", card(), flush=True)
    for name, net, C, B in (("dcgan_64 C1", dcgan_64, 1, 100), ("vgg_64 C3", vgg_64, 3, 128)):
        model, x = make(net, C, B)
        base = {"T": T, "len_outputs": LENS, "nsample": NS, "reps": args.reps}
        row = dict(workload=name, B=B, **base, **timed({
            "split": lambda: evaluate.evaluate_split(model, [x], 1, LENS, NS),
            "looped": lambda: [model.p2p_evaluate(x, NS, len_output=L) for L in LENS]}, args.reps))
        row["split_speedup_vs_looped"] = round(row["looped"]["median_ms"] / row["split"]["median_ms"], 2)
        print(json.dumps(row), flush=True)
        if name.startswith("dcgan"):
            us, count, n_pairs = fold_device_us(model, x)
            print(json.dumps({"workload": name, "B": B, "kernel": "p2pvg_metrics_fold", "pairs": n_pairs, "launches": count,
                              "device_us_per_launch": us}), flush=True)
            batches = [x] + [clip(C, B, seed) for seed in range(3, 7)]
            reps = max(args.reps // 2, 1)
            row = dict(workload=name + " 50-batch split", B=B, **dict(base, reps=reps), batches=50, **timed({
                "split": lambda: evaluate.evaluate_split(model, itertools.islice(itertools.cycle(batches), 50), 50, LENS, NS)},
                reps))
            print(json.dumps(row), flush=True)
            del batches
        if not args.skip_eager:
            model._graphed_engine().clear()   # the B = 4 signatures would otherwise evict these graphs on every call
            torch.cuda.empty_cache()
            xs = x[:, :4].contiguous()
            row = dict(workload=name, B=4, **base, **timed({
                "split": lambda: evaluate.evaluate_split(model, [xs], 1, LENS, NS),
                "looped": lambda: [model.p2p_evaluate(xs, NS, len_output=L) for L in LENS]}, args.reps))
            t = host_ms(lambda: eager(model, xs))
            row["eager"] = {"single_run_ms": round(t, 1)}
            row["split_speedup_vs_eager"] = round(t / row["split"]["median_ms"], 1)
            print(json.dumps(row), flush=True)
        del model, x
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
