#!/usr/bin/env python
"""Generation through control points: eager p2p_generate and the graph-replayed p2p_generate_graphed, each chained by hand
over the segments (init_hidden=False after the first), against p2p_generate_multi_cp (the whole chain as one replay).
Every workload chains 4 segments of 8 frames (cp_ixs = [0, 7, 14, 21, 28], the clip's timing, skip_frame=False) with
randomly initialised weights and eval-mode BatchNorm:

  (a) misc/visualize.py:135 size   dcgan_64, C=1, B=100, 20 samples
  (b) generate.py:115-116 size     dcgan_64, C=1, B=1,   5 samples
  (c)                              vgg_64,   C=3, B=1,   1 sample
  (d)                              h36m_mlp, rnn_size 512, B=10, 1 sample

Paths: eager_looped (per sample, the segments' p2p_generate calls), graphed_looped (the segments' p2p_generate_graphed
calls with nsample), chain (one p2p_generate_multi_cp call with nsample).  Before timing, the chain is compared with the
looped graphed calls (same draws, nsample as timed) and with the eager calls (one sample).  The paths alternate; every time
is a host clock around calls that end in a device synchronise (median and spread of --reps).  Prints the card name, power
limit and SM clock, then one JSON line per workload."""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from p2pvg_b200.infer import eps_stream  # noqa: E402
from tools.bench_generate import card, make_model, timed  # noqa: E402

TOL = {"fp32": (2e-4, 2e-5), "bf16": (4e-2, 6e-3), "pose": (3e-4, 3e-5)}
WORKLOADS = (("a_d64_vis_seq", 64, 1, 100, 20), ("b_d64_generate_py", 64, 1, 1, 5), ("c_vgg64_rgb", "vgg64", 3, 1, 1),
             ("d_pose", "pose", 0, 10, 1))
SIDE = {"vgg64": 64}
CPS = [0, 7, 14, 21, 28]


def segments(x):
    return [x[a:b + 1] for a, b in zip(CPS, CPS[1:])]


def chained(gen, segs, **kw):
    return [gen(s, len(s), len(s) - 1, init_hidden=k == 0, **kw) for k, s in enumerate(segs)]


def flat(res, ns):
    """Frames of a chain result in (segment, sample, frame) order."""
    return [f for seg in res for seq in ([seg] if ns == 1 else seg) for f in seq]


def compare(a_fn, b_fn, rows, n_steps, ns, tol):
    g = torch.Generator().manual_seed(7)
    draws = [torch.randn(rows, 10, generator=g) for _ in range(2 * n_steps)]
    out = []
    for fn in (a_fn, b_fn):
        np.random.seed(3)
        with eps_stream(list(draws)):
            out.append([f.float().cpu() for f in flat(fn(), ns)])
    tmax, tmean = TOL[tol]
    worst = max((a - b).abs().max().item() for a, b in zip(*out))
    mean = max((a - b).abs().mean().item() for a, b in zip(*out))
    return dict(max_err=worst, mean_err=mean, within_tol=bool(len(out[0]) == len(out[1]) and worst <= tmax and mean <= tmean))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    ap.add_argument("--only", default="abcd", help="workload letters to run")
    args = ap.parse_args()
    prec = os.environ.get("P2PVG_PRECISION", "bf16")
    info = card()
    print("card (name, power limit, SM clock, max SM clock):", info, "| precision", prec, flush=True)
    T = CPS[-1] + 1
    steps = CPS[-1]   # executed steps of the chain: L_k - 1 = T_k - 1 per segment
    lines = []
    for name, width, C, B, ns in WORKLOADS:
        if name[0] not in args.only:
            continue
        model = make_model(width, C, B)
        gen = torch.Generator(device="cuda").manual_seed(2)
        if width == "pose":
            x = 3 * torch.randn(T, B, 17, 3, device="cuda", generator=gen)
        else:
            side = SIDE.get(width, width)
            x = torch.rand(T, B, C, side, side, device="cuda", generator=gen)
        tol = "pose" if width == "pose" else prec
        segs = segments(list(x))
        variants = {
            "eager_looped": lambda: [chained(model.p2p_generate, segs) for _ in range(ns)],
            "graphed_looped": lambda: chained(model.p2p_generate_graphed, segs, nsample=ns),
            "chain": lambda: model.p2p_generate_multi_cp(x, CPS, nsample=ns),
        }
        parity = dict(
            graphed_looped=compare(variants["graphed_looped"], variants["chain"], ns * B, steps, ns, tol),
            eager_looped_one_sample=compare(lambda: chained(model.p2p_generate, segs),
                                            lambda: model.p2p_generate_multi_cp(x, CPS), B, steps, 1, tol))
        for fn in variants.values():   # warm-up: module loads, graph capture
            fn()
        times = {k: [] for k in variants}
        for _ in range(args.reps):     # alternate the paths
            for k, fn in variants.items():
                times[k].append(timed(fn, 1))
        eng = model._gen_engine
        eng.clear()
        variants["chain"]()
        memory = dict(chain=eng.memory_bytes())
        frames = ns * B * steps
        res = dict(workload=name, backbone=width, channels=C, B=B, samples=ns, cp_ixs=CPS, precision=prec, card=info,
                   parity=parity, graph_memory_bytes=memory)
        for k, ts in times.items():
            ms = statistics.median(ts)
            res[k] = dict(ms=round(ms, 3), spread_ms=round(max(ts) - min(ts), 3), frames_per_s=round(frames / ms * 1e3, 1))
        res["chain_speedup_vs_graphed_looped"] = round(res["graphed_looped"]["ms"] / res["chain"]["ms"], 3)
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
