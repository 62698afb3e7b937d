#!/usr/bin/env python
"""Runs N eager (non-graph) train steps of the bench workload so that `ncu` can list every kernel launch:

    ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file launches.csv \
        python tools/profile_step.py --steps 2
"""
import argparse
import os
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from p2pvg_b200.models import dcgan_64, dcgan_128, h36m_mlp, vgg_64  # noqa: E402
from p2pvg_b200.models.p2p_model import P2PModel  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=2)
ap.add_argument("--batch", type=int, default=256)
ap.add_argument("--seq", type=int, default=30)
ap.add_argument("--backbone", default="dcgan_64", choices=["dcgan_64", "dcgan_128", "vgg_64", "h36m_mlp"])
ap.add_argument("--channels", type=int, default=1)
ap.add_argument("--rnn", type=int, default=256)
ap.add_argument("--phases", action="store_true")
ap.add_argument("--calls", action="store_true", help="time every kernel-API call with CUDA events (last step)")
args = ap.parse_args()
os.environ["P2PVG_GRAPH"] = "0"
net = dict(dcgan_64=dcgan_64, dcgan_128=dcgan_128, vgg_64=vgg_64, h36m_mlp=h36m_mlp)[args.backbone]
pose = args.backbone == "h36m_mlp"
width = 128 if args.backbone.endswith("128") else 64
opt = types.SimpleNamespace(dataset="h36m" if pose else "mnist", backbone_net=net, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0, weight_align=0.5,
                            skip_prob=0.0, n_past=1, last_frame_skip=False, batch_size=args.batch)
torch.manual_seed(1)
model = P2PModel(args.batch, args.channels, 128, 10, args.rnn, 1, 1, 2, opt=opt).cuda()
x = 3 * torch.randn(args.seq, args.batch, 17, 3, device="cuda") if pose else torch.rand(args.seq, args.batch, args.channels, width, width, device="cuda")
eng = model.engine(width)
calls = []


def wrap_kernels(K):
    import inspect
    for name, fn in inspect.getmembers(K, predicate=inspect.ismethod):
        if name.startswith("_") or name in ("gemm_workspace", "bn_workspace", "set_gemm_impl", "set_fp32_gemm_mode", "has_tc_gemm", "mse_chunks"):
            continue

        def make(name, fn):
            def w(*a, **kw):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                r = fn(*a, **kw)
                e1.record()
                ints = [str(v) for v in a if isinstance(v, int)][:7]
                calls.append((name, ",".join(ints), e0, e1, len(eng.phase_events) if eng.phase_events is not None else 0))
                return r
            return w
        setattr(K, name, make(name, fn))


for i in range(args.steps):
    if args.calls and i == args.steps - 1:
        wrap_kernels(eng.K)
        args.phases = True
    n0 = eng.K.launches
    eng.phase_events = [] if args.phases else None
    out = eng.step(x, use_graph=False, return_device=True)
    torch.cuda.synchronize()
    if args.phases and i == args.steps - 1:
        ev = eng.phase_events
        for (_, a), (name, b) in zip(ev[:-1], ev[1:]):
            print(f"  phase {name:14s} {a.elapsed_time(b):8.3f} ms")
        print(f"  total {ev[0][1].elapsed_time(ev[-1][1]):8.3f} ms")
    if args.calls and i == args.steps - 1:
        names = [n for n, _ in eng.phase_events]
        rows = [(c[2].elapsed_time(c[3]), c[0], c[1], names[min(c[4], len(names) - 1)]) for c in calls]
        from collections import defaultdict
        agg = defaultdict(lambda: [0, 0.0])
        for ms, nm, dims, ph in rows:
            agg[(ph, nm)][0] += 1
            agg[(ph, nm)][1] += ms
        print("  per phase / op (CUDA-event time incl. launch gaps):")
        for (ph, nm), (cnt, ms) in sorted(agg.items(), key=lambda kv: -kv[1][1])[:45]:
            print(f"    {ph:13s} {nm:20s} n={cnt:4d} {ms:8.3f} ms")
        print("  slowest single calls:")
        for ms, nm, dims, ph in sorted(rows, reverse=True)[:40]:
            print(f"    {ms:7.3f} ms {ph:13s} {nm:14s} {dims}")
    print(f"step {i}: {eng.K.launches - n0} kernel launches, losses {out.tolist()}", flush=True)
