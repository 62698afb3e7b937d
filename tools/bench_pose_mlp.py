#!/usr/bin/env python
"""One p2pvg_pose_mlp launch against the launch sequence it replaces (infer.mlp_encoder_forward / mlp_decoder_forward:
per residual block 4 x (exact fp32 GEMM + activation), the residual accumulate and the LayerNorm, plus the final Linear and
the decoder's torch.cat), for the h36m_mlp encoder and decoder at g_dim 128.  Rows: 10, 200 and 300 (B, nsample * B and
T * B of the vis_seq-shaped pose workload: B = 10, 20 samples, 30 frames).

Both sides are captured in CUDA graphs of --calls back-to-back calls and timed with CUDA events over --reps replays,
alternating; each reports the median time per call.  Outputs are compared before timing.  Prints the card name, power
limit and SM clock, then one JSON line per (module, rows)."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from p2pvg_b200.infer import kernels_for, mlp_decoder_forward, mlp_encoder_forward  # noqa: E402
from p2pvg_b200.models import h36m_mlp  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def graphed(fn, calls):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(calls):
            fn()
    return g


def time_graph(g, calls):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    g.replay()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / calls   # us per call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--g", type=int, default=128)
    ap.add_argument("--calls", type=int, default=200, help="calls per captured graph")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    info = card()
    print("card (name, power limit, SM clock, max SM clock):", info, flush=True)
    torch.manual_seed(0)
    g = args.g
    enc = h36m_mlp.encoder(out_dim=g, h_dim=g).cuda()
    dec = h36m_mlp.decoder(in_dim=g, h_dim=g).cuda()
    K = kernels_for("cuda")
    lines = []
    for rows in (10, 200, 300):
        x = 3 * torch.randn(rows, 17, 3, device="cuda")
        vec = torch.tanh(torch.randn(rows, g, device="cuda"))
        h, h1, h2 = (torch.empty(rows, g, device="cuda") for _ in range(3))
        pose = torch.empty(rows, 17, 3, device="cuda")
        s1, s2 = torch.randn(rows, g, device="cuda"), torch.randn(rows, g, device="cuda")
        cases = {
            "encoder": (lambda: K.pose_mlp(enc, False, x, h, rows, h1=h1, h2=h2), lambda: mlp_encoder_forward(enc, x),
                        lambda: h, lambda r: r[0]),
            "decoder": (lambda: K.pose_mlp(dec, True, vec, pose, rows, skips=[s1, s2], nsrc=rows),
                        lambda: mlp_decoder_forward(dec, vec, [s1, s2]), lambda: pose, lambda r: r),
        }
        for name, (fused, eager, fused_out, eager_out) in cases.items():
            fused()
            ref = eager_out(eager())
            err = (fused_out() - ref).abs().max().item()
            n0 = K.launches
            eager()
            eager_launches = K.launches - n0
            gf, ge = graphed(fused, args.calls), graphed(eager, args.calls)
            tf, te = [], []
            for _ in range(args.reps):   # alternate the two graphs
                tf.append(time_graph(gf, args.calls))
                te.append(time_graph(ge, args.calls))
            res = dict(module=name, g=g, rows=rows, card=info, max_abs_err=err, project_launches_replaced=eager_launches,
                       fused_us=round(statistics.median(tf), 2), eager_us=round(statistics.median(te), 2),
                       fused_spread_us=round(max(tf) - min(tf), 2), eager_spread_us=round(max(te) - min(te), 2),
                       speedup=round(statistics.median(te) / statistics.median(tf), 2))
            line = json.dumps(res)
            print(line, flush=True)
            lines.append(line)
            del gf, ge
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
