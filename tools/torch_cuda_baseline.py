#!/usr/bin/env python
"""Library baseline (BASELINE.md §3 (ii)): the reference's train step -- restated by oracle/p2p_oracle.py, i.e. plain PyTorch
ops + autograd + the legacy Adam -- run on the same GPU through stock torch-CUDA (cuDNN / cuBLAS), on the bench workload
(mnist dcgan_64, T=30, B=256, skip_prob 0).  Test / measurement infrastructure only; nothing in the product path imports it."""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import p2p_oracle as O  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=256)
ap.add_argument("--seq", type=int, default=30)
ap.add_argument("--steps", type=int, default=3)
args = ap.parse_args()
CFG = dict(g_dim=128, z_dim=10, rnn_size=256, channels=1, image_width=64, predictor_rnn_layers=2, posterior_rnn_layers=1,
           prior_rnn_layers=1)
T, B = args.seq, args.batch
dev = torch.device("cuda")
opt = O.default_opt(batch_size=B)
x = torch.rand(T, B, 1, 64, 64, device=dev)
probs = np.random.RandomState(0).uniform(0, 1, T - 1)
eps = O.draw_eps(T - 1, B, CFG["z_dim"], seed=3).to(dev)


def run(label, tf32, autocast):
    torch.backends.cudnn.allow_tf32 = tf32
    torch.backends.cuda.matmul.allow_tf32 = tf32
    torch.backends.cudnn.benchmark = True
    state = {m: {k: v.to(dev) for k, v in sd.items()} for m, sd in O.build_state(CFG, seed=1).items()}
    adam = {m: O.new_adam_state(state[m]) for m in O.MODULES}
    times = []
    for it in range(args.steps + 2):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            out = O.train_step(state, adam, x, opt, 64, eps, probs, mode="A")
        e1.record()
        torch.cuda.synchronize()
        if it >= 2:
            times.append(e0.elapsed_time(e1))
    ms = float(np.median(times))
    print(f"torch-CUDA {label}: {ms:.1f} ms/step = {T * B / ms * 1e3:,.0f} frames/s  peak mem {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB  "
          f"losses {[round(float(v), 5) for v in out['losses']]}", flush=True)


run("fp32 (TF32 off)", False, False)
run("TF32 (allow_tf32)", True, False)
run("bf16 autocast", True, True)
