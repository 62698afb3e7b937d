#!/usr/bin/env python
"""Held-out scoring (P2PModel.p2p_losses) at the bench.py shapes, bf16, randomly initialised weights, skip_prob 0:

  C2    dcgan_64, C = 1, T = 30, B = 256
  C3    vgg_64,   C = 3, T = 30, B = 128
  pose  h36m_mlp, rnn_size 512, T = 60, B = 256 (C5's per-GPU batch)

  losses     p2p_losses(x) (one CUDA-graph replay, the NumPy / torch draws and the read-back of the scalars included)
  step       forward(x): a full training step (graph replay) on the same batch shape
  torch      the same eval-mode forward in stock PyTorch-CUDA under no_grad and bf16 autocast (cuDNN / cuBLAS), on the plain-
             PyTorch modules tools/torch_cuda_baseline.py runs (the oracle's layer functions, restated in eval mode by
             tests/loss_eval_ref.py)

Host clock around calls that end in a device synchronise, after warm-up, median and range of --reps.  Prints the card
name, power limit and maximum SM clock, then one JSON line per shape."""
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from p2pvg_b200.models import dcgan_64, h36m_mlp, vgg_64  # noqa: E402
from p2pvg_b200.models.p2p_model import MODULES, P2PModel  # noqa: E402
from tests.loss_eval_ref import forward_losses_eval  # noqa: E402

SHAPES = {"C2": (dcgan_64, 1, 30, 256, 256), "C3": (vgg_64, 3, 30, 128, 256), "pose": (h36m_mlp, 1, 60, 256, 512)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts), min(ts), max(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", nargs="*", default=list(SHAPES))
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--torch-reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_losses measures on a CUDA device")
    print("card:", card(), flush=True)
    for name in args.shapes:
        net, C, T, B, R = SHAPES[name]
        pose = net is h36m_mlp
        opt = types.SimpleNamespace(dataset="h36m" if pose else "mnist", backbone_net=net, lr=1e-3, beta1=0.9, beta=1e-4,
                                    weight_cpc=100.0, weight_align=0.5, skip_prob=0.0, n_past=1, last_frame_skip=False, batch_size=B)
        torch.manual_seed(1)
        model = P2PModel(B, C, 128, 10, R, 1, 1, 2, opt=opt).cuda()
        x = torch.randn(T, B, 17, 3, device="cuda") if pose else torch.rand(T, B, C, 64, 64, device="cuda")
        model.train()
        for _ in range(3):
            model(x)
        step = timed(lambda: model(x), args.reps)
        eng = model._engine
        graphs0, gen0 = {k: v for k, v in eng._graphs.items() if v != "warm"}, eng.graph_generation()
        model.eval()
        for _ in range(3):
            v = model.p2p_losses(x)
        losses = timed(lambda: model.p2p_losses(x), args.reps)
        model.train()
        model(x)
        torch.cuda.synchronize()
        kept = eng.graph_generation() == gen0 and all(eng._graphs.get(k) is g for k, g in graphs0.items())
        # stock PyTorch-CUDA eval forward on the same weights and buffers
        state = {m: dict(getattr(model, m).state_dict()) for m in MODULES}
        width = "mlp" if pose else ("vgg" if net is vgg_64 else 64)
        fopt = dict(skip_prob=0.0, n_past=1, last_frame_skip=False, batch_size=B)
        probs = np.zeros(T - 1)
        eps = torch.randn(T - 1, 2, B, 10, device="cuda")
        torch.backends.cudnn.benchmark = True

        def torch_eval():
            with torch.autocast("cuda", dtype=torch.bfloat16):
                return forward_losses_eval(state, x, fopt, width, eps, probs)
        torch_eval()
        tor = timed(torch_eval, args.torch_reps)
        rec = dict(shape=name, T=T, B=B, rnn_size=R, p2p_losses_ms=round(losses[0], 3), p2p_losses_range=[round(losses[1], 3), round(losses[2], 3)],
                   train_step_ms=round(step[0], 3), train_step_range=[round(step[1], 3), round(step[2], 3)],
                   torch_eval_ms=round(tor[0], 2), torch_eval_range=[round(tor[1], 2), round(tor[2], 2)],
                   speedup_vs_torch=round(tor[0] / losses[0], 2), losses_over_step=round(losses[0] / step[0], 3),
                   training_graph_kept=kept, losses=[v[k] for k in ("mse", "kld", "cpc", "align")])
        print(json.dumps(rec), flush=True)
        del model, eng, state
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
