#!/usr/bin/env python
"""Representative launches of the wgmma GEMM (shapes of the dcgan_64 batch-256 train step) for
`ncu --set full -k regex:gemm_tc_kernel`:  conv forward (K-major), ConvT forward (MN-major B, output-bound),
weight gradient (MN-major A and B, split-K).  `--shape M,N,K,a_mn,b_mn,f32out` (repeatable) overrides the list;
`--time` prints the CUDA-event time of each launch (second repetition)."""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from p2pvg_b200._lib import CudaKernels  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--shape", action="append", default=[])
ap.add_argument("--time", action="store_true")
ap.add_argument("--bias", action="store_true")
args = ap.parse_args()
K = CudaKernels("cuda")
bf = torch.bfloat16
shapes = [  # M, N, K, a_mn, b_mn, c dtype
    (491520, 256, 2048, False, False, bf),          # encoder c3 forward
    (1966080, 1024, 128, False, True, bf),          # decoder upc4 forward (col buffer, output-bound)
    (512, 4096, 122880, True, True, torch.float32),  # decoder upc2 weight gradient (split-K)
]
if args.shape:
    shapes = []
    for s in args.shape:
        M, N, Kd, a, b, f = (int(v) for v in s.split(","))
        shapes.append((M, N, Kd, bool(a), bool(b), torch.float32 if f else bf))
for rep in range(2):
    for M, N, Kd, a_mn, b_mn, cdt in shapes:
        A = torch.randn((Kd, M) if a_mn else (M, Kd), device="cuda", dtype=bf)
        B = torch.randn((Kd, N) if b_mn else (N, Kd), device="cuda", dtype=bf)
        C = torch.empty(M, N, device="cuda", dtype=cdt)
        bias = torch.randn(N, device="cuda") if args.bias else None
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        K.gemm(A, B, C, M, N, Kd, a_mn=a_mn, b_mn=b_mn, bias=bias)
        e1.record()
        torch.cuda.synchronize()
        if args.time and rep == 1:
            ms = e0.elapsed_time(e1)
            gb = (A.numel() * 2 + B.numel() * 2 + C.numel() * C.element_size()) / 1e9
            print(f"gemm M={M} N={N} K={Kd} a_mn={int(a_mn)} b_mn={int(b_mn)}: {ms:.3f} ms  {2 * M * N * Kd / ms / 1e9:.1f} TFLOP/s  {gb / ms * 1e3:.0f} GB/s")
        del A, B, C
print("done")
