#!/usr/bin/env python
"""Representative launches of the implicit-GEMM convolution kernel (shapes of the dcgan_64 batch-256 step) for
`ncu --set full -k regex:conv_gemm_kernel`: conv forward c3, ConvT forward upc3, weight gradient c3, ConvT upc4 (with the skip addend), c3 forward with fused BatchNorm statistics."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from p2pvg_b200._lib import CudaKernels  # noqa: E402

K = CudaKernels("cuda")
bf = torch.bfloat16
N = 7680
for rep in range(2):
    x = torch.randn(N, 16, 16, 128, device="cuda", dtype=bf)          # big map of c3
    w = torch.randn(256, 16 * 128, device="cuda", dtype=bf) * 0.02
    y = torch.empty(N, 8, 8, 256, device="cuda", dtype=bf)
    K.conv_gemm(0, x, w, y, N, 8, 8, 128, 256)                        # kind 0: conv forward
    xs = torch.randn(N, 8, 8, 256, device="cuda", dtype=bf)
    wt = torch.randn(256, 16 * 128, device="cuda", dtype=bf) * 0.02
    yb = torch.empty(N, 16, 16, 128, device="cuda", dtype=bf)
    K.conv_gemm(2, xs, wt, yb, N, 8, 8, 256, 128)                     # kind 2: ConvT forward
    gw = torch.empty(256, 16 * 128, device="cuda")
    K.conv_gemm(1, xs, x, gw, N, 8, 8, 0, 128, Cm=256)                # kind 1: weight gradient
    # upc4 shape (128 -> 64 channels, 16x16 -> 32x32): one 128x64 tile per output-parity phase
    x4 = torch.randn(N, 16, 16, 128, device="cuda", dtype=bf)
    w4 = torch.randn(128, 16 * 64, device="cuda", dtype=bf) * 0.02
    add = torch.randn(256, 32, 32, 64, device="cuda")
    src = torch.zeros(N // 256, dtype=torch.int32, device="cuda")
    y4 = torch.empty(N, 32, 32, 64, device="cuda", dtype=bf)
    K.conv_gemm(2, x4, w4, y4, N, 16, 16, 128, 64, addend=add, grp_src=src, imgs_per_group=256)
    # c3 forward with the BatchNorm statistics fused into the epilogue
    part = torch.empty((N * 64 // 128) * 256 * 2, device="cuda")
    K.conv_gemm(0, x, w, y, N, 8, 8, 128, 256, stat_partial=part)
    torch.cuda.synchronize()
print("done")
