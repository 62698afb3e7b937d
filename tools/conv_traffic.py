"""Per-launch time and operand traffic of the implicit-GEMM convolutions (kinds 0 and 2) of one C2 training step.

    python tools/conv_traffic.py [--config C2] [--reps 20] [--out FILE.json]

Runs one eager step of the bench configuration, records every kind-0 / kind-2 `conv_gemm` launch with its exact arguments
(shape, fused statistics, addend, grp_src), then replays each launch on its own: CUDA-event time over `--reps` launches
after warm-up.  For each launch it prints the time, TFLOP/s, and the operand bytes the persistent tile walk moves from L2
into shared memory (tiles x K blocks x stage bytes, computed from the shapes as conv_gemm.cu tiles them) with their rate.
The card's name, power limit and the SM clock sampled during the replays are printed with the table.
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (CONFIGS, synth_batch, ClockSampler)

ROW_BYTES = 128   # one pixel's 64 bf16 channels of an operand stage


def box_fits(P, H, W):
    """a P-pixel box {W, bh, bn} tiles the H x W maps (conv_gemm.cu box_for)"""
    HW = H * W
    if HW >= P:
        if P % W or H % (P // W):
            return False
        bh, bn = P // W, 1
    else:
        if P % HW:
            return False
        bh, bn = H, P // HW
    return bh * 2 <= 256 and W * 2 <= 256 and bn <= 256


def tile_shape(kind, H, W, Cn, stats):
    """BM x BN as conv_gemm.cu picks it: 256 x 64 for kind 2 with 64 output channels and no fused statistics, when
    256-pixel boxes tile the map; 128 x 64 / 128 x 128 otherwise"""
    BN = 128 if Cn > 64 else 64
    BM = 256 if kind == 2 and Cn == 64 and not stats and box_fits(256, H, W) else 128
    return BM, BN


def operand_bytes(kind, N, H, W, Ck, Cn, stats):
    """Bytes L2 -> shared memory of the tile walk of a kind-0 / kind-2 launch (4x4 filters): every BM x BN tile loads a
    BM-pixel box and a BN x 64 weight tile per K block (kind 0: 16 taps x Ck / 64 blocks; kind 2: 4 taps per phase)."""
    BM, BN = tile_shape(kind, H, W, Cn, stats)
    tiles = -(-N * H * W // BM) * -(-Cn // BN) * (4 if kind == 2 else 1)
    nkb = (16 if kind == 0 else 4) * (Ck // 64)
    return tiles * nkb * (BM + BN) * ROW_BYTES


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={q}", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, plim, mx = [s.strip() for s in out.split(",")]
        return dict(name=name, power_limit=plim, sm_max_clock=mx)
    except Exception as e:  # reported, never fatal
        return dict(name=torch.cuda.get_device_name(), power_limit=f"unavailable ({e!r:.60})", sm_max_clock=None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C2", choices=["C2", "C4"])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    c = bench.CONFIGS[args.config]
    import importlib
    from p2pvg_b200.models.p2p_model import P2PModel

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    os.environ["P2PVG_PRECISION"] = "bf16"
    os.environ["P2PVG_GRAPH"] = "0"
    torch.manual_seed(1)
    np.random.seed(0)
    T, B = c["T"], c["per_gpu"]
    backbone = importlib.import_module(f"p2pvg_b200.models.{c['backbone']}")
    opt = types.SimpleNamespace(dataset=c["dataset"], backbone_net=backbone, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0,
                                weight_align=0.5, skip_prob=0.0, n_past=1, last_frame_skip=False, batch_size=B)
    model = P2PModel(B, c["channels"], bench.G_DIM, bench.Z_DIM, c["rnn"], 1, 1, 2, opt=opt).cuda()
    model.train()
    x = bench.synth_batch(c, T, B, torch.Generator().manual_seed(1234)).to(dev)
    eng = model.engine(c["width"] or 0)
    K = eng.K
    eng.step(x, use_graph=False, return_device=True)   # allocations, plan

    calls = []
    orig = K.conv_gemm

    def rec(kind, a, b, cc, N, H, W, Ck, Cn, Cm=0, **kw):
        orig(kind, a, b, cc, N, H, W, Ck, Cn, Cm=Cm, **kw)
        if kind in (0, 2):
            calls.append((kind, a, b, cc, N, H, W, Ck, Cn, Cm, kw))

    K.conv_gemm = rec
    eng._serial = True
    try:
        np.random.seed(0)
        eng.step(x, use_graph=False, return_device=True)
        torch.cuda.synchronize()
    finally:
        eng._serial = False
        del K.conv_gemm

    sampler = bench.ClockSampler(0)
    sampler.start()
    time.sleep(0.3)
    t0 = time.time()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    rows = []
    for (kind, a, b, cc, N, H, W, Ck, Cn, Cm, kw) in calls:
        for _ in range(3):
            orig(kind, a, b, cc, N, H, W, Ck, Cn, Cm=Cm, **kw)
        e0.record()
        for _ in range(args.reps):
            orig(kind, a, b, cc, N, H, W, Ck, Cn, Cm=Cm, **kw)
        e1.record()
        torch.cuda.synchronize()
        t = e0.elapsed_time(e1) / args.reps
        flop = 2.0 * N * H * W * 16 * Ck * Cn
        stats = kw.get("stat_partial") is not None
        by = operand_bytes(kind, N, H, W, Ck, Cn, stats)
        BM, BN = tile_shape(kind, H, W, Cn, stats)
        rows.append(dict(kind=kind, N=N, H=H, Ck=Ck, Cn=Cn, stats=stats, addend=kw.get("addend") is not None,
                         grp_src=kw.get("grp_src") is not None, tile=f"{BM}x{BN}", tflop=flop / 1e12, ms=t, tflops=flop / (t * 1e-3) / 1e12,
                         operand_gb=by / 1e9, operand_tbs=by / (t * 1e-3) / 1e12, flop_per_byte=flop / by))
    t1 = time.time()
    clocks = sampler.stop(t0, t1)
    info = gpu_info()
    info["sm_clock_during_replays"] = clocks
    print(f"# {info['name']}, power limit {info['power_limit']}, max SM clock {info['sm_max_clock']}, "
          f"SM clock during the replays {clocks}")
    print("# operand bytes: L2 -> shared memory of the tile walk (computed); FLOP/B: FLOP per filled operand byte; "
          "time: CUDA events, mean of %d launches" % args.reps)
    print(f"{'kind':>4} {'N':>5} {'H':>3} {'Ck':>4} {'Cn':>4} {'epilogue':>13} {'tile':>7} | {'ms':>7} {'TFLOP/s':>7} {'GB':>6} "
          f"{'TB/s':>5} {'FLOP/B':>6}")
    for r in rows:
        epi = " ".join(n for n in ("stats", "addend") if r[n])
        print(f"{r['kind']:>4} {r['N']:>5} {r['H']:>3} {r['Ck']:>4} {r['Cn']:>4} {epi or '-':>13} {r['tile']:>7} | "
              f"{r['ms']:>7.3f} {r['tflops']:>7.0f} {r['operand_gb']:>6.2f} {r['operand_tbs']:>5.2f} {r['flop_per_byte']:>6.1f}")
    print(f"# sum over {len(rows)} launches: {sum(r['ms'] for r in rows):.3f} ms")
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(dict(gpu=info, config=args.config, reps=args.reps, launches=rows), open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
