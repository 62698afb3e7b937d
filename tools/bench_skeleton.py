#!/usr/bin/env python
"""The GPU skeleton renderer (p2pvg_b200.skeleton) on the workload of one h36m vis_seq call at train.py's settings.

  (a) one p2pvg_skeleton_render launch of the 3150 pictures of a vis_seq call ((nsample 20 + 1 ground truth) x 5 row blocks
      x 30 frames), fp32 output as vis_seq takes it, poses N(0, 3^2) per coordinate (the loader's scale); CUDA events over
      many launches, and the 363 MB it writes against the H100 SXM's 3.35 TB/s.
  (b) one whole h36m vis_seq call (B = 5 rows shown, nsample 20, seq_len = output_len 30) through the drop-ins: the device
      renderer (dropin/human36m.py), the GPU PNG and GIF writers (dropin/misc/visualize.py) and the drop-in SummaryWriter,
      writing real files in a temporary directory; both skip_frame settings; host clock around the call.
  (c) the host baseline: one matplotlib 3-D figure set up as the reference's visualizer describes it (2 x 2 in at 64 dpi,
      reversed X and Z limits, 16 coloured 3-pt lines), drawn and read back per frame -- when matplotlib imports; otherwise
      "not measured".

Writes skeletons.png (rows: camera views 0..3; columns: poses of tests/golden/pose_data_ref.pt) and results.json to --out.
Prints the card name and power limit first, then one JSON line per part."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from p2pvg_b200 import skeleton as S  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet
NSAMPLE, N_BLOCK, LEN = 20, 5, 30


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def stats(ts):
    return {"median_ms": round(statistics.median(ts), 4), "min_ms": round(min(ts), 4), "max_ms": round(max(ts), 4)}


def part_a(reps):
    n = (NSAMPLE + 1) * N_BLOCK * LEN
    g = torch.Generator(device="cuda").manual_seed(0)
    poses = 3 * torch.randn(n, 17, 3, device="cuda", generator=g)
    views = (torch.arange(n, device="cuda") % N_BLOCK % 4).int()
    out = torch.empty(n, 3, S.SIZE, S.SIZE, device="cuda")
    from p2pvg_b200._lib import kernels_for
    K = kernels_for(poses.device)
    par, col, mats = S.check_parents(S.H36M_PARENTS), S.limb_colors(16).astype(np.float32), S.kernel_matrices((-6, 6))

    def launch():
        K.skeleton_render(poses, views, par, col, mats, out, None)
    for _ in range(3):
        launch()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(20):
            launch()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) / 20)
    med = statistics.median(ts)
    written = out.numel() * 4
    bound_ms = written / HBM_BYTES_PER_S * 1e3
    return {"part": "a", "images": n, "poses": "N(0, 3^2)", "launch": stats(ts), "bytes_written": written,
            "achieved_TB_s": round(written / (med * 1e-3) / 1e12, 3), "hbm_bound_ms": round(bound_ms, 4),
            "share_of_hbm_bound": round(bound_ms / med, 3)}


def part_b(reps, d):
    sys.path.insert(0, os.path.join(ROOT, "dropin"))
    import human36m
    import misc.visualize as dropin_vis
    from tensorboardX import SummaryWriter
    from p2pvg_b200.models import h36m_mlp
    from p2pvg_b200.models.p2p_model import P2PModel
    assert human36m.Skeleton3DVisualizer is S.Skeleton3DVisualizer
    if "imageio" not in sys.modules:
        try:
            import imageio  # noqa: F401
        except ImportError:
            sys.modules["imageio"] = types.SimpleNamespace(mimsave=lambda *a, **k: None)   # the drop-in writes its own GIF
    vis = human36m.Skeleton3DVisualizer(S.H36M_PARENTS, plot_3d_limit=[-6, 6])
    opt = types.SimpleNamespace(dataset="h36m", backbone_net=h36m_mlp, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0,
                                weight_align=0.5, skip_prob=0.5, n_past=1, last_frame_skip=False, batch_size=N_BLOCK,
                                nsample=NSAMPLE, log_dir=d)
    os.makedirs(os.path.join(d, "gen_vis"), exist_ok=True)
    torch.manual_seed(1)
    model = P2PModel(N_BLOCK, 1, 128, 10, 512, 1, 1, 2, opt=opt).cuda().eval()
    g = torch.Generator().manual_seed(5)
    x = (torch.randn(LEN, N_BLOCK, 17, 2, generator=g).cuda(), 3 * torch.randn(LEN, N_BLOCK, 17, 3, generator=g).cuda(),
         torch.arange(N_BLOCK).cuda() % 4)
    w = SummaryWriter(os.path.join(d, "tb"))
    rows = []
    for skip in (False, True):
        def call():
            dropin_vis.vis_seq(model, x, 0, LEN, skip_frame=skip, h36m_visualizer=vis, writer=w, opt=opt)
            w.flush()
        with torch.no_grad():
            call()
            ts = []
            for _ in range(reps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                call()
                torch.cuda.synchronize()
                ts.append((time.perf_counter() - t0) * 1e3)
        rows.append({"part": "b", "workload": f"h36m_mlp vis_seq B={N_BLOCK} nsample={NSAMPLE} output_len={LEN} "
                     f"skip_frame={skip}", "pictures": (NSAMPLE + 1) * N_BLOCK * LEN, **stats(ts)})
    w.close()
    return rows


def part_c(reps):
    try:
        import matplotlib
        matplotlib.use("Agg")
        import matplotlib.pyplot as plt
        from mpl_toolkits.mplot3d import Axes3D  # noqa: F401
    except Exception as e:   # noqa: BLE001
        return {"part": "c", "host_matplotlib_ms_per_frame": "not measured", "reason": f"matplotlib: {type(e).__name__}: {e}"}
    fig = plt.figure(figsize=(2, 2), dpi=64)
    fig.subplots_adjust(left=0.0, right=1.0, top=1.0, bottom=0.0, wspace=0.0, hspace=0.0)
    ax = fig.add_subplot(1, 1, 1, projection="3d")
    ax.set_xlim3d(6, -6)
    ax.set_ylim3d(-6, 6)
    ax.set_zlim3d(6, -6)
    lines = [ax.plot([0.0, 1.0], [0.0, 1.0], [0.0, 1.0], c=tuple(c), linewidth=3)[0] for c in S.limb_colors(16)]
    rs = np.random.RandomState(0)
    poses = 3 * rs.randn(reps * 4, 17, 3)
    ts = []
    for k, p in enumerate(poses):
        t0 = time.perf_counter()
        ax.view_init(elev=15.0, azim=S.AZIMUTHS[k % 4])
        for j in range(1, 17):
            q = S.H36M_PARENTS[j]
            lines[j - 1].set_data_3d([p[j, 0], p[q, 0]], [p[j, 2], p[q, 2]], [p[j, 1], p[q, 1]])
        fig.canvas.draw()
        np.asarray(fig.canvas.buffer_rgba())[15:113, 15:113, :3].copy()
        ts.append((time.perf_counter() - t0) * 1e3)
    med = statistics.median(ts[2:])
    return {"part": "c", "host_matplotlib_ms_per_frame": round(med, 3), "frames": len(ts) - 2,
            "matplotlib": matplotlib.__version__, "vis_seq_pictures_s": round(med * (NSAMPLE + 1) * N_BLOCK * LEN / 1e3, 2)}


def grid_png(out_dir):
    from p2pvg_b200 import png
    fix = torch.load(os.path.join(ROOT, "tests", "golden", "pose_data_ref.pt"), weights_only=False)
    poses = torch.stack([torch.as_tensor(a[len(a) // 2]).float() for a in fix["train"]["pose_3d"][:8]]).cuda()
    imgs = torch.cat([S.render_poses(poses, v) for v in range(4)])                    # [4 * 8, 3, 98, 98]
    grid = imgs.view(4, len(poses), 3, S.SIZE, S.SIZE).permute(2, 0, 3, 1, 4).reshape(3, 4 * S.SIZE, len(poses) * S.SIZE)
    path = os.path.join(out_dir, "skeletons.png")
    png.save_image(grid.contiguous(), path)
    return path


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--parts", default="abc")
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    c = card()
    print("card:", c, flush=True)
    results = {"card": c}
    if "a" in args.parts:
        results["a"] = part_a(args.reps)
        print(json.dumps(results["a"]), flush=True)
    if "b" in args.parts:
        with tempfile.TemporaryDirectory() as d:
            results["b"] = part_b(max(3, args.reps // 2), d)
        for r in results["b"]:
            print(json.dumps(r), flush=True)
    if "c" in args.parts:
        results["c"] = part_c(args.reps)
        print(json.dumps(results["c"]), flush=True)
    results["png"] = grid_png(args.out)
    print("wrote", results["png"], flush=True)
    with open(os.path.join(args.out, "results.json"), "w") as f:
        json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
