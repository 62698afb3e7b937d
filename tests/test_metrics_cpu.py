"""The float64 restatement of the frame and pose scores (tests/metrics_ref.py) against first principles, and the host parts of
p2pvg_b200/metrics.py that need no GPU: the pair planner of P2PModel.p2p_evaluate, the best-sample pick and the input
checks that run before any launch."""
import math

import numpy as np
import pytest
import torch

from p2pvg_b200 import metrics
from tests import metrics_ref as R


def brute_ssim(p, g, data_range):
    """One window at a time, each statistic summed in a loop."""
    C, H, W = p.shape
    c1, c2 = (0.01 * data_range) ** 2, (0.03 * data_range) ** 2
    per_channel = []
    for c in range(C):
        vals = []
        for i in range(H - 6):
            for j in range(W - 6):
                x = [float(v) for v in p[c, i:i + 7, j:j + 7].ravel()]
                y = [float(v) for v in g[c, i:i + 7, j:j + 7].ravel()]
                ux, uy = sum(x) / 49, sum(y) / 49
                vx = sum((a - ux) ** 2 for a in x) / 48
                vy = sum((b - uy) ** 2 for b in y) / 48
                vxy = sum((a - ux) * (b - uy) for a, b in zip(x, y)) / 48
                vals.append((2 * ux * uy + c1) * (2 * vxy + c2) / ((ux * ux + uy * uy + c1) * (vx + vy + c2)))
        per_channel.append(sum(vals) / len(vals))
    return sum(per_channel) / C


@pytest.mark.parametrize("shape", [(1, 7, 7), (1, 9, 12), (2, 11, 8), (3, 8, 10)])
@pytest.mark.parametrize("data_range", [1.0, 2.0])
def test_restatement_matches_brute_force(shape, data_range):
    rng = np.random.default_rng(sum(shape))
    p, g = rng.random(shape) * data_range, rng.random(shape) * data_range
    mse, psnr, ssim = R.frame_scores(p, g, data_range)
    d = [(a - b) ** 2 for a, b in zip(p.ravel(), g.ravel())]
    want_mse = sum(d) / len(d)
    assert abs(mse - want_mse) <= 1e-12
    assert abs(psnr - 10 * math.log10(data_range ** 2 / want_mse)) <= 1e-12
    assert abs(ssim - brute_ssim(p, g, data_range)) <= 1e-12


def test_identical_frames():
    p = np.random.default_rng(1).random((3, 16, 16))
    mse, psnr, ssim = R.frame_scores(p, p.copy())
    assert mse == 0 and psnr == math.inf and abs(ssim - 1) <= 1e-15


@pytest.mark.parametrize("a,b,data_range", [(0.3, 0.7, 1.0), (0.0, 1.0, 1.0), (0.95, 0.95, 1.0), (1.5, 0.25, 2.0)])
def test_constant_frames(a, b, data_range):
    p, g = np.full((2, 10, 12), a), np.full((2, 10, 12), b)
    c1 = (0.01 * data_range) ** 2
    mse, _, ssim = R.frame_scores(p, g, data_range)
    assert abs(mse - (a - b) ** 2) <= 1e-15
    assert abs(ssim - (2 * a * b + c1) / (a * a + b * b + c1)) <= 1e-12


def test_symmetry_and_channel_average():
    rng = np.random.default_rng(2)
    p, g = rng.random((3, 12, 16)), 1 / (1 + np.exp(-rng.normal(size=(3, 12, 16))))
    a, b = R.frame_scores(p, g), R.frame_scores(g, p)
    assert np.allclose(a, b, rtol=0, atol=1e-14)
    per_channel = [R.frame_scores(p[c:c + 1], g[c:c + 1])[2] for c in range(3)]
    assert abs(a[2] - sum(per_channel) / 3) <= 1e-14
    # mse is the mean over all elements: with equal channel sizes, the mean of the per-channel mse
    assert abs(a[0] - np.mean([R.frame_scores(p[c:c + 1], g[c:c + 1])[0] for c in range(3)])) <= 1e-15


def test_pose_restatement():
    rng = np.random.default_rng(3)
    p = rng.normal(size=(17, 3))
    assert R.pose_scores(p, p) == (0.0, 0.0)
    q = p.copy()
    q[:, 0] += 0.5   # every joint moved 0.5 along x
    mse, mpjpe = R.pose_scores(q, p)
    assert abs(mse - 0.25 / 3) <= 1e-15 and abs(mpjpe - 0.5) <= 1e-15
    q = p.copy()
    q[4] += np.array([3.0, 4.0, 0.0])   # one joint moved by 5
    mse, mpjpe = R.pose_scores(q, p)
    assert abs(mse - 25 / 51) <= 1e-14 and abs(mpjpe - 5 / 17) <= 1e-14


# ---- the pair planner: (output row, input row) per scored (frame, b, sample) -------------------------------------------
# output store: [n_dec][nsample * B] rows, frame i at row block i - n_past, sample-major; input store: [T][B] rows
@pytest.mark.parametrize("L,T,n_past,nsample,B,frames,pairs", [
    (3, 3, 1, 1, 1, [1, 2], [[0, 1], [1, 2]]),
    (5, 5, 3, 1, 2, [3, 4], [[0, 6], [1, 7], [2, 8], [3, 9]]),
    (4, 4, 3, 4, 2, [3], [[0, 6], [2, 6], [4, 6], [6, 6], [1, 7], [3, 7], [5, 7], [7, 7]]),
    (4, 4, 1, 4, 1, [1, 2, 3], [[0, 1], [1, 1], [2, 1], [3, 1], [4, 2], [5, 2], [6, 2], [7, 2], [8, 3], [9, 3], [10, 3], [11, 3]]),
    (6, 4, 1, 1, 2, [5], [[8, 6], [9, 7]]),
    (3, 5, 1, 4, 1, [2], [[4, 4], [5, 4], [6, 4], [7, 4]]),
    (7, 5, 3, 4, 1, [6], [[12, 4], [13, 4], [14, 4], [15, 4]]),
    (4, 8, 3, 1, 3, [3], [[0, 21], [1, 22], [2, 23]]),
])
def test_plan_pairs(L, T, n_past, nsample, B, frames, pairs):
    got_frames, got = metrics.plan_pairs(L, T, n_past, nsample, B)
    assert got_frames == frames
    assert got.dtype == torch.int32 and got.tolist() == pairs


@pytest.mark.parametrize("L,n_past", [(1, 1), (3, 3), (2, 3)])
def test_plan_pairs_rejects_nothing_generated(L, n_past):
    with pytest.raises(ValueError):
        metrics.plan_pairs(L, L, n_past, 1, 1)


def test_best_of_picks_best_mean_first_on_ties():
    # [nsample=3, F=2, B=3]
    ssim = torch.tensor([[[0.5, 0.9, 0.2], [0.5, 0.1, 0.2]],
                         [[0.6, 0.5, 0.2], [0.6, 0.5, 0.2]],
                         [[0.7, 0.5, 0.2], [0.3, 0.5, 0.2]]], dtype=torch.float64)
    mse = 1 - ssim
    best = metrics.best_of({"ssim": ssim, "mse": mse}, ("ssim", "mse"))
    idx, curve = best["ssim"]
    # b = 0: means 0.5, 0.6, 0.5 -> 1; b = 1: 0.5, 0.5, 0.5 -> 0 (first); b = 2: all equal -> 0
    assert idx.tolist() == [1, 0, 0]
    assert torch.equal(curve, torch.stack([ssim[i, :, b] for b, i in enumerate(idx.tolist())], 1))
    assert best["mse"][0].tolist() == [1, 0, 0]
    # an identical frame (psnr inf) makes the sample's mean inf; equal inf means go to the first sample
    psnr = torch.tensor([[[30.0, math.inf], [30.0, 30.0]], [[math.inf, math.inf], [30.0, 30.0]]], dtype=torch.float64)
    assert metrics.best_of({"psnr": psnr}, ("psnr",))["psnr"][0].tolist() == [1, 0]


def test_wrappers_reject_before_any_launch():
    x = torch.zeros(2, 1, 8, 8)
    with pytest.raises(ValueError, match="CUDA"):
        metrics.frame_metrics(x, x)
    with pytest.raises(ValueError, match="CUDA"):
        metrics.pose_metrics(torch.zeros(2, 17, 3), torch.zeros(2, 17, 3))
    for bad in (0.0, -1.0, math.inf, math.nan):
        with pytest.raises(ValueError):
            metrics._check_range(bad)
