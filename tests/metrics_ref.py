"""Float64 NumPy restatement of the frame and pose scores (p2pvg_b200/metrics.py, include/p2pvg_b200.h), written from the
formulas: 7x7 uniform windows that lie fully inside the frame (sliding_window_view), sample (ddof 1) variances and
covariance, C1 = (0.01 R)^2, C2 = (0.03 R)^2, channels averaged.  No scipy filters, no scikit-image."""
import numpy as np
from numpy.lib.stride_tricks import sliding_window_view

WIN = 7


def ssim_map(p, g, data_range=1.0):
    """S at every 7x7 window of one channel: float64 [H - 6, W - 6]."""
    p, g = np.asarray(p, np.float64), np.asarray(g, np.float64)
    wp, wg = sliding_window_view(p, (WIN, WIN)), sliding_window_view(g, (WIN, WIN))
    n = WIN * WIN
    ux, uy = wp.mean((-2, -1)), wg.mean((-2, -1))
    unb = n / (n - 1)
    vx = unb * ((wp * wp).mean((-2, -1)) - ux * ux)
    vy = unb * ((wg * wg).mean((-2, -1)) - uy * uy)
    vxy = unb * ((wp * wg).mean((-2, -1)) - ux * uy)
    c1, c2 = (0.01 * data_range) ** 2, (0.03 * data_range) ** 2
    return (2 * ux * uy + c1) * (2 * vxy + c2) / ((ux * ux + uy * uy + c1) * (vx + vy + c2))


def frame_scores(p, g, data_range=1.0):
    """(mse, psnr, ssim) of one [C, H, W] pair in float64."""
    p, g = np.asarray(p, np.float64), np.asarray(g, np.float64)
    mse = float(((p - g) ** 2).mean())
    psnr = float("inf") if mse == 0 else float(10 * np.log10(data_range ** 2 / mse))
    ssim = float(np.mean([ssim_map(p[c], g[c], data_range).mean() for c in range(p.shape[0])]))
    return mse, psnr, ssim


def frame_scores_many(pred, gt, pairs, data_range=1.0):
    """float64 [n, 3] scores of pred[pairs[:, 0]] against gt[pairs[:, 1]]."""
    pred, gt = np.asarray(pred), np.asarray(gt)
    return np.array([frame_scores(pred[i], gt[j], data_range) for i, j in np.asarray(pairs)], np.float64).reshape(-1, 3)


def pose_scores(p, g):
    """(mse, mpjpe) of one [J, 3] pair in float64."""
    d = np.asarray(p, np.float64) - np.asarray(g, np.float64)
    return float((d * d).mean()), float(np.sqrt((d * d).sum(1)).mean())


def pose_scores_many(pred, gt, pairs):
    pred, gt = np.asarray(pred), np.asarray(gt)
    return np.array([pose_scores(pred[i], gt[j]) for i, j in np.asarray(pairs)], np.float64).reshape(-1, 2)
