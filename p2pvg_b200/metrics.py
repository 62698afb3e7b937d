"""Quantitative scores of generated videos and poses on the GPU (p2pvg_frame_metrics / p2pvg_pose_metrics,
include/p2pvg_b200.h).

Frames: per pair mse, psnr (+inf for identical frames) and ssim -- the 7x7 uniform-window SSIM with sample covariance,
K1 = 0.01, K2 = 0.03 and the windows that lie fully inside the frame, averaged over channels (what
skimage.metrics.structural_similarity computes at its defaults with data_range=R and channel averaging).  Poses: per pair
mse over the J * 3 values and mpjpe, the mean over joints of the Euclidean joint error.

``frame_metrics`` / ``pose_metrics`` score any set of (pred index, gt index) pairs of two stores in one launch, so the
generated frames of several samples can be scored against one copy of the ground truth.  ``plan_pairs`` (one call) and
``plan_pairs_multi_cp`` (a chain through control points) are the pair lists ``P2PModel.p2p_evaluate`` scores inside the
generation engine's buffers; ``plan_pairs_lengths`` is the list ``P2PModel.p2p_evaluate_lengths`` scores (every output length
of one generate_lengths replay).
"""
from __future__ import annotations

import math

import torch

from ._lib import kernels_for

FRAME_METRICS = ("mse", "psnr", "ssim")
POSE_METRICS = ("mse", "mpjpe")
# True where a higher score is better (the best sample maximises it)
HIGHER_IS_BETTER = {"mse": False, "psnr": True, "ssim": True, "mpjpe": False}


def plan_pairs(len_output, len_x, n_past, nsample, B):
    """The frames P2PModel.p2p_evaluate scores and the pairs that score them.

    The generation engine decodes frame i (n_past <= i < len_output) of sample s, batch row b into row
    (i - n_past) * nsample * B + s * B + b of its output store, and holds ground-truth frame t, row b in row t * B + b of its
    input store.  When len_output == len_x every generated frame i is scored against x[i]; otherwise only the control
    point len_output - 1, against x[len_x - 1].  Returns (frames, pairs): the scored frame indices and an int32
    [len(frames) * B * nsample, 2] tensor of (output row, input row), ordered (frame, b, sample) so that the samples of one
    ground-truth frame are scored next to each other."""
    if len_output <= n_past:
        raise ValueError(f"nothing is generated to score: len_output = {len_output} <= n_past = {n_past}")
    if len_output == len_x:
        frames, gts = list(range(n_past, len_output)), list(range(n_past, len_output))
    else:
        frames, gts = [len_output - 1], [len_x - 1]
    return frames, _pairs([f - n_past for f in frames], gts, nsample, B)


def plan_pairs_multi_cp(cp_ixs, n_past, nsample, B):
    """plan_pairs of a multi-control-point call with the clip's timing (P2PModel.p2p_evaluate with cp_ixs): segment k
    generates frames n_past .. T_k - 1 of x[cp_ixs[k] : cp_ixs[k + 1] + 1] (T_k = cp_ixs[k + 1] - cp_ixs[k] + 1), decoded in
    chain order into the output store, and each is scored against its clip frame cp_ixs[k] + i.  Returns (frames, pairs)
    with frames the sorted clip indices; every control point cp_ixs[1:] is among them."""
    frames, dec = [], []
    for a, b in zip(cp_ixs, cp_ixs[1:]):
        if b - a + 1 <= n_past:
            raise ValueError(f"nothing is generated to score in segment [{a}, {b}]: {b - a + 1} frames <= n_past = {n_past}")
        dec += [len(dec) + j for j in range(b - a + 1 - n_past)]
        frames += [a + i for i in range(n_past, b - a + 1)]
    return frames, _pairs(dec, frames, nsample, B)


def plan_pairs_lengths(lens, len_x, n_past, nsample, B):
    """plan_pairs of every output length of ONE generate_lengths replay (P2PModel.p2p_evaluate_lengths).  The lengths
    engine gives length lens[k] the row group g = gen_engine.lengths_order(lens).index(k) of nsample * B rows, and decodes
    its frame i (n_past <= i < lens[k]) of sample s, batch row b into row (i - n_past) * rows + g * nsample * B + s * B + b of
    its output store (rows = len(lens) * nsample * B).  Each length's frames and gt rows are plan_pairs'.

    Returns (frames, pairs, offsets): per length its scored frame indices; int32 [n, 2] pairs, the lengths in caller order,
    each length's pairs ordered (frame, b, sample) as plan_pairs orders them; per length the index of its first pair."""
    from .gen_engine import lengths_order
    order = lengths_order(lens)
    grows = nsample * B
    rows = len(lens) * grows
    frames, parts, offsets, n = [], [], [], 0
    for k, L in enumerate(lens):
        fk, pk = plan_pairs(L, len_x, n_past, nsample, B)
        pred = pk[:, 0].to(torch.int64)
        # plan_pairs' row f * grows + r of a one-length store is row f * rows + g * grows + r here
        pk = torch.stack([(pred // grows) * rows + order.index(k) * grows + pred % grows, pk[:, 1].to(torch.int64)], 1)
        frames.append(fk)
        parts.append(pk.to(torch.int32))
        offsets.append(n)
        n += len(pk)
    return frames, torch.cat(parts), offsets


def _pairs(dec, gts, nsample, B):
    """int32 [len(dec) * B * nsample, 2] pairs (output row, input row) of decoded frame dec[j], sample s, batch row b (row
    (dec[j] * nsample + s) * B + b of the output store) against ground-truth frame gts[j] (row gts[j] * B + b), ordered
    (frame, b, sample)."""
    rows = nsample * B
    f = torch.tensor(dec, dtype=torch.int64).view(-1, 1, 1)
    t = torch.tensor(gts, dtype=torch.int64).view(-1, 1, 1)
    b = torch.arange(B).view(1, -1, 1)
    s = torch.arange(nsample).view(1, 1, -1)
    pred = f * rows + s * B + b
    gt = (t * B + b).expand_as(pred)
    return torch.stack([pred.reshape(-1), gt.reshape(-1)], 1).to(torch.int32)


def _check_store(name, t, tail_dims):
    if not torch.is_tensor(t) or t.device.type != "cuda":
        raise ValueError(f"{name} must be a CUDA tensor")
    if t.dtype != torch.float32:
        raise ValueError(f"{name} must be float32 (got {t.dtype})")
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")
    if t.dim() != tail_dims + 1:
        raise ValueError(f"{name} must have {tail_dims + 1} dimensions (got shape {tuple(t.shape)})")


def _check_pairs(pred, gt, pairs):
    """int32 [n, 2] pairs on pred's device; ValueError for a wrong shape or an index out of range."""
    if pairs is None:
        if pred.shape[0] != gt.shape[0]:
            raise ValueError(f"pairs=None scores pred[i] against gt[i]: {pred.shape[0]} and {gt.shape[0]} frames")
        i = torch.arange(pred.shape[0], dtype=torch.int32)
        return torch.stack([i, i], 1).to(pred.device)
    p = torch.as_tensor(pairs)
    if p.dtype.is_floating_point or p.dtype.is_complex or p.dtype == torch.bool:
        raise ValueError(f"pairs must hold integers (got {p.dtype})")
    if p.dim() != 2 or p.shape[1] != 2:
        raise ValueError(f"pairs must be [n, 2] (got shape {tuple(p.shape)})")
    if p.numel():
        lo, hi = p.min(0).values.tolist(), p.max(0).values.tolist()
        if lo[0] < 0 or hi[0] >= pred.shape[0] or lo[1] < 0 or hi[1] >= gt.shape[0]:
            raise ValueError(f"pair indices out of range: pred [{lo[0]}, {hi[0]}] of {pred.shape[0]} frames, gt [{lo[1]}, {hi[1]}] "
                             f"of {gt.shape[0]} frames")
    return p.to(device=pred.device, dtype=torch.int32).contiguous()


def _check_range(data_range):
    if not (isinstance(data_range, (int, float)) and math.isfinite(data_range) and data_range > 0):
        raise ValueError(f"data_range must be finite and positive (got {data_range!r})")


def launch_frame_metrics(pred, gt, pairs, shape, data_range):
    """One p2pvg_frame_metrics launch on checked operands: fp64 [n, 3] on the device."""
    out = torch.empty(pairs.shape[0], 3, dtype=torch.float64, device=pred.device)
    C, H, W = shape
    kernels_for(pred.device).frame_metrics(pred, gt, pairs, pairs.shape[0], C, H, W, float(data_range), out)
    return out


def launch_pose_metrics(pred, gt, pairs, J):
    """One p2pvg_pose_metrics launch on checked operands: fp64 [n, 2] on the device."""
    out = torch.empty(pairs.shape[0], 2, dtype=torch.float64, device=pred.device)
    kernels_for(pred.device).pose_metrics(pred, gt, pairs, pairs.shape[0], J, out)
    return out


def frame_metrics(pred, gt, pairs=None, data_range=1.0):
    """mse, psnr and ssim of pred[pairs[p, 0]] against gt[pairs[p, 1]] for fp32 contiguous CUDA stores pred [N, C, H, W] and
    gt [M, C, H, W] (pairs=None: pred[i] against gt[i]).  H >= 7, W >= 8 and a multiple of 4, W <= 128.  Returns a dict of
    float64 [n] tensors on the device; bad inputs raise ValueError before any launch."""
    _check_store("pred", pred, 3)
    _check_store("gt", gt, 3)
    if gt.device != pred.device or tuple(gt.shape[1:]) != tuple(pred.shape[1:]):
        raise ValueError(f"pred {tuple(pred.shape)} on {pred.device} and gt {tuple(gt.shape)} on {gt.device} must share frame "
                         "shape and device")
    C, H, W = (int(v) for v in pred.shape[1:])
    if H < 7 or W < 8 or W % 4 or W > 128:
        raise ValueError(f"frames of {H} x {W}: needs H >= 7 and 8 <= W <= 128 with W % 4 == 0")
    _check_range(data_range)
    pairs = _check_pairs(pred, gt, pairs)
    out = launch_frame_metrics(pred, gt, pairs, (C, H, W), data_range)
    return {k: out[:, i] for i, k in enumerate(FRAME_METRICS)}


def pose_metrics(pred, gt, pairs=None):
    """mse and mpjpe of pred[pairs[p, 0]] against gt[pairs[p, 1]] for fp32 contiguous CUDA pose stores pred [N, J, 3] and
    gt [M, J, 3] (pairs=None: pred[i] against gt[i]).  Returns a dict of float64 [n] tensors on the device; bad inputs
    raise ValueError before any launch."""
    _check_store("pred", pred, 2)
    _check_store("gt", gt, 2)
    if gt.device != pred.device or tuple(gt.shape[1:]) != tuple(pred.shape[1:]) or pred.shape[2] != 3 or pred.shape[1] < 1:
        raise ValueError(f"pred {tuple(pred.shape)} and gt {tuple(gt.shape)} must be [.., J, 3] poses on one device")
    pairs = _check_pairs(pred, gt, pairs)
    out = launch_pose_metrics(pred, gt, pairs, int(pred.shape[1]))
    return {k: out[:, i] for i, k in enumerate(POSE_METRICS)}


def best_of(scores, names):
    """Per metric, the sample with the best mean over the scored frames of a [nsample, F, B] score tensor, first on ties:
    (index [B], its curve [F, B])."""
    best = {}
    for k in names:
        v = scores[k]
        m = v.mean(1)
        idx = m.argmax(0) if HIGHER_IS_BETTER[k] else m.argmin(0)
        best[k] = (idx, v.gather(0, idx.view(1, 1, -1).expand(1, v.shape[1], -1))[0])
    return best
