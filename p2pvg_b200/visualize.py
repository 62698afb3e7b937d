"""The reference's qualitative pictures (misc/visualize.py ``vis_seq``) on the graphed generator and one composition launch.

``vis_seq`` takes the reference's arguments and writes the same PNG and GIF files and TensorBoard entries.  Only the rows the
pictures show are generated: the first ``n_block`` = min(batch_size, 10) sequences (5 for h36m), all ``opt.nsample`` samples
in one CUDA-graph replay (``P2PModel.p2p_generate_graphed`` with nsample; eval-mode rows are independent, so a row does not
depend on the rows generated with it).  The picture is then composed by ONE p2pvg_vis_canvas launch from the graph's own input
and output buffers: control-point borders, the sample padding, the row blocks of the PNG canvas, the video frames and the
uint8 GIF frames (``plan_tiles`` holds the reference's layout rules, the kernel only gathers).

Random streams end where the reference's 20 eager ``p2p_generate`` calls leave them:
  * NumPy: the ``np.random.uniform(0, 1, L - 1)`` draw of each of the nsample calls, then per row block the
    ``np.random.randint(nsample, size=4)`` of its sample rows, in block order;
  * torch's CUDA generator: per call and executed step ``torch.randn(B, z_dim)`` for the posterior, then for the prior, at
    the reference's batch B (the whole test batch; n_block for h36m, which the reference slices first); rows [:n_block] of
    those draws are the graph's noise (``infer.eps_stream``).
With skip_frame=True every reference call has its own skip pattern, so the samples are nsample graphed calls of one sample.

Afterwards ``.hidden`` of the LSTMs holds the graph's nsample * n_block rows (the last call's n_block rows with
skip_frame=True); the reference's leaves the last call's B rows.  ``P2PModel.forward`` does not read it.

Poses (h36m): the n_block displayed sequences are generated graphed.  When ``h36m_visualizer`` is a
``p2pvg_b200.skeleton.Skeleton3DVisualizer`` the pose store (every sample's frames, then the ground truth padded to
output_len) and each image's camera view are assembled on the device and drawn by ONE p2pvg_skeleton_render launch straight
into the fp32 frame store, with no pose copied to the host.  Any other visualizer draws them with ``set_data`` in the
reference's order and with its arguments; the rendered images, scaled as the reference scales them, are uploaded as one
frame store.  Either store is composed by the same kernel, with the same tile table and the same random draws.

``check_vis_seq`` raises ValueError, before any draw or launch, for anything this path does not take.
"""
from __future__ import annotations

import numpy as np
import torch

from . import gen_engine, infer, skeleton

NROW = 6        # rows per block: the ground truth and five samples (misc/visualize.py:105)
ORANGE, RED = 1, 2


def n_block_of(opt):
    """Row blocks the reference draws (misc/visualize.py:111, 121)."""
    return min(int(opt.batch_size), 5 if opt.dataset == "h36m" else 10)


def file_names(opt, epoch, output_len, model_mode, recon_mode):
    """(png, gif) names of misc/visualize.py:231-234, 257-260, with their len_ / len- difference."""
    if recon_mode in ("train", "test"):
        stem = "%s/gen_vis/recon_%s-model_%s-len_%d-epoch_%d" % (opt.log_dir, recon_mode, model_mode, output_len, epoch)
    else:
        stem = "%s/gen_vis/gen-model_%s-len-%d-epoch_%d" % (opt.log_dir, model_mode, output_len, epoch)
    return stem + ".png", stem + ".gif"


def tags(output_len, model_mode, recon_mode):
    """(image tag, video tag) of misc/visualize.py:264-269."""
    if recon_mode in ("train", "test"):
        return "%s/%s-Gen" % (model_mode, recon_mode), "%s/%s-Video" % (model_mode, recon_mode)
    return "%s/Gen%d" % (model_mode, output_len), "%s/GenVideo%d" % (model_mode, output_len)


def plan_tiles(seq_len, output_len, n_block, nsample, gt_ref, sample_ref):
    """The tile table [r_len, n_block, 6, 3] int32 of p2pvg_vis_canvas, r_len = max(seq_len, output_len), drawing the
    reference's s_list of every row block from NumPy's global stream (misc/visualize.py:199) in block order.

    gt_ref(t) -> (store, frame of row 0) of ground-truth frame t < seq_len; sample_ref(s, t) -> the same for sample s's frame
    t < output_len, or None for a zero (skipped) frame; row b of a block is that frame + b.  Layout (misc/visualize.py:13-87,
    129-131, 176-227): row 0 of block i is the ground truth padded with its control point to output_len, with an orange
    border on frame 0 and a red one from frame seq_len - 1 on; rows 1-5 are samples [1] + s_list, padded to r_len with
    their frame output_len - 1, orange on frame 0 and red from output_len - 1 on."""
    r_len = max(seq_len, output_len)
    tiles = np.zeros((r_len, n_block, NROW, 3), np.int32)
    for i in range(n_block):
        s_list = [1] + list(np.random.randint(nsample, size=NROW - 2))
        for t in range(r_len):
            st, f = gt_ref(min(t, seq_len - 1))
            tiles[t, i, 0] = (st, f + i, RED if t >= seq_len - 1 else ORANGE if t == 0 else 0)
            for j, s in enumerate(s_list):
                ref = sample_ref(int(s), min(t, output_len - 1))
                st, f = (0, -1) if ref is None else (ref[0], ref[1] + i)
                tiles[t, i, j + 1] = (st, f, RED if t >= output_len - 1 else ORANGE if t == 0 else 0)
    return tiles


def compose(store0, store1, tiles, C, H):
    """ONE p2pvg_vis_canvas launch: (canvas [3, n_block*6*H, r_len*H] fp32, video [r_len, 3, n_block*H, 6*H] fp32, gif
    [r_len, n_block*H, 6*H, 3] uint8) on the stores' device.  store0 / store1: fp32 [n, C, H, H] frame stores (store1 may be
    None); tiles: plan_tiles' table."""
    from ._lib import kernels_for
    r_len, n_block = int(tiles.shape[0]), int(tiles.shape[1])
    dev = store0.device
    K = kernels_for(dev)
    fs = C * H * H
    stores = []
    for s in (store0, store1):
        if s is not None and (s.dtype != torch.float32 or not s.is_contiguous() or s.device != dev or s.numel() % fs):
            raise ValueError("compose takes contiguous fp32 frame stores of [n, C, H, H] frames on one device")
        stores.append((s, 0 if s is None else s.numel() // fs))
    tiles = np.ascontiguousarray(tiles, dtype=np.int32)
    canvas = torch.empty(3, n_block * NROW * H, r_len * H, device=dev)
    video = torch.empty(r_len, 3, n_block * H, NROW * H, device=dev)
    gif = torch.empty(r_len, n_block * H, NROW * H, 3, device=dev, dtype=torch.uint8)
    tiles_dev = torch.empty(tiles.size, device=dev, dtype=torch.int32)
    K.vis_canvas(stores[0][0], stores[0][1], stores[1][0], stores[1][1], C, H, tiles, tiles_dev, r_len, n_block, canvas, video,
                 gif)
    return canvas, video, gif


def _model_device(model):
    p = next(model.parameters(), None)
    return None if p is None else p.device


def check_vis_seq(model, x, output_len, model_mode="full", skip_frame=True, opt=None):
    """ValueError unless vis_seq below takes these arguments: a model p2p_generate_graphed takes (eval mode, on a CUDA
    device, a supported backbone and frame shape), opt.nsample >= 2 (the reference shows sample 1 in every block), at least
    n_block sequences in x, 1- or 3-channel square frames of at most 128 pixels.  Makes no draw and no launch."""
    opt = model.opt if opt is None else opt
    pose = getattr(opt, "dataset", None) == "h36m"
    if pose != bool(getattr(model, "is_pose", False)):
        raise ValueError("vis_seq: opt.dataset and the model's backbone disagree about poses")
    if not hasattr(model, "_graphed_engine"):
        raise ValueError("vis_seq needs a p2pvg_b200 P2PModel")
    eng = model._graphed_engine()
    eng._check_model()
    nsample = int(opt.nsample)
    if nsample < 2:
        raise ValueError(f"vis_seq needs opt.nsample >= 2 (got {nsample}): the reference shows sample 1 in every row block")
    if model_mode not in ("full", "posterior", "prior"):
        raise ValueError(f"unknown model_mode {model_mode!r}")
    dev = _model_device(model)
    if dev is None or dev.type != "cuda":
        raise ValueError("vis_seq runs on a CUDA device: move the model there first (model.cuda())")
    frames = x[1] if pose else x
    if pose and (not isinstance(x, (tuple, list)) or len(x) != 3):
        raise ValueError("vis_seq takes the (pose_2d, pose_3d, camera_view) tuple for h36m")
    seq_len = len(frames)
    f0 = frames[0]
    if not torch.is_tensor(f0) or f0.device != dev:
        raise ValueError(f"vis_seq: the frames must be tensors on the model's device {dev}")
    eng._frame_shape(f0)
    nb = n_block_of(opt)
    if int(f0.shape[0]) < nb:
        raise ValueError(f"vis_seq draws {nb} row blocks but x has {int(f0.shape[0])} sequences")
    if not pose:
        C, H, W = (int(v) for v in f0.shape[1:])
        if C not in (1, 3) or H != W or H > 128:
            raise ValueError(f"vis_seq composes 1- or 3-channel square frames of at most 128 pixels (got {C}x{H}x{W})")
    L, n_past = int(output_len), int(model.opt.n_past)
    if L < 2 or n_past < 1 or seq_len < min(n_past, L) or seq_len < 2:
        raise ValueError(f"vis_seq needs output_len >= 2, n_past >= 1 and at least max(2, min(n_past, output_len)) input frames "
                         f"(output_len {L}, n_past {n_past}, {seq_len} frames)")


def _eps(B, z, dev, n_exec, nb):
    """The reference call's posterior / prior draws: per executed step torch.randn(B, z) twice on the device's generator,
    rows [:nb] kept.  Returns [n_exec, 2, nb, z]."""
    out = torch.empty(n_exec, 2, nb, z, device=dev)
    for k in range(n_exec):
        for j in (0, 1):
            out[k, j] = torch.randn(B, z, device=dev)[:nb]
    return out


def _skip_draw_peek(L):
    st = np.random.get_state()
    probs = np.random.uniform(0, 1, L - 1)
    np.random.set_state(st)
    return probs


def _generate_skip(model, xg, L, model_mode, nsample, B, nb, seq_len):
    """skip_frame=True: nsample graphed calls of one sample, each with the reference call's own NumPy skip draw and noise.
    Returns the stacked frames [nsample * L * nb, ...] (sample s, frame t, row b at (s * L + t) * nb + b)."""
    opt, dev = model.opt, _model_device(model)
    out = []
    for _ in range(nsample):
        sl = gen_engine.plan_slots(L, seq_len, _skip_draw_peek(L), float(opt.skip_prob), int(opt.n_past), True, L - 1)
        eps = _eps(B, model.z_dim, dev, len(sl), nb)
        with infer.eps_stream([e for k in range(len(sl)) for e in (eps[k, 0], eps[k, 1])]):
            seq = model.p2p_generate_graphed(xg, L, L - 1, model_mode=model_mode, skip_frame=True)
        out.append(torch.stack(seq))
    return torch.stack(out).reshape(nsample * L * nb, *seq[0].shape[1:]).contiguous()


def _generate_batched(model, L, nsample, B, nb, run):
    """skip_frame=False: the nsample calls' noise for the nsample * nb rows of one replay (sample-major), the nsample - 1
    NumPy skip draws the one call does not make, then run() inside infer.eps_stream."""
    dev = _model_device(model)
    S = L - 1
    eps = torch.stack([_eps(B, model.z_dim, dev, S, nb) for _ in range(nsample)], 2)   # [S, 2, nsample, nb, z]
    for _ in range(nsample - 1):
        np.random.uniform(0, 1, L - 1)
    with infer.eps_stream([eps[k, j].reshape(nsample * nb, -1) for k in range(S) for j in (0, 1)]):
        return run()


def _render(vis, poses, camera_view, nb):
    """h36m_visualizer.set_data per sequence b of poses [T, nb, 17, 3] (misc/visualize.py:154-159, 169-173): fp32 images
    [T, nb, C, H, W] scaled as the reference scales them (uint8 -> float64 / 255 -> float32)."""
    imgs = [np.asarray(vis.set_data(poses[:, b].cpu().numpy(), camera_view[b].item())) for b in range(nb)]
    a = np.stack(imgs, 1).astype(np.float64) / 255.
    return torch.from_numpy(a.astype(np.float32)).permute(0, 1, 4, 2, 3)


def vis_seq(model, x, epoch, output_len, model_mode='full', recon_mode=None, skip_frame=True, h36m_visualizer=None, writer=None,
            opt=None, save_png=None, save_gif=None):
    """misc/visualize.py vis_seq (same arguments, files and TensorBoard entries) on the graphed generator and one
    p2pvg_vis_canvas launch; see the module docstring.  ``save_png(canvas, file_name)`` writes the PNG file
    (torchvision.utils.save_image when None; p2pvg_b200.png.save_image encodes it on the GPU).  ``save_gif(file_name,
    gif)`` writes the GIF file from the device's uint8 frames (imageio.mimsave of their host copy when None;
    p2pvg_b200.gif.save_gif encodes it on the GPU).  ValueError before any draw
    or launch when check_vis_seq rejects the arguments.  Returns (canvas, video, gif) on the device."""
    opt = model.opt if opt is None else opt
    check_vis_seq(model, x, output_len, model_mode, skip_frame, opt)
    import torchvision.utils as vutils
    nsample, nb, L = int(opt.nsample), n_block_of(opt), int(output_len)
    pose = opt.dataset == "h36m"
    dev = _model_device(model)
    with torch.no_grad():
        if pose:
            pose_2d, pose_3d, camera_view = x
            xg = (pose_2d[:, :nb], pose_3d[:, :nb], camera_view[:nb])
            frames, B = pose_3d[:, :nb], nb
        else:
            frames = x if torch.is_tensor(x) else torch.stack(list(x))
            B = int(frames.shape[1])
            frames = frames[:, :nb]
            xg = frames
        seq_len = len(frames)
        if skip_frame:
            samples = _generate_skip(model, xg, L, model_mode, nsample, B, nb, seq_len)
            sample_ref = lambda s, t: (1, (s * L + t) * nb)   # noqa: E731  (skipped frames are zeros in the store)
        elif not pose:
            def plan(gt_ref, sref):
                return plan_tiles(seq_len, L, nb, nsample, gt_ref, sref)
            canvas, video, gif = _generate_batched(
                model, L, nsample, B, nb, lambda: model._graphed_engine().vis_canvas(xg, L, model_mode, nsample, plan))
        else:
            seqs = _generate_batched(model, L, nsample, B, nb,
                                     lambda: model.p2p_generate_graphed(xg, L, L - 1, model_mode=model_mode, nsample=nsample))
            samples = torch.stack([torch.stack(s) for s in seqs]).reshape(nsample * L * nb, 17, 3)
            sample_ref = lambda s, t: (1, (s * L + t) * nb)   # noqa: E731
        if pose:
            # the reference's set_data order: every sample's sequences, then the ground truth padded to output_len
            gt = torch.cat([frames, frames[-1:].expand(max(L - seq_len, 0), *frames.shape[1:])])
            if isinstance(h36m_visualizer, skeleton.Skeleton3DVisualizer):
                # the same store drawn on the device: sample s frame t row b at (s L + t) nb + b, then the ground truth
                poses = torch.cat([samples.reshape(-1, *samples.shape[-2:]), gt.reshape(-1, *gt.shape[-2:]).float()])
                views = camera_view[:nb].repeat(poses.shape[0] // nb)
                store, C, H = h36m_visualizer.render_device(poses, views), 3, skeleton.SIZE
            else:
                sp = samples.view(nsample, L, nb, 17, 3)
                imgs = [_render(h36m_visualizer, sp[s], camera_view, nb) for s in range(nsample)]
                imgs.append(_render(h36m_visualizer, gt, camera_view, nb))
                C, H, W = imgs[0].shape[2:]
                if C not in (1, 3) or H != W or H > 128:
                    raise ValueError(f"vis_seq composes 1- or 3-channel square images of at most 128 pixels; the visualizer "
                                     f"drew {C}x{H}x{W}")
                store = torch.cat([i.reshape(-1, C, H, W) for i in imgs]).to(dev).contiguous()
            g0 = nsample * L * nb
            tiles = plan_tiles(seq_len, L, nb, nsample, lambda t: (0, g0 + t * nb), lambda s, t: (0, (s * L + t) * nb))
            canvas, video, gif = compose(store, None, tiles, C, H)
        elif skip_frame:
            store0 = frames.reshape(seq_len * nb, *frames.shape[2:]).float().contiguous()
            tiles = plan_tiles(seq_len, L, nb, nsample, lambda t: (0, t * nb), sample_ref)
            canvas, video, gif = compose(store0, samples, tiles, int(frames.shape[2]), int(frames.shape[3]))
    png_name, gif_name = file_names(opt, epoch, output_len, model_mode, recon_mode)
    (vutils.save_image if save_png is None else save_png)(canvas, png_name)
    if save_gif is None:
        import imageio
        imageio.mimsave(gif_name, list(gif.cpu().numpy()))
    else:
        save_gif(gif_name, gif)
    img_tag, vid_tag = tags(output_len, model_mode, recon_mode)
    writer.add_image(img_tag, canvas.cpu().numpy(), epoch)
    writer.add_video(vid_tag, video.unsqueeze(0).cpu().numpy(), epoch, fps=2)
    return canvas, video, gif
