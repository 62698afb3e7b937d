"""The reference's generate.py on the GPU: one start/end pair generated at several lengths and written out as PNG and GIF files.

``generate_video`` writes the files the reference's script writes, with the same pictures (per length L:
``len_L-gt.png``, ``len_L-gen_%03d.png`` and ``len_L-gen_%03d.gif`` per displayed sample, ``len_L-gen_full.png`` and
``len_L-gen_full.gif``).  Every length and sample comes from ONE ``P2PModel.p2p_generate_lengths`` replay (the rows of the
shorter lengths stop early), and every picture of every length from ONE p2pvg_vis_tiles launch that reads the graph's own
input and output buffers: ``plan_video`` holds the reference's layout rules (control-point borders, the ground truth padded
with its control point, ``padding=0`` grids), the kernel only gathers.  Per-sample PNG rows are row slices of the block
canvas and per-sample GIF frames column slices of the full GIF frames, so per length the kernel writes three things.

Random streams end where the reference's loop of nsamples eager ``p2p_generate`` calls per length leaves them:
  * NumPy, per length in order: nsamples ``np.random.uniform(0, 1, L - 1)`` skip draws, then
    ``np.random.choice(nsamples, ndisplays, replace=False)``;
  * torch's CUDA generator: per eager call and executed step ``torch.randn(B, z_dim)`` for the posterior, then the prior;
    those draws are the replay's noise (``infer.eps_stream``).

``python -m p2pvg_b200.generate --ckpt model.pth --video clip.mp4 [--output_root gen_outputs] [--seed 1]`` runs the
reference's script: same arguments, same seeding (``random``, ``torch``, ``torch.cuda``; NumPy is not seeded), a batch-1
model built from the checkpoint's options, the video read with imageio.
"""
from __future__ import annotations

import argparse
import os
import random

import numpy as np
import torch

from . import infer
from .visualize import ORANGE, RED, _eps, _model_device

GEN_LENGTHS = (10, 20, 30)   # generate.py:92-95
NSAMPLES = NDISPLAYS = 5


def file_names(output_root, L, ndisplays):
    """The files generate.py writes for length L, in its order."""
    return (["%s/len_%d-gt.png" % (output_root, L)] + ["%s/len_%d-gen_%03d.png" % (output_root, L, ix) for ix in range(ndisplays)]
            + ["%s/len_%d-gen_full.png" % (output_root, L)]
            + ["%s/len_%d-gen_%03d.gif" % (output_root, L, ix) for ix in range(ndisplays)]
            + ["%s/len_%d-gen_full.gif" % (output_root, L)])


def plan_video(seq_len, lens, idxs, H, gt_ref, sample_ref):
    """The tables of p2pvg_vis_tiles for every length: (images int64 [3 * len(lens), 4], tiles int32 [n, 6], layout).

    gt_ref(t) -> (store, frame) of ground-truth frame t < seq_len; sample_ref(k, s, t) -> the same for frame t of sample s of
    length lens[k]; idxs[k]: the displayed samples of length k (np.random.choice).  Per length three images (layout[k] =
    their (offset, shape)): the ground-truth strip fp32 [3, H, R * H], R = max(seq_len, L), padded with its control point,
    orange on frame 0 and red from frame seq_len - 1 on (misc/visualize.py add_gt_cp_border); the block canvas fp32
    [3, nd * H, L * H], displayed sample ix in rows ix * H, orange on frame 0 and red on frame L - 1 (add_samples_cp_border);
    the full GIF frames uint8 [L, H, nd * H, 3], frame t of sample ix at columns ix * H."""
    images, tiles, layout = [], [], []
    off_f = off_u = 0
    for k, L in enumerate(lens):
        R, nd = max(seq_len, L), len(idxs[k])
        gi, bi, fi = len(images), len(images) + 1, len(images) + 2
        images += [(off_f, 0, H, R * H), (off_f + 3 * H * R * H, 0, nd * H, L * H), (off_u, 1, L * H, nd * H)]
        layout.append(((off_f, (3, H, R * H)), (off_f + 3 * H * R * H, (3, nd * H, L * H)), (off_u, (L, H, nd * H, 3))))
        off_f += 3 * H * R * H + 3 * nd * H * L * H
        off_u += 3 * L * H * nd * H
        for t in range(R):
            st, f = gt_ref(min(t, seq_len - 1))
            tiles.append((st, f, RED if t >= seq_len - 1 else ORANGE if t == 0 else 0, gi, 0, t * H))
        for ix, s in enumerate(idxs[k]):
            for t in range(L):
                st, f = sample_ref(k, int(s), t)
                border = RED if t == L - 1 else ORANGE if t == 0 else 0
                tiles.append((st, f, border, bi, ix * H, t * H))
                tiles.append((st, f, border, fi, t * H, ix * H))
    return (np.array(images, np.int64).reshape(-1, 4), np.array(tiles, np.int32).reshape(-1, 6), layout, off_f, off_u)


def compose(store0, store1, plan, C, H):
    """ONE p2pvg_vis_tiles launch for plan_video's plan: per length (gt strip, block canvas, full GIF frames) on the device."""
    from ._lib import kernels_for
    images, tiles, layout, n_f, n_u8 = plan
    dev = store0.device
    fs = C * H * H
    stores = []
    for s in (store0, store1):
        if s is not None and (s.dtype != torch.float32 or not s.is_contiguous() or s.device != dev or s.numel() % fs):
            raise ValueError("compose takes contiguous fp32 frame stores of [n, C, H, H] frames on one device")
        stores.append((s, 0 if s is None else s.numel() // fs))
    out_f = torch.empty(n_f, device=dev)
    out_u8 = torch.empty(n_u8, device=dev, dtype=torch.uint8)
    tables = torch.empty(4 * len(images) + 3 * len(tiles), device=dev, dtype=torch.int64)
    kernels_for(dev).vis_tiles(stores[0][0], stores[0][1], stores[1][0], stores[1][1], C, H, np.ascontiguousarray(tiles),
                               np.ascontiguousarray(images), tables, out_f, out_u8)
    return [tuple((out_f if len(shape) == 3 else out_u8)[o:o + int(np.prod(shape))].view(shape) for o, shape in lay)
            for lay in layout]


def check_generate(model, seq, gen_lengths, nsamples, ndisplays):
    """ValueError unless generate_video takes these arguments: a model p2p_generate_graphed takes (not h36m, on a CUDA
    device), seq [T, 1, C, H, H] on its device with C 1 or 3 and H <= 128, lengths generate_lengths takes,
    1 <= ndisplays <= nsamples.  Makes no draw and no launch."""
    from .gen_engine import check_lengths
    if getattr(model, "is_pose", False):
        raise ValueError("generate_video draws image frames; h36m poses are drawn by vis_seq (p2pvg_b200.skeleton)")
    if not hasattr(model, "_graphed_engine"):
        raise ValueError("generate_video needs a p2pvg_b200 P2PModel")
    model._graphed_engine()._check_model()
    dev = _model_device(model)
    if dev is None or dev.type != "cuda":
        raise ValueError("generate_video runs on a CUDA device: move the model there first (model.cuda())")
    if not torch.is_tensor(seq) or seq.dim() != 5 or int(seq.shape[1]) != 1 or seq.device != dev:
        raise ValueError("generate_video takes seq as a [T, 1, C, H, W] tensor on the model's device (generate.py's read_video)")
    C, H, W = (int(v) for v in seq.shape[2:])
    if C not in (1, 3) or H != W or H > 128:
        raise ValueError(f"generate_video composes 1- or 3-channel square frames of at most 128 pixels (got {C}x{H}x{W})")
    model._graphed_engine()._frame_shape(seq[0])
    if not 1 <= int(ndisplays) <= int(nsamples):
        raise ValueError(f"generate_video needs 1 <= ndisplays <= nsamples (got {ndisplays}, {nsamples})")
    return check_lengths(gen_lengths, len(seq), int(model.opt.n_past))


def generate_video(model, seq, output_root, gen_lengths=GEN_LENGTHS, nsamples=NSAMPLES, ndisplays=NDISPLAYS):
    """generate.py's loop (:108-163): the same files in output_root, the same pictures, the random streams left where it
    leaves them; see the module docstring.  ValueError (check_generate) before any draw or launch.  Returns per length
    (gt strip [3, H, R * H], block canvas [3, nd * H, L * H], GIF frames uint8 [L, H, nd * H, 3]) on the device."""
    lens = check_generate(model, seq, gen_lengths, nsamples, ndisplays)
    imageio = _imageio()
    dev, z = _model_device(model), model.z_dim
    T, C, H = len(seq), int(seq.shape[2]), int(seq.shape[3])
    eng = model._graphed_engine()
    with torch.no_grad():
        draws = []
        for L in lens:   # the eager calls' draws: per call and executed step, the posterior's then the prior's
            e = torch.stack([_eps(1, z, dev, L - 1, 1) for _ in range(nsamples)], 2)   # [L - 1, 2, nsamples, 1, z]
            draws += [e[s, j].reshape(nsamples, z) for s in range(L - 1) for j in (0, 1)]
        st = np.random.get_state()
        with infer.eps_stream(draws):
            G, _, _, order = eng._replay_lengths(seq, lens, "full", nsamples)
        # NumPy as the reference's loop leaves it: per length nsamples skip draws, then the displayed samples
        np.random.set_state(st)
        idxs = []
        for L in lens:
            for _ in range(nsamples):
                np.random.uniform(0, 1, L - 1)
            idxs.append(np.random.choice(nsamples, ndisplays, replace=False))
        c = G.cfg
        n_past, rows, gr = c["n_past"], c["rows"], c["grows"]

        def sample_ref(k, s, t):
            if t < n_past:   # frame 0 and the teacher-forced frames are the input's
                return 0, t
            return 1, (t - n_past) * rows + order.index(k) * gr + s

        plan = plan_video(T, lens, idxs, H, lambda t: (0, t), sample_ref)
        pics = compose(G.bufs["x"], G.bufs["out"], plan, C, H)
    write_files(output_root, lens, pics, ndisplays, imageio)
    return pics


def write_files(output_root, lens, pics, ndisplays, imageio):
    """generate.py's files from compose's pictures, in its order: PNGs with torchvision's save_image, GIFs with
    imageio.mimsave; the per-sample PNGs are row slices of the block canvas, the per-sample GIFs column slices of the full
    GIF frames."""
    import torchvision.utils as vutils
    os.makedirs(output_root, exist_ok=True)
    for L, (gt, block, gif) in zip(lens, pics):
        H = int(gt.shape[1])
        names = iter(file_names(output_root, L, ndisplays))
        gt, block, gif = gt.cpu(), block.cpu(), gif.cpu().numpy()
        vutils.save_image(gt, next(names))
        for ix in range(ndisplays):
            vutils.save_image(block[:, ix * H:(ix + 1) * H], next(names))
        vutils.save_image(block, next(names))
        for ix in range(ndisplays):
            imageio.mimsave(next(names), [np.ascontiguousarray(f[:, ix * H:(ix + 1) * H]) for f in gif])
        imageio.mimsave(next(names), list(gif))


def _imageio():
    try:
        import imageio
    except ImportError:
        raise RuntimeError("reading videos and writing GIFs needs the imageio package (pip install imageio imageio-ffmpeg)") \
            from None
    return imageio


def read_video(vid_name):
    """generate.py's read_video: the video's frames as a float32 [T, 1, C, H, W] tensor in [0, 1]."""
    imageio = _imageio()
    frames = [torch.from_numpy((np.asarray(im) / 255.).astype(np.float32)) for im in imageio.get_reader(vid_name)]
    return torch.stack(frames).permute(0, 3, 1, 2).unsqueeze(1)


def backbone_of(opt):
    """The backbone module generate.py picks from a checkpoint's options (:52-66); ValueError for h36m."""
    if opt.dataset == "h36m":
        raise ValueError("h36m checkpoints are not supported: the reference's generate.py reads an mp4 video and has no "
                         "pose path")
    from .models import dcgan_64, dcgan_128, vgg_64, vgg_128
    nets = {("dcgan", 64): dcgan_64, ("dcgan", 128): dcgan_128, ("vgg", 64): vgg_64, ("vgg", 128): vgg_128}
    net = nets.get((opt.backbone, int(opt.image_width)))
    if net is None:
        raise ValueError(f"Unknown backbone: {opt.backbone} at image_width {opt.image_width}")
    return net


def main(argv=None):
    parser = argparse.ArgumentParser(description="generate.py on the GPU: one video's first and last frames generated at "
                                                 "lengths 10, 20 and 30, 5 samples each, written as PNG and GIF files")
    parser.add_argument('--ckpt', type=str, default='', help='your model.pth file')
    parser.add_argument('--video', type=str, default='', help='your .mp4 video file')
    parser.add_argument('--output_root', type=str, default='gen_outputs')
    parser.add_argument('--seed', type=int, default=1, help='seed to use')
    args = parser.parse_args(argv)
    if not args.video:
        parser.error("--video is required")
    from .models.p2p_model import P2PModel
    states = torch.load(args.ckpt, weights_only=False)
    opt = states['opt']
    opt.backbone_net = backbone_of(opt)
    random.seed(args.seed)
    torch.manual_seed(args.seed)
    torch.cuda.manual_seed_all(args.seed)
    model = P2PModel(1, opt.channels, opt.g_dim, opt.z_dim, opt.rnn_size, opt.prior_rnn_layers, opt.posterior_rnn_layers,
                     opt.predictor_rnn_layers, opt=opt)
    model.cuda()
    model.load(states=states)
    model.eval()
    seq = read_video(args.video).cuda()
    generate_video(model, seq, args.output_root or 'gen_outputs')


if __name__ == "__main__":
    main()
