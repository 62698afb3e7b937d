"""Test-side restatements for p2pvg_b200.visualize (tests/test_vis_*.py, tools/bench_vis_seq.py, tests/golden/make_golden_vis.py).

  compose_ref      the reference's composition (misc/visualize.py:13-87, 129-131, 176-254) of gt frames [T_gt, n, C, H, W]
                   and samples [nsample, L, n, C, H, W] with given s_lists, in plain torch / NumPy: (canvas, video, gif)
  compose_tiles    a torch statement of p2pvg_vis_canvas: the same three outputs gathered from a tile table
  vis_seq_ref      the reference's vis_seq restated over the model's eager p2p_generate (same draws, files and entries)
  PoseStub         a deterministic stand-in for the h36m visualizer: set_data maps poses to small uint8 images
  FrameSource      a stand-in model whose p2p_generate returns seeded frames (the composition cases of the fixture)
  Recorder         fake imageio / torchvision.utils / writer that record what they are given
"""
import types

import numpy as np
import torch

ORANGE = (1.0, 165. / 255., 0.0)
RED = (1.0, 0.0, 0.0)


def case_input(c):
    """The input of a tests/golden/vis_seq.pt case, redrawn from its seed."""
    g = torch.Generator().manual_seed(c["x_seed"])
    if c["net"] == "mlp":
        T, B = c["T"], c["B"]
        return (torch.randn(T, B, 17, 2, generator=g), 3 * torch.randn(T, B, 17, 3, generator=g), torch.arange(B) % 4)
    return torch.rand(c["T"], c["B"], c["channels"], 64, 64, generator=g)


class FrameSource:
    """Stands in for P2PModel where only the composition is under test: p2p_generate(x, output_len, ...) makes the
    reference's NumPy skip draw (models/p2p_model.py:128) and returns x[0], then output_len - 1 frames torch.rand(x[0].shape)
    from a generator seeded with seed + the call's index, the frames in `zero` all zeros (as skipped frames are).  So the
    fixture's samples are redrawn from two numbers, like its inputs."""

    def __init__(self, seed, zero=()):
        self.seed, self.zero, self.calls = seed, set(zero), 0

    def _frames(self, x, output_len, call):
        g = torch.Generator().manual_seed(self.seed + call)
        out = [x[0]]
        for i in range(1, output_len):
            f = torch.rand(x[0].shape, generator=g)
            out.append(torch.zeros_like(f) if i in self.zero else f)
        return out

    def p2p_generate(self, x, output_len, eval_cp_ix, start_ix=0, cp_ix=-1, model_mode="full", skip_frame=False):
        np.random.uniform(0, 1, output_len - 1)
        self.calls += 1
        return self._frames(x, output_len, self.calls - 1)

    def samples(self, x, nsample, output_len):
        """[nsample, output_len, B, ...]: what calls 0 .. nsample - 1 return (no draw)."""
        return torch.stack([torch.stack(self._frames(x, output_len, k)) for k in range(nsample)])


def _border(f, color, pad=3):
    """f [..., 3, H, W]: a copy with a pad-pixel frame of `color` (the interior [pad:W-pad, pad:W-pad] kept)."""
    H, W = f.shape[-2:]
    out = torch.empty_like(f)
    for c in range(3):
        out[..., c, :, :] = color[c]
    out[..., pad:W - pad, pad:W - pad] = f[..., pad:W - pad, pad:W - pad]
    return out


def compose_ref(gt, samples, seq_len, output_len, s_lists):
    """gt [seq_len, n, C, H, W] (before padding), samples [nsample, output_len, n, C, H, W] -> (canvas, video, gif)."""
    if gt.shape[2] == 1:
        gt, samples = gt.expand(-1, -1, 3, -1, -1), samples.expand(-1, -1, -1, 3, -1, -1)
    r_len = max(seq_len, output_len)
    g = [gt[t] for t in range(seq_len)] + [gt[seq_len - 1]] * max(output_len - seq_len, 0)
    g[0] = _border(g[0], ORANGE)
    for t in range(seq_len - 1, len(g)):
        g[t] = _border(gt[seq_len - 1], RED)
    sm = [samples[:, t] for t in range(output_len)]
    sm[0] = _border(sm[0], ORANGE)
    sm[output_len - 1] = _border(sm[output_len - 1], RED)
    sm += [sm[output_len - 1]] * (r_len - output_len)
    g, sm = torch.stack(g), torch.stack(sm, 1)                      # [r_len, n, 3, H, W], [ns, r_len, n, 3, H, W]
    n, H, W = g.shape[1], g.shape[-2], g.shape[-1]
    blocks = torch.stack([torch.stack([g[:, i]] + [sm[s, :, i] for s in s_lists[i]]) for i in range(n)])  # [n, 6, r, 3, H, W]
    canvas = blocks.permute(3, 0, 1, 4, 2, 5).reshape(3, n * 6 * H, r_len * W)
    video = blocks.permute(2, 3, 0, 4, 1, 5).reshape(r_len, 3, n * H, 6 * W)
    gif = (video.permute(0, 2, 3, 1).cpu().numpy() * 255).astype(np.uint8)
    return canvas.contiguous(), video.contiguous(), gif


def compose_tiles(store0, store1, tiles, C, H):
    """Torch statement of p2pvg_vis_canvas (include/p2pvg_b200.h)."""
    r_len, n, nrow, _ = tiles.shape
    zero = torch.zeros(C, H, H, dtype=store0.dtype, device=store0.device)
    out = torch.empty(r_len, n, nrow, 3, H, H, dtype=store0.dtype, device=store0.device)
    colors = {1: ORANGE, 2: RED}
    for t in range(r_len):
        for i in range(n):
            for j in range(nrow):
                st, f, b = (int(v) for v in tiles[t, i, j])
                fr = zero if f < 0 else (store0 if st == 0 else store1).view(-1, C, H, H)[f]
                fr = fr.expand(3, H, H) if C == 1 else fr
                out[t, i, j] = _border(fr, colors[b]) if b else fr
    canvas = out.permute(3, 1, 2, 4, 0, 5).reshape(3, n * nrow * H, r_len * H)
    video = out.permute(0, 3, 1, 4, 2, 5).reshape(r_len, 3, n * H, nrow * H)
    gif = (video.permute(0, 2, 3, 1).cpu().numpy() * 255).astype(np.uint8)
    return canvas.contiguous(), video.contiguous(), gif


class PoseStub:
    """set_data(pose_3d [T, 17, 3], camera_view) -> uint8 [T, S, S, 3]: pixel (y, x, c) = 255 * (0.5 + 0.5 tanh(p / 3 +
    0.1 view)) truncated, p = pose[t, (y S + x) % 17, c].  Records its calls."""

    def __init__(self, size=16):
        self.size, self.calls = size, []

    def set_data(self, pose_3d, camera_view):
        self.calls.append((np.array(pose_3d, copy=True), camera_view))
        S = self.size
        j = (np.arange(S * S) % 17).reshape(S, S)
        p = np.asarray(pose_3d, np.float64)[:, j, :]                  # [T, S, S, 3]
        return (255 * (0.5 + 0.5 * np.tanh(p / 3 + 0.1 * camera_view))).astype(np.uint8)


class Recorder:
    """fake imageio (mimsave), torchvision.utils (save_image) and SummaryWriter (add_image, add_video)."""

    def __init__(self):
        self.saved, self.gifs, self.images, self.videos = [], [], [], []
        self.imageio = types.SimpleNamespace(mimsave=lambda name, frames: self.gifs.append((name, [np.array(f) for f in frames])))
        self.vutils = types.SimpleNamespace(save_image=lambda t, name: self.saved.append((name, t.detach().cpu().clone())))

    def add_image(self, tag, img, step):
        self.images.append((tag, img, step))

    def add_video(self, tag, vid, step, fps=None):
        self.videos.append((tag, vid, step, fps))


def vis_seq_ref(model, x, epoch, output_len, model_mode="full", recon_mode=None, skip_frame=True, h36m_visualizer=None,
                writer=None, opt=None, rec=None):
    """The reference's vis_seq restated (generation by the model's eager p2p_generate on the whole batch, nsample calls;
    the pictures by compose_ref), writing through the Recorder rec."""
    from p2pvg_b200 import visualize as V
    nsample, nb = int(opt.nsample), V.n_block_of(opt)
    pose = opt.dataset == "h36m"
    with torch.no_grad():
        if pose:
            p2, p3, cam = x
            x = (p2[:, :nb], p3[:, :nb], cam[:nb])
            gt = p3[:, :nb]
        else:
            gt = x[:, :nb] if torch.is_tensor(x) else torch.stack(list(x))[:, :nb]
        seq_len = len(gt)
        samples = []
        for _ in range(nsample):
            seq = model.p2p_generate(x, output_len, output_len - 1, model_mode=model_mode, skip_frame=skip_frame)
            samples.append(torch.stack(seq)[:, :nb])
        samples = torch.stack(samples)
        if pose:
            def render(poses):
                ims = [h36m_visualizer.set_data(poses[:, b].cpu().numpy(), cam[b].item()) for b in range(nb)]
                return torch.from_numpy((np.stack(ims, 1).astype(np.float64) / 255.).astype(np.float32)).permute(0, 1, 4, 2, 3)
            samples = torch.stack([render(samples[s]) for s in range(nsample)])
            gpad = torch.cat([gt, gt[-1:].expand(max(output_len - seq_len, 0), *gt.shape[1:])])
            gt = render(gpad)[:seq_len]
        s_lists = [[1] + list(np.random.randint(nsample, size=4)) for _ in range(nb)]
        canvas, video, gif = compose_ref(gt.float(), samples.float(), seq_len, output_len, s_lists)
    png, gifn = V.file_names(opt, epoch, output_len, model_mode, recon_mode)
    rec.vutils.save_image(canvas, png)
    rec.imageio.mimsave(gifn, list(gif))
    it, vt = V.tags(output_len, model_mode, recon_mode)
    writer.add_image(it, canvas.cpu().numpy(), epoch)
    writer.add_video(vt, video.unsqueeze(0).cpu().numpy(), epoch, fps=2)
    return canvas, video, gif
