#!/usr/bin/env python
"""Qualitative-picture fixture from the UNMODIFIED reference (build container only, the shims of make_golden.py plus):

  * stub ``imageio`` (mimsave recorded), ``misc.utils.get_progress_bar`` / ``clear_progressbar`` (silent), a capturing
    ``torchvision.utils.save_image`` and a recording writer (tests/vis_ref.Recorder);
  * ``np.float`` = float (the reference's h36m branch uses the alias NumPy 1.24 removed);
  * tests/vis_ref.PoseStub as the h36m visualizer.

  vis_seq.pt   the reference's own ``misc/visualize.py vis_seq`` on the CPU, in two kinds of cases (name: channels, B,
               nsample, seq_len, output_len, recon_mode, model_mode, skip_frame):
               * generation, with the reference's real ``P2PModel`` (eval mode, BatchNorm running statistics moved off
                 (0, 1) by make_golden_extra.warm_bn):
                   d64_c1_eq     dcgan_64, 1, 3, 3, 6, 6, 'test', full, False
                   d64_c1_above  dcgan_64, 1, 3, 4, 6, 8, None, posterior, True (skip_prob 0.5)
                   d64_c3_below  dcgan_64, 3, 3, 3, 7, 5, None, full, False
                   h36m          h36m_mlp, poses, 2, 3, 6, 8, 'test', prior, False
                 stored: the eps stream (torch.manual_seed(seed), one [B, z] normal_ per posterior / prior call), the poses
                 in full and the set_data calls (h36m), and for the frame cases a 2048-value digest of the saved canvas
                 (the generated frames themselves are too large to keep);
               * composition, with tests/vis_ref.FrameSource standing in for the model (seeded frames, some all-zero as
                 skipped frames are), so that the samples are redrawn from the stored seed:
                   syn_c1_eq     1, 3, 3, 6, 6, 'test', full, False
                   syn_c1_above  1, 3, 4, 6, 8, None, prior, False (frames 3 and 5 zero)
                   syn_c3_below  3, 12, 4, 7, 5, 'train', posterior, False (10 of the 12 rows drawn)
               Stored for every case: the NumPy seed, the nsample skip draws and the per-block s_lists (redrawn from the seed),
               sha256 of the saved canvas, the video tensor and the GIF frames, the file names, tags and steps, and NumPy's
               state afterwards.

    python tests/golden/make_golden_vis.py
"""
import hashlib
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import ROOT, import_reference, make_opt  # noqa: E402
from make_golden_extra import warm_bn  # noqa: E402

sys.path.insert(0, ROOT)
from oracle.p2p_oracle import tensor_digest  # noqa: E402
from tests.vis_ref import FrameSource, PoseStub, Recorder, case_input  # noqa: E402

CASES = {
    "d64_c1_eq": dict(net=64, channels=1, B=3, nsample=3, T=6, L=6, recon="test", mode="full", skip=False, opt={}),
    "d64_c1_above": dict(net=64, channels=1, B=3, nsample=4, T=6, L=8, recon=None, mode="posterior", skip=True,
                         opt=dict(skip_prob=0.5)),
    "d64_c3_below": dict(net=64, channels=3, B=3, nsample=3, T=7, L=5, recon=None, mode="full", skip=False, opt={}),
    "h36m": dict(net="mlp", B=2, nsample=3, T=6, L=8, recon="test", mode="prior", skip=False, opt={}),
    "syn_c1_eq": dict(net="source", channels=1, B=3, nsample=3, T=6, L=6, recon="test", mode="full", skip=False, zero=()),
    "syn_c1_above": dict(net="source", channels=1, B=3, nsample=4, T=6, L=8, recon=None, mode="prior", skip=False, zero=(3, 5)),
    "syn_c3_below": dict(net="source", channels=3, B=12, nsample=4, T=7, L=5, recon="train", mode="posterior", skip=False,
                         zero=()),
}
OPT_KEYS = ("beta", "weight_cpc", "weight_align", "skip_prob", "n_past", "last_frame_skip", "lr", "beta1", "batch_size")


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def install_stubs(rec):
    sys.modules["imageio"] = types.SimpleNamespace(mimsave=rec.imageio.mimsave)
    import torchvision.utils as vutils
    vutils.save_image = rec.vutils.save_image
    import misc.utils as mu
    bar = types.SimpleNamespace(update=lambda *a: None, finish=lambda: None)
    mu.get_progress_bar = lambda *a, **k: bar
    mu.clear_progressbar = lambda: None
    np.float = float


def run_case(name, c, p2p_model, backbones, rec):
    pose, source = c["net"] == "mlp", c["net"] == "source"
    torch.manual_seed(1)
    if source:
        opt = make_opt(None, batch_size=c["B"])
        c = dict(c, src_seed=5150 + len(name))
        model = FrameSource(c["src_seed"], c["zero"])
        cfg, bn = {}, {}
    elif pose:
        opt = make_opt(backbones["mlp"], dataset="h36m", batch_size=c["B"], **c["opt"])
        model = p2p_model.P2PModel(opt.batch_size, 1, 128, 10, 512, 1, 1, 2, opt=opt)
        model.eval()
        cfg = dict(g_dim=128, z_dim=10, rnn_size=512, backbone="mlp", predictor_rnn_layers=2, posterior_rnn_layers=1,
                   prior_rnn_layers=1)
        bn = {}
    else:
        opt = make_opt(backbones[c["net"]], batch_size=c["B"], **c["opt"])
        model = p2p_model.P2PModel(opt.batch_size, c["channels"], 128, 10, 256, 1, 1, 2, opt=opt)
        warm_bn(model, dict(channels=c["channels"], width=64), torch.Generator().manual_seed(4321))
        cfg = dict(g_dim=128, z_dim=10, rnn_size=256, channels=c["channels"], image_width=64, predictor_rnn_layers=2,
                   posterior_rnn_layers=1, prior_rnn_layers=1)
        mods = dict(encoder=model.encoder, decoder=model.decoder)
        bn = {m: {k: v.detach().clone() for k, v in mods[m].state_dict().items() if "running_" in k or "num_batches" in k}
              for m in mods}
    opt.nsample, opt.log_dir = c["nsample"], "LOGDIR"
    c = dict(c, x_seed=2468 + len(name))
    x = case_input(c)
    seed = 900 + len(name)
    calls = []
    hooks = [] if source else [getattr(model, m).register_forward_hook(lambda *a: calls.append(1)) for m in ("posterior", "prior")]
    vis = PoseStub() if pose else None
    for lst in (rec.saved, rec.gifs, rec.images, rec.videos):
        lst.clear()
    np.random.seed(seed)
    torch.manual_seed(seed)
    from misc import visualize
    with torch.no_grad():
        visualize.vis_seq(model, x, 7, c["L"], model_mode=c["mode"], recon_mode=c["recon"], skip_frame=c["skip"],
                          h36m_visualizer=vis, writer=rec, opt=opt)
    np_after = np.random.get_state()
    for h in hooks:
        h.remove()
    nb = min(c["B"], 5 if pose else 10)
    torch.manual_seed(seed)
    B_gen = nb if pose else c["B"]
    eps = torch.stack([torch.empty(B_gen, 10).normal_() for _ in calls]) if calls else torch.empty(0, B_gen, 10)
    rs = np.random.RandomState(seed)
    probs = [rs.uniform(0, 1, c["L"] - 1) for _ in range(c["nsample"])]
    s_lists = [[1] + [int(v) for v in rs.randint(c["nsample"], size=4)] for _ in range(nb)]
    assert rs.get_state()[2] == np_after[2] and (rs.get_state()[1] == np_after[1]).all()
    (png_name, canvas), = rec.saved
    (gif_name, gif), = rec.gifs
    (img_tag, img, img_step), = rec.images
    (vid_tag, vid, vid_step, fps), = rec.videos
    assert np.array_equal(img, canvas.numpy()) and vid.shape[0] == 1
    gif = np.stack(gif)
    fix = dict(case=name, spec=c, init_seed=1, cfg=cfg, opt={k: getattr(opt, k) for k in OPT_KEYS}, nsample=c["nsample"],
               bn_buffers=bn, np_seed=seed, probs=probs, s_lists=s_lists, eps=eps, n_calls=len(calls), n_block=nb,
               canvas=dict(shape=tuple(canvas.shape), sha=sha(canvas.numpy()), digest=tensor_digest(canvas, 32 if source else 2048)),
               video=dict(shape=tuple(vid.shape), dtype=str(vid.dtype), sha=sha(vid), digest=tensor_digest(torch.from_numpy(vid))),
               gif=dict(shape=tuple(gif.shape), n=len(rec.gifs[0][1]), dtype=str(gif.dtype), sha=sha(gif)),
               names=(png_name, gif_name), tags=(img_tag, vid_tag), steps=(img_step, vid_step), fps=fps,
               np_state_after=(np_after[0], np_after[1].copy(), np_after[2], np_after[3], np_after[4]))
    if pose:
        fix["set_data"] = [(p, v) for p, v in vis.calls]
    print(f"[{name}] canvas {tuple(canvas.shape)} gif {gif.shape} {png_name} {img_tag} s_lists {s_lists} eps {len(calls)}")
    return fix


def main():
    torch.set_num_threads(8)
    p2p_model, backbones = import_reference()
    rec = Recorder()
    install_stubs(rec)
    fix = dict(cases=[run_case(name, c, p2p_model, backbones, rec) for name, c in CASES.items()])
    path = os.path.join(HERE, "vis_seq.pt")
    torch.save(fix, path)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
