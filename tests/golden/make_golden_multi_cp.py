#!/usr/bin/env python
"""Multi-control-point generation fixture from the UNMODIFIED reference (build container only, same shims as make_golden.py):

  multi_cp_gen.pt   the reference's own ``P2PModel.p2p_generate`` (models/p2p_model.py:80-183) chained through control
                    points by hand, as its ``init_hidden`` flag allows: segment 0 of x[cp_ixs[0] : cp_ixs[1] + 1] with
                    init_hidden=True, every later segment x[cp_ixs[k] : cp_ixs[k + 1] + 1] with init_hidden=False (the LSTM
                    state of the previous segment), each with len_outputs[k] frames and eval_cp_ix = len_outputs[k] - 1.
                    Eval mode, BatchNorm on running statistics moved off (0, 1) by make_golden_extra.warm_bn.  Cases:
                      d64_np1      dcgan_64, 1 channel, B = 2, n_past 1, 3 unequal segments, one len_output longer than
                                   its slice (the posterior falls back to h_cpaw there)
                      d64_np2_lfs  dcgan_64, 1 channel, B = 2, n_past 2 + last_frame_skip, 3 unequal segments
                      vgg64_rgb    vgg_64, 3 channels, B = 1, n_past 1, 2 segments
                      h36m_np1     h36m_mlp (rnn_size 512), B = 2, n_past 1, 3 segments
                    each for skip_frame in {False, True} x model_mode in {full, one of posterior / prior}.  Stored per run:
                    the NumPy seed and each segment's skip draw, the eps stream of the whole chain, the executed-step count,
                    per segment the zero-frame pattern and digests of every frame; the last frame of every segment in full
                    for the first run of each image case, every pose in full.  Frames are redrawn from their stored seed.

The file name matches neither gen_*.pt nor step_*.pt: tests glob those names for dcgan generation and training fixtures.

    python tests/golden/make_golden_multi_cp.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import ROOT, import_reference, make_opt  # noqa: E402
from make_golden_extra import warm_bn  # noqa: E402

sys.path.insert(0, ROOT)
from oracle.p2p_oracle import tensor_digest  # noqa: E402

CASES = {
    "d64_np1": dict(net=64, width=64, channels=1, T_in=9, B=2, cp_ixs=[0, 3, 5, 8], len_outputs=[4, 5, 4], alt="posterior",
                    opt=dict(skip_prob=0.5)),
    "d64_np2_lfs": dict(net=64, width=64, channels=1, T_in=9, B=2, cp_ixs=[0, 2, 6, 8], len_outputs=None, alt="prior",
                        opt=dict(skip_prob=0.5, n_past=2, last_frame_skip=True)),
    "vgg64_rgb": dict(net="vgg", width=64, channels=3, T_in=6, B=1, cp_ixs=[0, 2, 5], len_outputs=None, alt="posterior",
                      opt=dict(skip_prob=0.5)),
    "h36m_np1": dict(net="mlp", T_in=8, B=2, cp_ixs=[0, 3, 5, 7], len_outputs=None, alt="prior", opt=dict(skip_prob=0.5)),
}
OPT_KEYS = ("beta", "weight_cpc", "weight_align", "skip_prob", "n_past", "last_frame_skip", "lr", "beta1", "batch_size")


def frames(spec):
    """The case's input clip, redrawn from the stored seed: frames in [0, 1), or poses 3 * randn (the loader's std)."""
    g = torch.Generator().manual_seed(spec["x_seed"])
    if spec["net"] == "mlp":
        return 3 * torch.randn(spec["T_in"], spec["B"], 17, 3, generator=g)
    return torch.rand(spec["T_in"], spec["B"], spec["channels"], spec["width"], spec["width"], generator=g)


def segments(spec):
    """(x slice start, slice length, len_output) per segment."""
    cps = spec["cp_ixs"]
    lens = spec["len_outputs"] or [b - a + 1 for a, b in zip(cps, cps[1:])]
    return [(a, b - a + 1, L) for a, b, L in zip(cps, cps[1:], lens)]


def run_case(name, spec, p2p_model, backbones):
    pose = spec["net"] == "mlp"
    torch.manual_seed(1)
    if pose:
        opt = make_opt(backbones["mlp"], dataset="h36m", batch_size=spec["B"], **spec["opt"])
        model = p2p_model.P2PModel(opt.batch_size, 1, 128, 10, 512, 1, 1, 2, opt=opt)
        model.eval()
        cfg = dict(g_dim=128, z_dim=10, rnn_size=512, backbone="mlp", predictor_rnn_layers=2, posterior_rnn_layers=1,
                   prior_rnn_layers=1)
        bn = {}
    else:
        opt = make_opt(backbones[spec["net"]], batch_size=spec["B"], **spec["opt"])
        model = p2p_model.P2PModel(opt.batch_size, spec["channels"], 128, 10, 256, 1, 1, 2, opt=opt)
        warm_bn(model, spec, torch.Generator().manual_seed(4321))
        cfg = dict(g_dim=128, z_dim=10, rnn_size=256, channels=spec["channels"], image_width=spec["width"],
                   predictor_rnn_layers=2, posterior_rnn_layers=1, prior_rnn_layers=1)
        if spec["net"] == "vgg":
            cfg.update(backbone="vgg", vgg_width=spec["width"])
        mods = dict(encoder=model.encoder, decoder=model.decoder)
        bn = {m: {k: v.detach().clone() for k, v in mods[m].state_dict().items() if "running_" in k or "num_batches" in k}
              for m in mods}
    spec = dict(spec, x_seed=1357 + len(name))
    x = frames(spec)
    segs = segments(spec)
    case = dict(case=name, backbone=spec["net"], init_seed=1, cfg=cfg, opt={k: getattr(opt, k) for k in OPT_KEYS},
                x_seed=spec["x_seed"], x_shape=tuple(x.shape), cp_ixs=spec["cp_ixs"], len_outputs=[L for (_, _, L) in segs],
                bn_buffers=bn, runs=[])
    n_calls = []
    hook = model.posterior.register_forward_hook(lambda *a: n_calls.append(1))
    for mode in ("full", spec["alt"]):
        for skip_frame in (False, True):
            seed = 700 + 10 * len(case["runs"]) + len(name)
            np.random.seed(seed)
            probs = [torch.from_numpy(np.random.uniform(0, 1, L - 1)) for (_, _, L) in segs]
            np.random.seed(seed)
            torch.manual_seed(seed)
            n_calls.clear()
            out = []
            with torch.no_grad():
                for k, (a, n, L) in enumerate(segs):
                    xk = (None, x[a:a + n], None) if pose else x[a:a + n]
                    out.append(model.p2p_generate(xk, L, L - 1, model_mode=mode, skip_frame=skip_frame, init_hidden=k == 0))
            n_exec = len(n_calls)
            torch.manual_seed(seed)
            eps = torch.empty(n_exec, 2, spec["B"], 10)
            for s in range(n_exec):
                eps[s, 0].normal_()
                eps[s, 1].normal_()
            rec = dict(model_mode=mode, skip_frame=skip_frame, np_seed=seed, probs=probs, eps=eps, n_exec=n_exec,
                       zero_frames=[[bool((f == 0).all()) for f in seq] for seq in out])
            if pose:
                rec.update(poses=[torch.stack([f.detach().clone() for f in seq]) for seq in out])
            else:
                rec.update(digests=[[tensor_digest(f) for f in seq] for seq in out])
                if not case["runs"]:
                    rec.update(last=[seq[-1].detach().clone() for seq in out])
            case["runs"].append(rec)
            print(f"[{name}] mode={mode} skip_frame={skip_frame}: executed {n_exec}, zero frames {rec['zero_frames']}")
    hook.remove()
    return case


def main():
    torch.set_num_threads(8)
    p2p_model, backbones = import_reference()
    fix = dict(cases=[run_case(name, spec, p2p_model, backbones) for name, spec in CASES.items()])
    path = os.path.join(HERE, "multi_cp_gen.pt")
    torch.save(fix, path)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
