#!/usr/bin/env python
"""vgg generation fixture from the UNMODIFIED reference (build container only, same shims as make_golden.py):

  vgg_gen.pt   the reference's own ``P2PModel.p2p_generate`` (models/p2p_model.py:80-183) with the vgg_64 / vgg_128
               backbones (models/vgg_64.py, models/vgg_128.py) in eval mode, BatchNorm on running statistics moved off
               (0, 1) by make_golden_extra.warm_bn, for model_mode in {full, posterior, prior} x skip_frame in {False, True}:
                 vgg64_rgb      3 channels, B = 1, n_past 1, len_output past len(x) (the posterior falls back to h_cpaw)
                 vgg64_np2_lfs  1 channel, B = 2, n_past 2 + last_frame_skip
                 vgg128_gray    vgg_128, 1 channel, B = 1
               Stored: the frames' seed (they are redrawn with torch.rand, as make_golden.py does), NumPy seeds and skip
               draws, the eps stream, the BatchNorm buffers and digests of every generated frame of every run; the middle
               and last frames in full for the model_mode="full", skip_frame=False run of each case only, which keeps the
               file small (a full frame of the 128-pixel case is 64 KB).  Weights are re-created from the init seed.

The file name matches neither gen_*.pt nor step_*.pt: tests glob those names for dcgan generation and training fixtures.

    python tests/golden/make_golden_vgg_gen.py
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
    "vgg64_rgb": dict(net="vgg", width=64, channels=3, T_in=5, len_output=7, B=1, opt=dict(skip_prob=0.5)),
    "vgg64_np2_lfs": dict(net="vgg", width=64, channels=1, T_in=4, len_output=6, B=2,
                          opt=dict(skip_prob=0.5, n_past=2, last_frame_skip=True)),
    "vgg128_gray": dict(net="vgg128", width=128, channels=1, T_in=3, len_output=5, B=1, opt=dict(skip_prob=0.5)),
}


def frames(name, spec):
    """The case's input frames, redrawn from the stored seed."""
    g = torch.Generator().manual_seed(spec["x_seed"])
    return torch.rand(spec["T_in"], spec["B"], spec["channels"], spec["width"], spec["width"], generator=g)


def run_case(name, spec, p2p_model, backbones):
    torch.manual_seed(1)
    opt = make_opt(backbones[spec["net"]], batch_size=spec["B"], **spec["opt"])
    model = p2p_model.P2PModel(opt.batch_size, spec["channels"], 128, 10, 256, 1, 1, 2, opt=opt)
    warm_bn(model, spec, torch.Generator().manual_seed(4321))
    spec = dict(spec, x_seed=2468 + len(name))
    x = frames(name, spec)
    L = spec["len_output"]
    mods = dict(encoder=model.encoder, decoder=model.decoder)
    case = dict(case=name, init_seed=1,
                cfg=dict(g_dim=128, z_dim=10, rnn_size=256, channels=spec["channels"], image_width=spec["width"], backbone="vgg",
                         vgg_width=spec["width"], predictor_rnn_layers=2, posterior_rnn_layers=1, prior_rnn_layers=1),
                opt={k: getattr(opt, k) for k in ("beta", "weight_cpc", "weight_align", "skip_prob", "n_past", "last_frame_skip", "lr",
                                                  "beta1", "batch_size")},
                x_seed=spec["x_seed"], x_shape=tuple(x.shape), len_output=L, eval_cp_ix=L - 1,
                bn_buffers={m: {k: v.detach().clone() for k, v in mods[m].state_dict().items() if "running_" in k or "num_batches" in k}
                            for m in mods},
                runs=[])
    n_calls = []
    hook = model.posterior.register_forward_hook(lambda *a: n_calls.append(1))
    for mode in ("full", "posterior", "prior"):
        for skip_frame in (False, True):
            seed = 500 + 10 * len(case["runs"]) + len(name)
            np.random.seed(seed)
            probs = np.random.uniform(0, 1, L - 1)
            np.random.seed(seed)
            torch.manual_seed(seed)
            n_calls.clear()
            with torch.no_grad():
                seq = model.p2p_generate(x, L, L - 1, model_mode=mode, skip_frame=skip_frame)
            n_exec = len(n_calls)
            torch.manual_seed(seed)
            eps = torch.empty(n_exec, 2, spec["B"], 10)
            for s in range(n_exec):
                eps[s, 0].normal_()
                eps[s, 1].normal_()
            zeros = [bool((f == 0).all()) for f in seq]
            rec = dict(model_mode=mode, skip_frame=skip_frame, np_seed=seed, probs=torch.from_numpy(probs), eps=eps, n_exec=n_exec,
                       zero_frames=zeros, digests=[tensor_digest(f) for f in seq])
            if mode == "full" and not skip_frame:
                rec.update(last=seq[-1].detach().clone(), mid=seq[len(seq) // 2].detach().clone())
            case["runs"].append(rec)
            print(f"[{name}] mode={mode} skip_frame={skip_frame}: executed {n_exec}, zero frames {zeros}")
    hook.remove()
    return case


def main():
    torch.set_num_threads(8)
    p2p_model, backbones = import_reference()
    fix = dict(cases=[run_case(name, spec, p2p_model, backbones) for name, spec in CASES.items()])
    path = os.path.join(HERE, "vgg_gen.pt")
    torch.save(fix, path)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
