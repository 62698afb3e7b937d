#!/usr/bin/env python
"""Generate tests/golden/losses_eval.pt: the unmodified reference's P2PModel.forward with every module in eval mode.

Runs only in the build container (needs the reference checkout), under the shims of make_golden.py.  For each case the
model is built from torch seed 1, its BatchNorm running statistics are moved off (0, 1) by a few train-mode encoder /
decoder calls without touching a weight (make_golden_extra.warm_bn), then model.eval() and one forward(x): its returned
losses are computed before its update, so they are the held-out losses P2PModel.p2p_losses returns for the same draws.
The fixture keeps the draws (x seed or poses, NumPy probs, eps), the executed steps with their time counters as the
reference's posterior received them, the BatchNorm buffers and the four losses.

    python tests/golden/make_golden_losses.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import ROOT, LegacyAdam, import_reference, make_opt  # noqa: E402
from make_golden_extra import warm_bn  # noqa: E402

sys.path.insert(0, ROOT)

CASES = {
    "d64_skip": dict(net=64, width=64, channels=1, T=8, B=3, opt=dict(skip_prob=0.5), np_seed=0),
    "d64_np2_lfs": dict(net=64, width=64, channels=1, T=7, B=2, opt=dict(skip_prob=0.5, n_past=2, last_frame_skip=True), np_seed=5),
    "d128_rgb": dict(net=128, width=128, channels=3, T=4, B=2, opt={}, np_seed=1),
    "vgg64_rgb": dict(net="vgg", width=64, channels=3, T=4, B=2, opt={}, np_seed=6),
    "vgg128_gray": dict(net="vgg128", width=128, channels=1, T=3, B=2, opt=dict(skip_prob=0.5), np_seed=8),
    # the h36m test loader's B = 10 under a configured batch_size of 16: KL divides by the configured one
    "h36m_mlp": dict(net="mlp", width="mlp", channels=1, T=7, B=10, opt=dict(dataset="h36m", skip_prob=0.3, batch_size=16), np_seed=4),
}


def run_case(name, spec, p2p_model, backbones):
    torch.manual_seed(1)
    opt = make_opt(backbones[spec["net"]], **spec["opt"])
    if opt.batch_size is None:
        opt.batch_size = spec["B"]
    model = p2p_model.P2PModel(opt.batch_size, spec["channels"], 128, 10, 256, 1, 1, 2, opt=opt)
    model.opt.optimizer = LegacyAdam
    model.init_optimizer()
    mods = dict(encoder=model.encoder, decoder=model.decoder)
    if spec["net"] != "mlp":
        warm_bn(model, spec, torch.Generator().manual_seed(4321))
    model.eval()
    backbone = {"mlp": "mlp", "vgg": "vgg", "vgg128": "vgg"}.get(spec["net"], "dcgan")
    fix = dict(case=name, init_seed=1,
               cfg=dict(g_dim=128, z_dim=10, rnn_size=256, channels=spec["channels"], image_width=spec["width"], backbone=backbone,
                        vgg_width=spec["width"] if backbone == "vgg" else 64, predictor_rnn_layers=2, posterior_rnn_layers=1, prior_rnn_layers=1),
               opt={k: getattr(opt, k) for k in ("beta", "weight_cpc", "weight_align", "skip_prob", "n_past", "last_frame_skip", "lr",
                                                 "beta1", "batch_size")},
               bn_buffers={m: {k: v.detach().clone() for k, v in mods[m].state_dict().items() if "running_" in k or "num_batches" in k}
                           for m in mods})
    T, B = spec["T"], spec["B"]
    gen = torch.Generator().manual_seed(1357 + len(name))
    if spec["net"] == "mlp":
        x = torch.randn(T, B, 17, 3, generator=gen)
        fix["x"] = x
    else:
        fix["x_seed"] = 1357 + len(name)
        x = torch.rand(T, B, spec["channels"], spec["width"], spec["width"], generator=gen)
        fix["x_shape"] = tuple(x.shape)
    counters = []
    hook = model.posterior.register_forward_hook(lambda mod, inp, out: counters.append(inp[0][0, -2:].detach().clone()))
    np.random.seed(spec["np_seed"])
    probs = np.random.uniform(0, 1, T - 1)
    np.random.seed(spec["np_seed"])
    torch.manual_seed(99)
    losses = model((None, x, None) if spec["net"] == "mlp" else x, 0, T - 1)
    hook.remove()
    n_exec = len(counters)
    torch.manual_seed(99)
    eps = torch.empty(n_exec, 2, B, 10)
    for s in range(n_exec):
        eps[s, 0].normal_()
        eps[s, 1].normal_()
    fix.update(probs=torch.from_numpy(probs), eps=eps, losses=[float(v) for v in losses], counters=torch.stack(counters),
               torch=torch.__version__)
    print(f"[{name}] executed {n_exec}: losses {fix['losses']}")
    return fix


def main():
    torch.set_num_threads(8)
    p2p_model, backbones = import_reference()
    out = {name: run_case(name, spec, p2p_model, backbones) for name, spec in CASES.items()}
    path = os.path.join(HERE, "losses_eval.pt")
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
