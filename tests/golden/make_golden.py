#!/usr/bin/env python
"""Generate the golden fixtures in this directory by running the UNMODIFIED reference.

Runs only in the build container (needs /root/reference; read-only, nothing is copied from it).
The reference is imported as-is under the shims SURVEY.md §8(c) describes:

  1. ``misc.utils`` cannot be imported (matplotlib/skimage/imageio missing) -> a stub module is
     registered that exposes the reference's *real* ``init_weights`` (the function's source lines are
     exec'd from the reference file at run time).
  2. hard-coded ``.cuda()`` (models/lstm.py:24-25,58,63-64) -> identity on this CPU-only box.
  3. "Mode A": the two-phase update of models/p2p_model.py:261-269 is illegal on torch>=1.5; the
     reference's own hook ``opt.optimizer`` + ``init_optimizer()`` installs an Adam that applies the
     torch-1.0 update formula through ``p.data`` (no autograd version bump), after which the
     unmodified ``P2PModel.forward`` runs.

Outputs (committed): tests/golden/step_<case>.pt — inputs (x, eps, probs, seeds), the four losses,
per-call intermediate tensors captured with forward hooks, BN buffers, and compact digests
(oracle.p2p_oracle.tensor_digest) of every initial weight, gradient and post-step weight.

    python tests/golden/make_golden.py          # rewrites all fixtures
"""
import argparse
import math
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("P2PVG_REF", "/root/reference")
sys.path.insert(0, ROOT)
from oracle.p2p_oracle import tensor_digest  # noqa: E402  (digest format shared with the tests)


class LegacyAdam(torch.optim.Optimizer):
    """torch-1.0 ``optim.Adam.step`` arithmetic, applied through ``p.data``."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps))

    def step(self):
        for group in self.param_groups:
            b1, b2 = group["betas"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                g = p.grad.data
                st = self.state[p]
                if len(st) == 0:
                    st["step"] = 0
                    st["exp_avg"] = torch.zeros_like(p.data)
                    st["exp_avg_sq"] = torch.zeros_like(p.data)
                st["step"] += 1
                st["exp_avg"].mul_(b1).add_(g, alpha=1 - b1)
                st["exp_avg_sq"].mul_(b2).addcmul_(g, g, value=1 - b2)
                denom = st["exp_avg_sq"].sqrt().add_(group["eps"])
                bc1 = 1 - b1 ** st["step"]
                bc2 = 1 - b2 ** st["step"]
                p.data.addcdiv_(st["exp_avg"], denom, value=-group["lr"] * math.sqrt(bc2) / bc1)


def import_reference():
    if not os.path.isdir(REF):
        raise SystemExit(f"reference checkout not found at {REF}")
    sys.path.insert(0, REF)
    # shim 1: stub misc.utils with the real init_weights
    src = open(os.path.join(REF, "misc", "utils.py")).read().split("\n")
    start = next(i for i, l in enumerate(src) if l.startswith("def init_weights"))
    end = next(i for i in range(start + 1, len(src)) if src[i] and not src[i].startswith((" ", "\t")))
    ns = {}
    exec("\n".join(src[start:end]), ns)
    import misc  # the reference package (namespace)
    stub = types.ModuleType("misc.utils")
    stub.init_weights = ns["init_weights"]
    sys.modules["misc.utils"] = stub
    misc.utils = stub
    # shim 2: .cuda() -> identity
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.nn.Module.cuda = lambda self, *a, **k: self
    import models.p2p_model as p2p_model
    backbones = {}
    import models.dcgan_64 as d64
    import models.dcgan_128 as d128
    import models.h36m_mlp as mlp
    import models.vgg_64 as vgg64
    import models.vgg_128 as vgg128
    backbones[64] = d64
    backbones[128] = d128
    backbones["mlp"] = mlp
    backbones["vgg"] = vgg64
    backbones["vgg128"] = vgg128
    return p2p_model, backbones


def make_opt(backbone_net, **kw):
    o = types.SimpleNamespace(dataset="mnist", backbone_net=backbone_net, lr=1e-3, beta1=0.9, beta=1e-4,
                              weight_cpc=100.0, weight_align=0.5, skip_prob=0.0, n_past=1, last_frame_skip=False,
                              batch_size=None)
    for k, v in kw.items():
        setattr(o, k, v)
    return o


CASES = {
    # name: dict(width, channels, T, B, steps, opt overrides, np seed)
    "d64_plain": dict(width=64, channels=1, T=5, B=3, steps=2, opt={}, np_seed=3),
    "d64_skip": dict(width=64, channels=1, T=8, B=2, steps=1, opt=dict(skip_prob=0.5), np_seed=0),
    "d64_lfs": dict(width=64, channels=1, T=7, B=2, steps=1, opt=dict(skip_prob=0.5, n_past=2, last_frame_skip=True), np_seed=5),
    "d128_plain": dict(width=128, channels=3, T=4, B=2, steps=1, opt={}, np_seed=1),
    # configured batch_size != runtime batch: KL divides by the configured one (misc/criterion.py:15)
    "d64_cfgbatch": dict(width=64, channels=1, T=4, B=2, steps=1, opt=dict(batch_size=5), np_seed=2),
    # vgg_64 backbone (models/vgg_64.py), 3-channel frames (weizmann shape)
    "vgg64_rgb": dict(width="vgg", channels=3, T=4, B=2, steps=1, opt={}, np_seed=6),
    # vgg_128 backbone (models/vgg_128.py), 1-channel 128x128 frames
    "vgg128_gray": dict(width="vgg128", channels=1, T=3, B=2, steps=1, opt={}, np_seed=8),
    # human3.6m pose backbone (models/h36m_mlp.py): x is the tuple (pose_2d, pose_3d, camera_view), MSE on [B,17,3]
    "h36m_mlp": dict(width="mlp", channels=1, T=7, B=4, steps=1, opt=dict(dataset="h36m", skip_prob=0.3), np_seed=4),
}


def run_case(name, spec, p2p_model, backbones):
    torch.manual_seed(1)
    g_dim, z_dim, rnn = 128, 10, 256
    opt = make_opt(backbones[spec["width"]], **spec["opt"])
    if opt.batch_size is None:
        opt.batch_size = spec["B"]
    model = p2p_model.P2PModel(opt.batch_size, spec["channels"], g_dim, z_dim, rnn, 1, 1, 2, opt=opt)
    model.opt.optimizer = LegacyAdam  # shim 3 (Mode A) through the reference's own hook
    model.init_optimizer()
    model.train()
    mods = dict(frame_predictor=model.frame_predictor, posterior=model.posterior, prior=model.prior,
                encoder=model.encoder, decoder=model.decoder)
    fix = dict(case=name, cfg=dict(g_dim=g_dim, z_dim=z_dim, rnn_size=rnn, channels=spec["channels"],
                                   image_width=("vgg" if spec["width"] == "vgg128" else spec["width"]), vgg_width=(128 if spec["width"] == "vgg128" else 64),
                                   predictor_rnn_layers=2, posterior_rnn_layers=1,
                                   prior_rnn_layers=1, backbone=({"mlp": "mlp", "vgg": "vgg", "vgg128": "vgg"}.get(spec["width"], "dcgan"))),
               opt={k: getattr(opt, k) for k in ("beta", "weight_cpc", "weight_align", "skip_prob", "n_past",
                                                 "last_frame_skip", "lr", "beta1", "batch_size")},
               init_seed=1, torch=torch.__version__)
    fix["init_digest"] = {m: {k: tensor_digest(v) for k, v in mod.state_dict().items() if v.is_floating_point()}
                          for m, mod in mods.items()}
    fix["steps"] = []

    # forward hooks: record every module call in order
    tape = []
    hooks = []
    for mname in ("encoder", "decoder", "posterior", "prior", "frame_predictor"):
        def hook(mod, inp, out, mname=mname):
            if mname == "encoder":
                rec = dict(m=mname, latent=out[0].detach().clone(), skip_digest=[tensor_digest(s) for s in out[1]])
            elif mname == "decoder":
                rec = dict(m=mname, out_digest=tensor_digest(out), vec=inp[0][0].detach().clone())
            elif mname == "frame_predictor":
                rec = dict(m=mname, inp=inp[0].detach().clone(), out=out.detach().clone())
            else:
                rec = dict(m=mname, inp=inp[0].detach().clone(), z=out[0].detach().clone(),
                           mu=out[1].detach().clone(), logvar=out[2].detach().clone())
            tape.append(rec)
        hooks.append(mods[mname].register_forward_hook(hook))

    # image inputs are not stored (files would exceed 1 MB): the fixture keeps the seed and the shapes, and
    # tests/test_oracle_golden.py:load_fixture draws them again, one torch.rand per step
    x_seed = 1234 + len(name)
    gen = torch.Generator().manual_seed(x_seed)
    if spec["width"] != "mlp":
        fix["x_seed"] = x_seed
    for step in range(spec["steps"]):
        T, B, C, W = spec["T"], spec["B"], spec["channels"], spec["width"]
        if W == "mlp":
            x = torch.randn(T, B, 17, 3, generator=gen)
        else:
            side = {"vgg": 64, "vgg128": 128}.get(W, W)
            x = torch.rand(T, B, C, side, side, generator=gen)
        np.random.seed(spec["np_seed"] + step)
        probs = np.random.uniform(0, 1, T - 1)
        np.random.seed(spec["np_seed"] + step)  # forward() redraws the same vector
        eps_seed = 77 + step
        # how many executed steps -> replay the eps stream afterwards
        torch.manual_seed(eps_seed)
        tape.clear()
        grads1 = {}
        orig_update = model.update_model_without_prior

        def snap_then_update():
            for m in ("frame_predictor", "posterior", "encoder", "decoder"):
                grads1[m] = {k: p.grad.detach().clone() for k, p in mods[m].named_parameters() if p.grad is not None}
            orig_update()

        model.update_model_without_prior = snap_then_update
        model.zero_grad()
        losses = model((None, x, None) if W == "mlp" else x, 0, T - 1)
        model.update_model_without_prior = orig_update
        n_exec = sum(1 for r in tape if r["m"] == "posterior")
        torch.manual_seed(eps_seed)
        eps = torch.empty(n_exec, 2, B, z_dim)
        for s in range(n_exec):
            eps[s, 0].normal_()
            eps[s, 1].normal_()
        # sanity: z = eps*exp(.5 logvar)+mu reproduces the recorded z
        posts = [r for r in tape if r["m"] == "posterior"]
        priors = [r for r in tape if r["m"] == "prior"]
        for s in range(n_exec):
            for r, e in ((posts[s], eps[s, 0]), (priors[s], eps[s, 1])):
                z = e * (r["logvar"] * 0.5).exp() + r["mu"]
                assert torch.allclose(z, r["z"], atol=1e-6), "eps replay failed"
        gprior = {k: p.grad.detach().clone() for k, p in model.prior.named_parameters()}
        rec = dict(probs=torch.from_numpy(probs), np_seed=spec["np_seed"] + step, eps=eps,
                   losses=[float(l) for l in losses], n_exec=n_exec,
                   tape=[dict(r) for r in tape],
                   grad_digest={m: {k: tensor_digest(v) for k, v in g.items()} for m, g in {**grads1, "prior": gprior}.items()},
                   post_digest={m: {k: tensor_digest(v) for k, v in mod.state_dict().items() if v.is_floating_point()}
                                for m, mod in mods.items()},
                   bn_buffers={m: {k: v.detach().clone() for k, v in mods[m].state_dict().items()
                                   if "running_" in k or "num_batches" in k} for m in ("encoder", "decoder")})
        if spec["width"] == "mlp":
            rec["x"] = x
        else:
            rec["x_shape"] = tuple(x.shape)
        fix["steps"].append(rec)
        print(f"[{name}] step {step}: exec={n_exec} losses={rec['losses']}")
    for h in hooks:
        h.remove()
    path = os.path.join(HERE, f"step_{name}.pt")
    torch.save(fix, path)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("cases", nargs="*", default=list(CASES))
    args = ap.parse_args()
    torch.set_num_threads(8)
    p2p_model, backbones = import_reference()
    for name in args.cases:
        run_case(name, CASES[name], p2p_model, backbones)


if __name__ == "__main__":
    main()
