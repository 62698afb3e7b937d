#!/usr/bin/env python
"""Pose generation fixture from the UNMODIFIED reference (build container only, same shims as make_golden.py):

  pose_gen_h36m.pt   the reference's own ``P2PModel.p2p_generate`` (models/p2p_model.py:80-183) with the h36m_mlp backbone
                     (models/h36m_mlp.py), g_dim 128, z_dim 10, rnn_size 512, for model_mode in {full, posterior, prior} x
                     skip_frame in {False, True}, in two cases: n_past 1, and n_past 2 with last_frame_skip.  len_output runs
                     past len(x), so the posterior falls back to h_cpaw.  Stored: inputs (3 * randn poses, the loader's std,
                     data/human3.6m.py), NumPy seeds and skip draws, the eps stream, the executed-step counts, digests of the
                     initial weights and every generated pose in full.

The file name matches neither gen_*.pt nor step_*.pt: tests glob those names for dcgan generation and training fixtures.

    python tests/golden/make_golden_pose_gen.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import ROOT, import_reference, make_opt  # noqa: E402

sys.path.insert(0, ROOT)
from oracle.p2p_oracle import tensor_digest  # noqa: E402

G_DIM, Z_DIM, RNN = 128, 10, 512
CASES = {
    # n_past = 1 (the training default): ground truth is only the first pose
    "np1": dict(T_in=6, len_output=9, B=3, opt=dict(skip_prob=0.5)),
    # n_past = 2 + last_frame_skip: the `i < n_past` branch and fresh skips every step
    "np2_lfs": dict(T_in=5, len_output=8, B=2, opt=dict(skip_prob=0.5, n_past=2, last_frame_skip=True)),
}


def run_case(name, spec, p2p_model, mlp):
    torch.manual_seed(1)
    opt = make_opt(mlp, dataset="h36m", batch_size=spec["B"], **spec["opt"])
    model = p2p_model.P2PModel(opt.batch_size, 1, G_DIM, Z_DIM, RNN, 1, 1, 2, opt=opt)
    model.eval()
    mods = ("frame_predictor", "posterior", "prior", "encoder", "decoder")
    init_digest = {m: {k: tensor_digest(v) for k, v in getattr(model, m).state_dict().items() if v.is_floating_point()} for m in mods}
    gen = torch.Generator().manual_seed(2468 + len(name))
    x = 3 * torch.randn(spec["T_in"], spec["B"], 17, 3, generator=gen)
    L = spec["len_output"]
    case = dict(case=name, x=x, len_output=L, eval_cp_ix=L - 1,
                opt={k: getattr(opt, k) for k in ("beta", "weight_cpc", "weight_align", "skip_prob", "n_past", "last_frame_skip",
                                                  "lr", "beta1", "batch_size")},
                init_digest=init_digest, runs=[])
    n_calls = []
    hook = model.posterior.register_forward_hook(lambda *a: n_calls.append(1))
    for mode in ("full", "posterior", "prior"):
        for skip_frame in (False, True):
            seed = 300 + 10 * len(case["runs"]) + len(name)
            np.random.seed(seed)
            probs = np.random.uniform(0, 1, L - 1)
            np.random.seed(seed)
            torch.manual_seed(seed)
            n_calls.clear()
            with torch.no_grad():
                seq = model.p2p_generate((None, x, None), L, L - 1, model_mode=mode, skip_frame=skip_frame)
            n_exec = len(n_calls)
            torch.manual_seed(seed)
            eps = torch.empty(n_exec, 2, spec["B"], Z_DIM)
            for s in range(n_exec):
                eps[s, 0].normal_()
                eps[s, 1].normal_()
            zeros = [bool((f == 0).all()) for f in seq]
            case["runs"].append(dict(model_mode=mode, skip_frame=skip_frame, np_seed=seed, probs=torch.from_numpy(probs), eps=eps,
                                     n_exec=n_exec, zero_frames=zeros, poses=torch.stack([f.detach().clone() for f in seq])))
            print(f"[{name}] mode={mode} skip_frame={skip_frame}: executed {n_exec}, zero frames {zeros}")
    hook.remove()
    return case


def main():
    torch.set_num_threads(8)
    p2p_model, backbones = import_reference()
    fix = dict(init_seed=1, cfg=dict(g_dim=G_DIM, z_dim=Z_DIM, rnn_size=RNN, backbone="mlp", predictor_rnn_layers=2,
                                     posterior_rnn_layers=1, prior_rnn_layers=1),
               cases=[run_case(name, spec, p2p_model, backbones["mlp"]) for name, spec in CASES.items()])
    path = os.path.join(HERE, "pose_gen_h36m.pt")
    torch.save(fix, path)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
