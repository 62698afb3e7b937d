#!/usr/bin/env python
"""generate.py fixture from the UNMODIFIED reference script (build container only, the shims of make_golden.py plus):

  * a stub ``imageio`` whose ``get_reader`` yields seeded uint8 frames (tests/generate_ref.video_frames; [H, W, 1] frames
    give a 1-channel clip) and whose ``mimsave`` records the GIF frames;
  * a capturing ``torchvision.utils.save_image``;
  * stand-ins for the imports the script makes but does not use here (matplotlib, data.data_utils);
  * a checkpoint written by the reference's own ``P2PModel.save`` (dcgan_64);
  * ``P2PModel.p2p_generate`` replaced by a stub that makes the reference call's NumPy skip draw and returns seeded frames
    (tests/generate_ref.stub_frames), so that the tests can redraw every sample.

  generate_ref.pt   the script run through ``runpy`` (argv --ckpt, --video, --output_root OUT) with its lengths 10, 20, 30
                    and 5 samples, in two kinds of cases:
                    * "composition": ``p2p_generate`` stubbed as above, on clips of
                        t20_c3   20 RGB frames of 64 x 64 (lengths below, equal to and above the clip)
                        t12_c1   12 one-channel frames of 64 x 64
                      stored: the seeds, the displayed samples of every length (np.random.choice, in order), the saved
                      files in order with a sha256 of every saved tensor and of every GIF frame, and NumPy's state before
                      and after;
                    * "generation": the reference's real ``p2p_generate`` (eval mode, BatchNorm running statistics moved
                      off (0, 1) by make_golden_extra.warm_bn) on a 12-frame RGB clip of 64 x 64, for
                        d64_c3   dcgan_64, 3 channels
                        vgg64_c3 vgg_64, 3 channels
                      stored: the init seed, configuration and BatchNorm buffers of the model, per-module parameter sums,
                      every eps draw of the reparameterisations in order ([1, z] each: per length, per call, per step,
                      posterior then prior), the saved files in order with a digest of every saved tensor (512 sampled
                      values) and of every GIF's stacked frames (256 values), and NumPy's state before and after.

    python tests/golden/make_golden_generate.py
"""
import hashlib
import os
import runpy
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import REF, ROOT, import_reference, make_opt  # noqa: E402
from make_golden_extra import warm_bn  # noqa: E402

sys.path.insert(0, ROOT)
from oracle.p2p_oracle import tensor_digest  # noqa: E402
from tests.generate_ref import stub_frames, video_frames  # noqa: E402

CASES = [dict(name="t20_c3", T=20, C=3, H=64), dict(name="t12_c1", T=12, C=1, H=64)]
GEN_CASES = [dict(name="d64_c3", net=64, backbone="dcgan", T=12, C=3, H=64), dict(name="vgg64_c3", net="vgg", backbone="vgg", T=12,
                                                                                  C=3, H=64)]
OPT_KEYS = ("beta", "weight_cpc", "weight_align", "skip_prob", "n_past", "last_frame_skip", "lr", "beta1", "batch_size")
CFG = dict(g_dim=128, z_dim=10, rnn_size=256, prior_rnn_layers=1, posterior_rnn_layers=1, predictor_rnn_layers=2)
LENS, NSAMPLES = [10, 20, 30], 5


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def run_script(c, files, model, np_seed):
    """generate.py on the saved model, the stub reader yielding c's clip; returns NumPy's state before and after."""
    with tempfile.TemporaryDirectory() as d:
        ckpt = os.path.join(d, "model.pth")
        model.save(ckpt, 1)
        sys.argv = ["generate.py", "--ckpt", ckpt, "--video", "clip.mp4", "--output_root", "OUT"]
        np.random.seed(np_seed)
        before = np.random.get_state()
        cwd = os.getcwd()
        os.chdir(d)
        try:
            runpy.run_path(os.path.join(REF, "generate.py"), run_name="__main__")
        finally:
            os.chdir(cwd)
        return before, np.random.get_state()


def make_model(p2p_model, backbones, c, init_seed):
    torch.manual_seed(init_seed)
    opt = make_opt(backbones[c["net"]], batch_size=1, backbone=c["backbone"], image_width=c["H"], channels=c["C"], **CFG)
    return p2p_model.P2PModel(1, c["C"], 128, 10, 256, 1, 1, 2, opt=opt), opt


def generation_case(p2p_model, backbones, c, i):
    import torchvision.utils as vutils
    import models.lstm as ref_lstm
    c = dict(c, video_seed=800 + i, np_seed=41 + i, init_seed=1, lens=LENS, nsamples=NSAMPLES)
    model, opt = make_model(p2p_model, backbones, c, c["init_seed"])
    warm_bn(model, dict(channels=c["C"], width=c["H"]), torch.Generator().manual_seed(4321))
    mods = dict(encoder=model.encoder, decoder=model.decoder)
    bn = {m: {k: v.detach().clone() for k, v in mods[m].state_dict().items() if "running_" in k or "num_batches" in k}
          for m in mods}
    sums = {m: float(sum(p.detach().double().sum() for p in getattr(model, m).parameters()))
            for m in ("encoder", "decoder", "frame_predictor", "posterior", "prior")}
    files, eps, recording = [], [], [False]
    sys.modules["imageio"] = types.SimpleNamespace(
        get_reader=lambda name: iter(list(video_frames(c))),
        mimsave=lambda name, frames: files.append((name, tensor_digest(torch.from_numpy(np.stack(frames)), 256))))
    vutils.save_image = lambda t, name, **kw: files.append((name, tensor_digest(t, 512)))
    real_normal = torch.Tensor.normal_

    def normal_(t, *a, **k):
        out = real_normal(t, *a, **k)
        if recording[0]:
            eps.append(out.detach().clone())
        return out

    def recorded(f):
        def rep(self, mu, logvar):
            recording[0] = True
            try:
                return f(self, mu, logvar)
            finally:
                recording[0] = False
        return rep

    saved = ref_lstm.gaussian_lstm.reparameterize
    torch.Tensor.normal_ = normal_
    ref_lstm.gaussian_lstm.reparameterize = recorded(saved)
    try:
        with torch.no_grad():
            before, after = run_script(c, files, model, c["np_seed"])
    finally:
        torch.Tensor.normal_ = real_normal
        ref_lstm.gaussian_lstm.reparameterize = saved
    assert len(eps) == 2 * NSAMPLES * sum(L - 1 for L in LENS), len(eps)
    print(c["name"], len(files), "files", len(eps), "eps draws")
    return dict(c, cfg=dict(CFG, channels=c["C"], image_width=c["H"]), opt={k: getattr(opt, k) for k in OPT_KEYS}, bn_buffers=bn,
                param_sums=sums, eps=torch.stack(eps), files=files, np_before=before, np_after=after)


def main():
    p2p_model, backbones = import_reference()
    # the script's imports that it does not use here
    plt = types.SimpleNamespace(switch_backend=lambda *a: None)
    sys.modules.setdefault("matplotlib", types.SimpleNamespace(pyplot=plt))
    sys.modules.setdefault("matplotlib.pyplot", plt)
    import data  # the reference package (namespace)
    sys.modules["data.data_utils"] = data.data_utils = types.ModuleType("data.data_utils")
    import torchvision.utils as vutils
    torch.serialization.add_safe_globals([types.SimpleNamespace, torch.optim.Adam])   # the reference's torch.load(ckpt)
    out = []
    for i, c in enumerate(CASES):
        c = dict(c, video_seed=700 + i, sample_seed=9000 + 100 * i, np_seed=31 + i, lens=LENS, nsamples=NSAMPLES)
        files, calls = [], {}
        sys.modules["imageio"] = types.SimpleNamespace(
            get_reader=lambda name, c=c: iter(list(video_frames(c))),
            mimsave=lambda name, frames: files.append((name, [sha(f) for f in frames])))
        vutils.save_image = lambda t, name, **kw: files.append((name, sha(t.detach().cpu().numpy())))

        def stub(self, x, len_output, eval_cp_ix, c=c, **kw):
            np.random.uniform(0, 1, len_output - 1)
            s = calls[len_output] = calls.get(len_output, -1) + 1
            return list(stub_frames(c, len_output, s))

        real_generate = p2p_model.P2PModel.p2p_generate
        p2p_model.P2PModel.p2p_generate = stub
        model, _ = make_model(p2p_model, backbones, dict(c, net=64, backbone="dcgan"), 3)
        try:
            before, after = run_script(c, files, model, c["np_seed"])
        finally:
            p2p_model.P2PModel.p2p_generate = real_generate
        np.random.set_state(before)
        idxs = []
        for L in LENS:
            for _ in range(NSAMPLES):
                np.random.uniform(0, 1, L - 1)
            idxs.append(np.random.choice(NSAMPLES, NSAMPLES, replace=False))
        assert sha(np.random.get_state()[1]) == sha(after[1])
        out.append(dict(c, idxs=idxs, files=files, np_before=before, np_after=after))
        print(c["name"], len(files), "files")
    gen = [generation_case(p2p_model, backbones, c, i) for i, c in enumerate(GEN_CASES)]
    torch.save({"composition": out, "generation": gen}, os.path.join(HERE, "generate_ref.pt"))


if __name__ == "__main__":
    main()
