"""Inputs of the composition cases of tests/golden/generate_ref.pt (make_golden_generate.py): the video the stub imageio
reader yields and the frames the stub p2p_generate returns, redrawn from the stored seeds."""
import numpy as np
import torch


def video_frames(c):
    """The stub reader's uint8 frames [T, H, W, C] (C = 1 frames are [H, W, 1] arrays)."""
    return np.random.RandomState(c["video_seed"]).randint(0, 256, size=(c["T"], c["H"], c["H"], c["C"])).astype(np.uint8)


def stub_frames(c, L, s):
    """What the stub p2p_generate returns for sample s (call s) of length L: L frames [1, C, H, H] in [0, 1)."""
    g = torch.Generator().manual_seed(c["sample_seed"] + 1000 * L + s)
    return torch.rand(L, 1, c["C"], c["H"], c["H"], generator=g)


def stub_samples(c):
    """(seq [T, 1, C, H, H] as generate.py's read_video makes it, {L: samples [nsamples, L, 1, C, H, H]})."""
    seq = torch.stack([torch.from_numpy((f / 255.).astype(np.float32)) for f in video_frames(c)]).permute(0, 3, 1, 2).unsqueeze(1)
    return seq, {L: torch.stack([stub_frames(c, L, s) for s in range(c["nsamples"])]) for L in c["lens"]}


def _border(f, color, pad=3):
    """f [.., 3, H, W] with a pad-wide border of color (misc/visualize.py add_gt_cp_border / add_samples_cp_border)."""
    out = torch.zeros_like(f)
    out[..., 0, :, :] = 1.
    if color == "orange":
        out[..., 1, :, :] = 165. / 255.
    W = f.shape[-1]
    out[..., pad:W - pad, pad:W - pad] = f[..., pad:W - pad, pad:W - pad]
    return out


def generate_ref(model, seq, output_root, save_image, mimsave, gen_lengths=(10, 20, 30), nsamples=5, ndisplays=5):
    """generate.py's loop (:108-163), restated in torch from reading it: nsamples eager p2p_generate calls per length, the
    displayed samples from np.random.choice, the control-point borders, padding=0 grids, per-frame host copies for the GIFs."""
    import torchvision.utils as vutils
    seq_len = len(seq)
    for L in gen_lengths:
        samples = torch.stack([torch.stack(model.p2p_generate(seq, L, L - 1, model_mode='full')) for _ in range(nsamples)])
        s = samples[np.random.choice(len(samples), ndisplays, replace=False)]
        padded = seq.clone()
        if L > seq_len:
            padded = torch.cat([padded, seq[seq_len - 1].repeat(L - seq_len, 1, 1, 1, 1)], 0)
        if padded.shape[2] == 1:
            padded, s = padded.repeat(1, 1, 3, 1, 1), s.repeat(1, 1, 1, 3, 1, 1)
        end = _border(padded[seq_len - 1], "red")
        padded[0] = _border(padded[0], "orange")
        padded[seq_len - 1] = end
        for i in range(seq_len, L):
            padded[i] = end
        s[:, 0], s[:, L - 1] = _border(s[:, 0], "orange"), _border(s[:, L - 1], "red")
        save_image(vutils.make_grid(padded[:, 0], nrow=len(padded), padding=0), '%s/len_%d-gt.png' % (output_root, L))
        block = []
        for ix, r in enumerate(s):
            row = vutils.make_grid(r[:, 0], nrow=len(r), padding=0)
            save_image(row, '%s/len_%d-gen_%03d.png' % (output_root, L, ix))
            block.append(row)
        save_image(torch.cat(block, 1), '%s/len_%d-gen_full.png' % (output_root, L))
        for ix, r in enumerate(s):
            mimsave('%s/len_%d-gen_%03d.gif' % (output_root, L, ix),
                    [(r[t, 0].permute(1, 2, 0).cpu().numpy() * 255).astype(np.uint8) for t in range(len(r))])
        gifs = [(vutils.make_grid(s[:, t, 0], nrow=ndisplays, padding=0).permute(1, 2, 0).cpu().numpy() * 255).astype(np.uint8)
                for t in range(L)]
        mimsave('%s/len_%d-gen_full.gif' % (output_root, L), gifs)


def fixture_model(c):
    """A generation case's model as a p2pvg_b200 P2PModel on the GPU in eval mode: the reference's weights (same init seed,
    checked against the stored per-module sums) and the case's BatchNorm buffers."""
    import types

    from p2pvg_b200.models import dcgan_64, vgg_64
    from p2pvg_b200.models.p2p_model import P2PModel
    o, cfg = c["opt"], c["cfg"]
    opt = types.SimpleNamespace(dataset="mnist", backbone_net=dcgan_64 if c["backbone"] == "dcgan" else vgg_64, **o)
    torch.manual_seed(c["init_seed"])
    model = P2PModel(o["batch_size"], cfg["channels"], cfg["g_dim"], cfg["z_dim"], cfg["rnn_size"], cfg["prior_rnn_layers"],
                     cfg["posterior_rnn_layers"], cfg["predictor_rnn_layers"], opt=opt)
    for m, want in c["param_sums"].items():
        got = float(sum(p.detach().double().sum() for p in getattr(model, m).parameters()))
        assert abs(got - want) <= 1e-9 * max(1.0, abs(want)), f"{m}: {got} != {want}"
    for m, bufs in c["bn_buffers"].items():
        mod = getattr(model, m)
        for k, v in bufs.items():
            owner, _, leaf = k.rpartition(".")
            getattr(mod.get_submodule(owner), leaf).copy_(v)
    return model.cuda().eval()
