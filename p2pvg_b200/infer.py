"""Stand-alone (no-autograd) forward passes of the drop-in modules on the sm_90a kernels: what
``p2p_generate`` / ``generate.py`` / ``misc/visualize.py`` of the reference call (SURVEY.md §3.4).

Same call signatures and return values as the reference modules:
    encoder(x[B,C,H,W]) -> (h[B,g], [skip maps, NCHW])          models/dcgan_64.py:48-54
    decoder([vec[B,g], skips]) -> x_hat[B,C,H,W]                  models/dcgan_64.py:81-88
    lstm(inp) -> [B,out]; gaussian_lstm(inp) -> (z, mu, logvar)   models/lstm.py:37-44, 83-94
BatchNorm honours ``module.training`` (batch statistics + running-stat update, or running statistics).
The results are plain tensors without an autograd graph: training goes through P2PModel.forward.
"""
import numpy as np
import torch

from ._lib import ACT_LRELU, ACT_NONE, ACT_SIGMOID, ACT_TANH, CudaKernels
from .layouts import cast, nchw_to_nhwc, nhwc_to_nchw, pack_conv4, pack_convt4, tile_bias

_EXACT = {}


def kernels_for(device):
    """Exact-fp32-GEMM view of the device's one kernel backend (fp32 operands only occur in parity mode on the
    stand-alone module forwards: keep them exact)."""
    from ._lib import kernels_for as backend_for
    base = backend_for(device)
    if base.device.index not in _EXACT:
        _EXACT[base.device.index] = base.with_mode(False)
    return _EXACT[base.device.index]


_EPS_STREAM = None


class eps_stream:
    """Context manager: the reparameterisation noise of every gaussian_lstm call inside comes from `draws` (a list of
    [B, z] tensors, consumed in call order) instead of torch.randn -- the reference draws from a global generator whose
    stream cannot be reproduced across devices, so parity tests inject the reference's own draws."""

    def __init__(self, draws):
        self.draws = list(draws)

    def __enter__(self):
        global _EPS_STREAM
        self.prev, _EPS_STREAM = _EPS_STREAM, self.draws
        return self

    def __exit__(self, *exc):
        global _EPS_STREAM
        _EPS_STREAM = self.prev
        return False


def _act_dtype():
    import os
    return torch.float32 if os.environ.get("P2PVG_PRECISION", "bf16") == "fp32" else torch.bfloat16


def _bn(K, bn_mod, raw, y, G, R, C, act, dev):
    """BatchNorm + activation of one call (G=1 group)."""
    scale = torch.empty(C, device=dev)
    shift = torch.empty(C, device=dev)
    if bn_mod.training:
        mean, invstd, varu = (torch.empty(C, device=dev) for _ in range(3))
        K.bn_fwd_stats(raw, G, R, C, bn_mod.weight.data, bn_mod.bias.data, mean, invstd, varu, scale, shift)
        order = torch.zeros(1, dtype=torch.int32, device=dev)
        K.bn_ema(bn_mod.running_mean, bn_mod.running_var, mean, varu, order, 1, C, 0.1)
        bn_mod.num_batches_tracked += 1
    else:
        K.bn_eval_coeffs(bn_mod.weight.data, bn_mod.bias.data, bn_mod.running_mean, bn_mod.running_var, C, scale, shift)
    K.bn_act(raw, y, scale, shift, G, R, C, act)


def _stages(mod):
    from .models.backbone import STAGE_CHANNELS
    return STAGE_CHANNELS[mod.image_width]


@torch.no_grad()
def encoder_forward(mod, x):
    K = kernels_for(x.device)
    dev, adt = x.device, _act_dtype()
    chans = _stages(mod)
    n = len(chans)
    B, nc, H = int(x.shape[0]), int(x.shape[1]), int(x.shape[2])
    a = torch.empty(B * H * H * nc, device=dev, dtype=adt)
    nchw_to_nhwc(K, x.contiguous().float(), a, B, H * H, nc)
    skips = []
    cin = nc
    for l in range(n):
        blk = getattr(mod, f"c{l + 1}").main
        conv, bn = blk[0], blk[1]
        cout, Ho = chans[l], H // 2
        M = B * Ho * Ho
        wp = torch.empty(cout * 16 * cin, device=dev, dtype=adt)
        pack_conv4(K, conv.weight.data, wp)
        col = torch.empty(M * 16 * cin, device=dev, dtype=adt)
        raw = torch.empty(M * cout, device=dev, dtype=adt)
        y = torch.empty(M * cout, device=dev, dtype=adt)
        K.im2col(a, col, B, H, H, cin)
        K.gemm(col, wp, raw, M, cout, 16 * cin, bias=conv.bias.data)
        _bn(K, bn, raw, y, 1, B * Ho * Ho, cout, ACT_LRELU, dev)
        nchw = torch.empty(B, cout, Ho, Ho, device=dev)
        nhwc_to_nchw(K, y, nchw, B, Ho * Ho, cout)
        nchw._p2pvg_nhwc = y  # decoder_forward reuses the NHWC copy when it gets this very tensor back
        skips.append(nchw)
        a, H, cin = y, Ho, cout
    return _encode_top(K, getattr(mod, f"c{n + 1}"), a, B, mod.dim, adt), skips


def _encode_top(K, top, a, B, g, adt):
    """The encoder's top layer ``top`` = Conv2d(512, g, 4, 1, 0) + BatchNorm + Tanh on the 4x4x512 maps a [B, 4, 4, 512] (NHWC):
    h [B, g] fp32."""
    conv, bn = top[0], top[1]
    dev = a.device
    wp = torch.empty(g * 16 * 512, device=dev, dtype=adt)
    pack_conv4(K, conv.weight.data, wp)
    raw = torch.empty(B * g, device=dev, dtype=adt)
    y = torch.empty(B * g, device=dev, dtype=adt)
    K.gemm(a, wp, raw, B, g, 16 * 512, bias=conv.bias.data)
    _bn(K, bn, raw, y, 1, B, g, ACT_TANH, dev)
    h = torch.empty(B, g, device=dev)
    cast(K, y, h, B * g)
    return h


def _decode_head(K, upc1, vec, g, adt):
    """The decoder's head ``upc1`` = ConvTranspose2d(g, 512, 4, 1, 0) + BatchNorm + LeakyReLU on the latents vec (any shape
    with B * g elements): (d [B, 4, 4, 512] NHWC, B)."""
    dev = vec.device
    vec = vec.reshape(-1, g).float().contiguous()
    B = int(vec.shape[0])
    hp = torch.empty(B * g, device=dev, dtype=adt)
    cast(K, vec, hp, B * g)
    convt, bn = upc1[0], upc1[1]
    wp = torch.empty(g * 16 * 512, device=dev, dtype=adt)
    pack_convt4(K, convt.weight.data, wp)
    b16 = torch.empty(16 * 512, device=dev)
    tile_bias(K, convt.bias.data, b16, 16)
    raw = torch.empty(B * 16 * 512, device=dev, dtype=adt)
    d = torch.empty_like(raw)
    K.gemm(hp, wp, raw, B, 16 * 512, g, b_mn=True, bias=b16)
    _bn(K, bn, raw, d, 1, B * 16, 512, ACT_LRELU, dev)
    return d, B


def _frames_out(K, raw, B, W, nc):
    """Decoder output raw [B, W, W, nc] (NHWC, activation dtype) -> Sigmoid, as fp32 NCHW frames."""
    dev = raw.device
    out32 = torch.empty(B * W * W * nc, device=dev)
    cast(K, raw, out32, B * W * W * nc)
    K.act_fwd(out32, out32.numel(), ACT_SIGMOID)
    out = torch.empty(B, nc, W, W, device=dev)
    nhwc_to_nchw(K, out32, out, B, W * W, nc)
    return out


def _to_nhwc(K, t, adt):
    cached = getattr(t, "_p2pvg_nhwc", None)
    if cached is not None and cached.dtype == adt:
        return cached
    B, C, H, W = (int(v) for v in t.shape)
    out = torch.empty(B * H * W * C, device=t.device, dtype=adt)
    nchw_to_nhwc(K, t.contiguous().float(), out, B, H * W, C)
    return out


@torch.no_grad()
def decoder_forward(mod, vec, skip):
    K = kernels_for(vec.device)
    dev, adt = vec.device, _act_dtype()
    chans = _stages(mod)
    n = len(chans)
    d, B = _decode_head(K, mod.upc1, vec, mod.dim, adt)
    Hi = 4
    src = torch.zeros(1, dtype=torch.int32, device=dev)
    for k in range(n):
        cd = chans[n - 1 - k]
        last = (k == n - 1)
        cout = mod.nc if last else chans[n - 2 - k]
        blk = getattr(mod, f"upc{k + 2}")
        convt = blk[0] if last else blk.main[0]
        sk = _to_nhwc(K, skip[n - 1 - k], adt)
        wp = torch.empty(2 * cd * 16 * cout, device=dev, dtype=adt)
        pack_convt4(K, convt.weight.data, wp)
        Md = B * Hi * Hi
        colD = torch.empty(Md * 16 * cout, device=dev, dtype=adt)
        colS = torch.empty(Md * 16 * cout, device=dev, dtype=adt)
        K.gemm(d, wp[:cd * 16 * cout], colD, Md, 16 * cout, cd, b_mn=True)
        K.gemm(sk, wp[cd * 16 * cout:], colS, Md, 16 * cout, cd, b_mn=True)
        raw = torch.empty(B * 4 * Hi * Hi * cout, device=dev, dtype=adt)
        K.col2im(colD, raw, B, Hi, Hi, cout, bias=convt.bias.data, col2=colS, grp_src=src, imgs_per_group=B)
        if not last:
            dn = torch.empty_like(raw)
            _bn(K, blk.main[1], raw, dn, 1, B * 4 * Hi * Hi, cout, ACT_LRELU, dev)
            d = dn
        Hi *= 2
    return _frames_out(K, raw, B, Hi, mod.nc)


def _lstm_cells(K, mod, inp):
    dev = inp.device
    R = mod.hidden_size
    x = inp.reshape(-1, mod.input_size).float().contiguous()
    B = int(x.shape[0])
    h_in = torch.empty(B, R, device=dev)
    K.gemm(x, mod.embed.weight.data, h_in, B, R, mod.input_size, bias=mod.embed.bias.data)
    for l, cell in enumerate(mod.lstm):
        h_prev, c_prev = mod.hidden[l]
        pre = torch.empty(B, 4 * R, device=dev)
        gates = torch.empty(B, 4 * R, device=dev)
        K.gemm(h_in, cell.weight_ih.data, pre, B, 4 * R, R, bias=cell.bias_ih.data)
        K.gemm(h_prev.contiguous().float(), cell.weight_hh.data, gates, B, 4 * R, R, bias=cell.bias_hh.data, addend=pre)
        c, h = torch.empty(B, R, device=dev), torch.empty(B, R, device=dev)
        K.lstm_pointwise_fwd(gates, c_prev.contiguous().float(), c, h, B, R)
        mod.hidden[l] = (h, c)
        h_in = h
    return h_in, B


@torch.no_grad()
def lstm_forward(mod, inp):
    K = kernels_for(inp.device)
    h, B = _lstm_cells(K, mod, inp)
    lin = mod.output[0]
    out = torch.empty(B, mod.output_size, device=inp.device)
    K.gemm(h, lin.weight.data, out, B, mod.output_size, mod.hidden_size, bias=lin.bias.data)
    K.act_fwd(out, out.numel(), ACT_TANH)
    return out


@torch.no_grad()
def gaussian_lstm_forward(mod, inp):
    K = kernels_for(inp.device)
    dev = inp.device
    h, B = _lstm_cells(K, mod, inp)
    z_dim, R = mod.output_size, mod.hidden_size
    mu, lv = torch.empty(B, z_dim, device=dev), torch.empty(B, z_dim, device=dev)
    K.gemm(h, mod.mu_net.weight.data, mu, B, z_dim, R, bias=mod.mu_net.bias.data)
    K.gemm(h, mod.logvar_net.weight.data, lv, B, z_dim, R, bias=mod.logvar_net.bias.data)
    if _EPS_STREAM is not None:   # parity tests replay the reference's own N(0,1) draws (eps_stream below)
        eps = _EPS_STREAM.pop(0).to(device=dev, dtype=torch.float32).reshape(B, z_dim).contiguous()
    else:
        eps = torch.randn(B, z_dim, device=dev)  # the reference draws from the device's global generator (models/lstm.py:78)
    z, zz = torch.empty_like(mu), torch.empty_like(mu)
    kl = torch.zeros(4, device=dev)
    K.reparam_kl_fwd(mu, lv, mu, lv, eps, eps, z, zz, B * z_dim, kl)
    return z, mu, lv


@torch.no_grad()
def p2p_generate(model, x, len_output, eval_cp_ix, model_mode="full", skip_frame=False, init_hidden=True):
    """Autoregressive point-to-point generation (reference models/p2p_model.py:80-183): one sample per input
    sequence; skipped frames are emitted as zeros; posterior sees ground truth only while it exists."""
    opt = model.opt
    if isinstance(x, tuple):  # h36m
        x = x[1]
    batch_size = x[0].shape[0]
    gen_seq = [x[0]]
    x_in = x[0]
    if init_hidden:
        model.init_hidden(batch_size=batch_size)
    seq_len = len(x)
    x_cp, global_z = model.get_global_descriptor(x, cp_ix=seq_len - 1)
    prev_i, skip_count = 0, 0
    max_skip_count = seq_len * opt.skip_prob
    probs = np.random.uniform(0, 1, len_output - 1)
    skip = None
    for i in range(1, len_output):
        if (probs[i - 1] <= opt.skip_prob and i >= opt.n_past and skip_count < max_skip_count and i != 1
                and i != (len_output - 1) and skip_frame):
            skip_count += 1
            gen_seq.append(torch.zeros_like(x_in))
            continue
        tuc = torch.full((batch_size, 1), (eval_cp_ix - i + 1) / eval_cp_ix, device=x_cp.device, dtype=torch.float32)
        dt = torch.full((batch_size, 1), (i - prev_i) / eval_cp_ix, device=x_cp.device, dtype=torch.float32)
        prev_i = i
        h, sk = model.encoder(x_in)
        if opt.last_frame_skip or i == 1 or i < opt.n_past:
            skip = sk
        h_cpaw = torch.cat([h, global_z, tuc, dt], 1)
        if i < opt.n_past:
            h_target = model.encoder(x[i])[0]
            zt, _, _ = model.posterior(torch.cat([h_target, global_z, tuc, dt], 1))
            zt_p, _, _ = model.prior(h_cpaw)
            model.frame_predictor(torch.cat([h, zt if model_mode in ("posterior", "full") else zt_p, tuc, dt], 1))
            x_in = x[i]
            gen_seq.append(x_in)
        else:
            if i < len(x):
                h_target = model.encoder(x[i])[0]
                h_target_cpaw = torch.cat([h_target, global_z, tuc, dt], 1)
            else:
                h_target_cpaw = h_cpaw
            zt, _, _ = model.posterior(h_target_cpaw)
            zt_p, _, _ = model.prior(h_cpaw)
            z_use = zt if model_mode == "posterior" else zt_p
            h_pred = model.frame_predictor(torch.cat([h, z_use, tuc, dt], 1))
            x_in = model.decoder([h_pred, skip])
            gen_seq.append(x_in)
    return gen_seq


@torch.no_grad()
def p2p_generate_samples(model, x, nsample, len_output, eval_cp_ix, model_mode="full", skip_frame=False):
    """`nsample` independent samples for every input sequence in ONE autoregressive pass (SURVEY.md §8f rank 2): the batch is
    tiled nsample times, so every kernel of a step runs once on nsample*B rows instead of nsample times on B rows
    (misc/visualize.py:135-144 loops `nsample` = 20 calls of p2p_generate).  In eval mode (BatchNorm on running statistics)
    rows are independent, so sample s equals what a separate call with the same noise draws would return; the NumPy
    frame-skip pattern (skip_frame=True) is drawn once and shared by the samples of a call.
    Returns a list of nsample sequences (each a list of len_output frames [B, ...])."""
    if isinstance(x, tuple):
        x = x[1]
    B = int(x[0].shape[0])
    tiled = [f.repeat(nsample, *([1] * (f.dim() - 1))) for f in x]
    seq = p2p_generate(model, tiled, len_output, eval_cp_ix, model_mode=model_mode, skip_frame=skip_frame)
    return [[f[s * B:(s + 1) * B] for f in seq] for s in range(nsample)]


# ---- human3.6m pose backbone (reference models/h36m_mlp.py:45-46, 61-69, 85-95) -----------------------------------------
def _linear(K, lin, x, rows, act=None):
    out = torch.empty(rows, lin.out_features, device=x.device)
    K.gemm(x, lin.weight.data, out, rows, lin.out_features, lin.in_features, bias=lin.bias.data)
    if act is not None:
        K.act_fwd(out, out.numel(), act)
    return out


def _residual_linear(K, rl, x, rows):
    from ._lib import ACT_RELU
    sc = _linear(K, rl.shortcut[0], x, rows, ACT_RELU)
    h = x
    for i in (0, 2, 4):
        h = _linear(K, rl.long_path[i], h, rows, ACT_RELU)
    K.permute4(h, sc, (sc.numel(), 1, 1, 1), (1, 0, 0, 0), accumulate=True)
    n = rl.norm.normalized_shape[0]
    y = torch.empty_like(sc)
    mean, rstd = torch.empty(rows, device=x.device), torch.empty(rows, device=x.device)
    K.layernorm_fwd(sc, rl.norm.weight.data, rl.norm.bias.data, y, mean, rstd, rows, n)
    return y


@torch.no_grad()
def mlp_encoder_forward(mod, x):
    K = kernels_for(x.device)
    B = int(x.shape[0])
    xf = x.reshape(B, -1).float().contiguous()
    h1 = _residual_linear(K, mod.fc1, xf, B)
    h2 = _residual_linear(K, mod.fc2, h1, B)
    return _linear(K, mod.fc3, h2, B, ACT_TANH), [h1, h2]


@torch.no_grad()
def mlp_decoder_forward(mod, vec, skip):
    K = kernels_for(vec.device)
    vec = vec.float().contiguous()
    B = int(vec.shape[0])
    d1 = _residual_linear(K, mod.fc1, vec, B)
    d2 = _residual_linear(K, mod.fc2, torch.cat([d1, skip[1].float()], 1).contiguous(), B)
    out = _linear(K, mod.fc3, torch.cat([d2, skip[0].float()], 1).contiguous(), B)
    return out.view(B, 17, 3)
