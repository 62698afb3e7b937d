"""Stand-alone (no-autograd) forward passes of the vgg_64 drop-in modules on the sm_90a kernels
(reference models/vgg_64.py:50-56, 94-105): what ``p2p_generate`` calls outside the train step.  Same conventions as
p2pvg_b200/infer.py: NCHW fp32 in / out, BatchNorm honours ``module.training``."""
import torch

from ._lib import ACT_LRELU
from .infer import _act_dtype, _bn, _decode_head, _encode_top, _frames_out, _to_nhwc, kernels_for
from .layouts import implicit_shape, nchw_to_nhwc, nhwc_to_nchw, pack_conv3, up8


def _conv3(K, a, conv, c0, cin, out, N, H, adt, dev, bias=True, accumulate_from=None):
    """out[N,H,H,cout] = conv3x3 over input channels [c0, c0+cin) of ``conv`` applied to a[N,H,H,cin]."""
    w = conv.weight.data
    cout = int(w.shape[0])
    ld = up8(9 * cin)
    scratch = torch.zeros(cout * 9 * cin + 8, device=dev, dtype=adt)
    wp = torch.empty(cout * ld, device=dev, dtype=adt) if ld != 9 * cin else scratch
    pack_conv3(K, w, wp, c0, cin, scratch=scratch)
    b = conv.bias.data if bias else None
    if adt == torch.bfloat16 and implicit_shape(cin, cout):
        K.conv_gemm(3, a, wp, out, N, H, H, cin, cout, bias=b)
        return
    col = torch.empty(N * H * H * ld, device=dev, dtype=adt)
    K.im2col3(a, col, N, H, H, cin, ld, 1)
    K.gemm(col, wp, out, N * H * H, cout, ld, bias=b)


def _layer(K, blk, a, N, H, adt, dev, extra=None):
    """vgg_layer: conv3x3 + BatchNorm + LeakyReLU.  ``extra`` = second input (the skip half of a torch.cat)."""
    conv, bn = blk.main[0], blk.main[1]
    cout = int(conv.weight.shape[0])
    cin = int(conv.weight.shape[1]) if extra is None else int(conv.weight.shape[1]) // 2
    raw = torch.empty(N * H * H * cout, device=dev, dtype=adt)
    _conv3(K, a, conv, 0, cin, raw, N, H, adt, dev)
    if extra is not None:
        part = torch.empty(N * H * H * cout, device=dev, dtype=torch.float32)
        _conv3(K, extra, conv, cin, cin, part, N, H, adt, dev, bias=False)
        K.gather_add(raw, part, torch.zeros(1, dtype=torch.int32, device=dev), 1, N * H * H * cout)
    y = torch.empty_like(raw)
    _bn(K, bn, raw, y, 1, N * H * H, cout, ACT_LRELU, dev)
    return y, cout


@torch.no_grad()
def vgg_encoder_forward(mod, x):
    K = kernels_for(x.device)
    dev, adt = x.device, _act_dtype()
    B, nc, H = int(x.shape[0]), int(x.shape[1]), int(x.shape[2])
    if H != mod.image_width or int(x.shape[3]) != mod.image_width:
        raise ValueError(f"this vgg backbone expects {mod.image_width}x{mod.image_width} frames")
    nst = mod.nstage
    a = torch.empty(B * H * H * nc, device=dev, dtype=adt)
    nchw_to_nhwc(K, x.contiguous().float(), a, B, H * H, nc)
    skips, C = [], nc
    for i in range(1, nst + 1):
        if i > 1:
            p = torch.empty(B * (H // 2) * (H // 2) * C, device=dev, dtype=adt)
            K.maxpool2_fwd(a, p, B, H, H, C)
            a, H = p, H // 2
        for blk in getattr(mod, f"c{i}"):
            a, C = _layer(K, blk, a, B, H, adt, dev)
        nchw = torch.empty(B, C, H, H, device=dev)
        nhwc_to_nchw(K, a, nchw, B, H * H, C)
        nchw._p2pvg_nhwc = a
        skips.append(nchw)
    p = torch.empty(B * 16 * C, device=dev, dtype=adt)
    K.maxpool2_fwd(a, p, B, H, H, C)
    return _encode_top(K, getattr(mod, f"c{nst + 1}"), p, B, mod.dim, adt), skips


@torch.no_grad()
def vgg_decoder_forward(mod, vec, skip):
    K = kernels_for(vec.device)
    dev, adt = vec.device, _act_dtype()
    nc = mod.nc
    d, B = _decode_head(K, mod.upc1, vec, mod.dim, adt)
    H, C = 4, 512
    nst, W0 = mod.nstage, mod.image_width
    for k in range(nst):
        H *= 2
        u = torch.empty(B * H * H * C, device=dev, dtype=adt)
        K.upsample2_fwd(d, u, B, H // 2, H // 2, C)
        sk = _to_nhwc(K, skip[nst - 1 - k], adt)
        blocks = list(getattr(mod, f"upc{k + 2}"))
        layers = blocks if k < nst - 1 else blocks[:1]
        d, C = _layer(K, layers[0], u, B, H, adt, dev, extra=sk)
        for blk in layers[1:]:
            d, C = _layer(K, blk, d, B, H, adt, dev)
    convt = getattr(mod, f"upc{nst + 1}")[1]
    ldl = up8(9 * nc)
    wl = torch.empty(64 * ldl, device=dev, dtype=adt)
    pack_conv3(K, convt.weight.data, wl, scratch=torch.zeros(64 * 9 * nc + 8, device=dev, dtype=adt))
    M = B * W0 * W0
    colT = torch.empty(M * ldl, device=dev, dtype=adt)
    K.gemm(d, wl, colT, M, ldl, 64, b_mn=True)
    raw = torch.empty(M * nc, device=dev, dtype=adt)
    K.col2im3(colT, raw, B, W0, W0, nc, ldl, bias=convt.bias.data)
    return _frames_out(K, raw, B, W0, nc)
