"""The vgg_64 and vgg_128 training steps' kernel launches, derived from the engine's layer tables, and the float64 statements
the launch tests check them against (tests/test_vgg_launches_gpu.py, tests/test_vgg128_launches_gpu.py), with the launch
checks and the audited step both files run.

`forward_launches` / `backward_launches` walk the backbone's layer tables (VGG_ENC / VGG_DEC for 64x64 frames, VGG_ENC_128 /
VGG_DEC_128 for 128x128) the way TrainEngineVGG.encode / decode / decoder_backward / encoder_backward do and ask the engine's
own rules (implicit_shape, TrainEngine.stat_buf with BN_FUSE_MIN) which launches take the implicit GEMM,
which get fused BatchNorm statistics and which carry the skip addend, so the list follows the engine when it changes.
precision "fp32" derives every launch of the fp32 step's backbone methods that launch_audit.FP32_OPS names instead: im2col3
(both tap signs), the gemm_simt GEMMs with their pitches, gather_add of the fp32 skip half, col2im3, group_sum, add_indexed,
the unfused BatchNorm passes, colsum and sigmoid_mse (tests/test_vgg_fp32_launches_gpu.py, test_fp32_launch_lists_cpu.py).

The checkers work in image chunks so that float64 references of C3-sized tensors (up to 10^9 elements) stay a few GiB:
  * conv3_sums64: per-(image, channel) sums of a kind-3 / kind-5 output from per-tap window sums of the input, O(N H W Ck);
  * wgrad_ref64: the kind-4 weight gradient, accumulated over image chunks (9 float64 GEMMs per chunk);
  * stat rows / finalize: every fused statistics row against the float64 sums of the stored rows it covers, and the
    finalized BatchNorm statistics per group against float64 statistics of the stored output.
"""
import math
import types

import torch
import torch.nn.functional as F

from p2pvg_b200.engine import TrainEngine
from p2pvg_b200.engine_vgg import VGG_DEC, VGG_DEC_128, VGG_ENC, VGG_ENC_128, TrainEngineVGG
from p2pvg_b200.layouts import implicit_shape, up8
from tests.launch_audit import (BENCH_OPT, NAN, SKIP_OPT, AuditKernels, addend_index, audit_step, gemm32, op32, randn, release,
                                slices_with_boundary)
from tests.ref64 import (A_STAT, CHUNK, assert_exact, binary01, bound_check, check_finalize_vs_output, finalize_ref,
                         gemm_ref64)
from tests.tc_schedule import BETA, alpha_for, assert_within, cdiv, conv_tiles, gemm_tc_tiles, rows_by_tile, sm_count


# ------------------------------------------------------------------ the launch list

def _stat_rule(M, C, rows_per_group, kred):
    """TrainEngine.stat_buf's decision (None: statistics come from a separate pass) on a stand-in engine."""
    stub = types.SimpleNamespace(fuse_stats=True, fbuf=lambda tag, n: None)
    return TrainEngine.stat_buf(stub, "", M, 1, C, rows_per_group, kred=kred)


def vgg_tables(W0):
    """(encoder, decoder) layer tables of the vgg backbone for W0 x W0 frames, as TrainEngineVGG.__init__ picks them."""
    if W0 not in (64, 128):
        raise ValueError(f"no vgg backbone for {W0}x{W0} frames")
    return (VGG_ENC_128, VGG_DEC_128) if W0 == 128 else (VGG_ENC, VGG_DEC)


def forward_launches(T, B, S, nskip, W0=64, precision="bf16", nc=3):
    """Every implicit-GEMM forward convolution of one bf16 vgg step (encode, then decode), in engine order.  precision "fp32":
    every launch of the fp32 step's encode and decode that launch_audit.FP32_OPS names (_forward32), with op32 / gemm32 keys."""
    if precision == "fp32":
        return _forward32(T, B, S, nskip, W0, nc)
    ENC, DEC = vgg_tables(W0)
    out = []
    N, H, C = T * B, W0, None
    for i, stage in enumerate(ENC):
        for j, (cin, cout) in enumerate(stage):
            if j == 0 and i > 0:
                H //= 2
            if cin is not None and implicit_shape(cin, cout):
                st = _stat_rule(N * H * H, cout, B * H * H, 9 * cin)
                out.append(dict(name=f"enc{i}.{j}", kind=3, N=N, H=H, Ck=cin, Cn=cout, bias=True, addend=False, ipg=0, stat=st, B=B))
    N, H = (S + 1) * B, 4
    for k, stage in enumerate(DEC):
        for j, (cin, cout) in enumerate(stage):
            if j == 0:
                H *= 2
                C = cin // 2
                if implicit_shape(C, cout):
                    out.append(dict(name=f"dec{k}.0.S", kind=3, N=nskip * B, H=H, Ck=C, Cn=cout, bias=True, addend=False, ipg=0,
                                    stat=None, B=B))
                    st = _stat_rule(N * H * H, cout, B * H * H, 9 * C)
                    out.append(dict(name=f"dec{k}.0.D", kind=3, N=N, H=H, Ck=C, Cn=cout, bias=False, addend=True, ipg=B, stat=st,
                                    B=B, nsrc=nskip))
            elif implicit_shape(cin, cout):
                st = _stat_rule(N * H * H, cout, B * H * H, 9 * cin)
                out.append(dict(name=f"dec{k}.{j}", kind=3, N=N, H=H, Ck=cin, Cn=cout, bias=True, addend=False, ipg=0, stat=st, B=B))
    return out


def _dgrad(name, N, H, cout, cin, B):
    return dict(name=name + " dgrad", kind=5, N=N, H=H, Ck=cout, Cn=cin, bias=False, addend=False, ipg=0, stat=None, B=B)


def _wgrad(name, N, H, cout, cin):
    return dict(name=name + " wgrad", kind=4, N=N, H=H, Cm=cout, Cn=cin)


def _decoder_backward(out, DEC, N, B, nskip, want_wgrad, want_skip, tag):
    """TrainEngineVGG.decoder_backward over N = (g1 - g0) B images: stages last to first, layers in reverse; a stage entry's
    upsampled half at N, its skip half (want_skip) over the nskip B skip images the group_sum of its output gradient feeds."""
    for k in range(len(DEC) - 1, -1, -1):
        H = 8 << k
        for j in range(len(DEC[k]) - 1, -1, -1):
            cin, cout = DEC[k][j]
            if j == 0:
                C = cin // 2
                if implicit_shape(cout, C):
                    out.append(_dgrad(f"{tag}dec{k}.0.D", N, H, cout, C, B))
                if want_wgrad and implicit_shape(C, cout):
                    out.append(_wgrad(f"{tag}dec{k}.0.D", N, H, cout, C))
                if want_skip:
                    if implicit_shape(cout, C):
                        out.append(_dgrad(f"{tag}dec{k}.0.S", nskip * B, H, cout, C, B))
                    if want_wgrad and implicit_shape(C, cout):
                        out.append(_wgrad(f"{tag}dec{k}.0.S", nskip * B, H, cout, C))
            else:
                if implicit_shape(cout, cin):
                    out.append(_dgrad(f"{tag}dec{k}.{j}", N, H, cout, cin, B))
                if want_wgrad and implicit_shape(cin, cout):
                    out.append(_wgrad(f"{tag}dec{k}.{j}", N, H, cout, cin))


def backward_launches(T, B, S, nskip, W0=64, has_cpc=True, precision="bf16", nc=3):
    """The data-gradient (kind 5) and weight-gradient (kind 4) launches of one bf16 vgg step, in the order the step enqueues
    them (engine.py TrainEngine.phases, mode A): backward_decoder's decoder_backward(0, S) with weight and skip gradients over
    the S B reconstruction images (engine.py:1236), the CPC decode's decoder_backward(S, S + 1) with data gradients only over
    B images (backward_prior, :1355), then encoder_backward over all T B frames, where the first layer (3 input channels) has
    an explicit weight gradient and no data gradient.  precision "fp32": _backward32."""
    if precision == "fp32":
        return _backward32(T, B, S, nskip, W0, nc, has_cpc)
    ENC, DEC = vgg_tables(W0)
    out = []
    _decoder_backward(out, DEC, S * B, B, nskip, True, True, "")
    if has_cpc:
        _decoder_backward(out, DEC, B, B, nskip, False, False, "cpc ")
    N = T * B
    for i in range(len(ENC) - 1, -1, -1):
        H = W0 >> i
        for j in range(len(ENC[i]) - 1, -1, -1):
            cin, cout = ENC[i][j]
            if cin is None:
                continue
            if implicit_shape(cin, cout):
                out.append(_wgrad(f"enc{i}.{j}", N, H, cout, cin))
            if implicit_shape(cout, cin):
                out.append(_dgrad(f"enc{i}.{j}", N, H, cout, cin, B))
    return out


# ------------------------------------------------------------------ the fp32 step's launches

def _conv3_fwd32(out, name, N, H, cin, cout, bias=True, add_groups=0):
    """TrainEngineVGG.conv3_fwd on the explicit path (engine_vgg.py:104-109): im2col3 into rows of pitch up8(9 cin), gemm_simt,
    and the fp32 skip addend gathered into the output (add_groups groups of N / add_groups images)."""
    ld = up8(9 * cin)
    out.append(op32("im2col3", name, N, H, cin, ld, 1))
    out.append(gemm32(name, N * H * H, cout, ld, bias=bias))
    if add_groups:
        out.append(op32("gather_add", f"{name} skip addend", add_groups, N // add_groups * H * H * cout))


def _conv3_dgrad32(out, name, N, H, cout, cin):
    """conv3_dgrad (engine_vgg.py:116-118): im2col3 of dy with the taps mirrored (sgn -1), pitch 9 cout."""
    out.append(op32("im2col3", f"{name} dgrad", N, H, cout, 9 * cout, -1))
    out.append(gemm32(f"{name} dgrad", N * H * H, cin, 9 * cout))


def _conv3_wgrad32(out, name, N, H, cout, cin):
    """conv3_wgrad (engine_vgg.py:126-129): im2col3 of the layer input, dy^T col over every pixel."""
    ld = up8(9 * cin)
    out.append(op32("im2col3", f"{name} wgrad", N, H, cin, ld, 1))
    out.append(gemm32(f"{name} wgrad", cout, ld, N * H * H, a_mn=True, b_mn=True, lda=cout, ldb=ld))


def _forward32(T, B, S, nskip, W0, nc):
    """TrainEngineVGG.encode (engine_vgg.py:132-156) and decode (:159-204) with TrainEngine.implicit off (act_dtype fp32)."""
    ENC, DEC = vgg_tables(W0)
    out = []
    N, H = T * B, W0
    for i, stage in enumerate(ENC):
        for j, (cin, cout) in enumerate(stage):
            if j == 0 and i > 0:
                H //= 2
            _conv3_fwd32(out, f"enc{i}.{j}", N, H, nc if cin is None else cin, cout)                    # :148
            out += [op32("bn_fwd_stats", f"enc{i}.{j}", T, B * H * H, cout), op32("bn_act", f"enc{i}.{j}", T, B * H * H, cout, 1)]
    out.append(gemm32("enc_top", N, 128, 16 * 512, bias=True))                                        # encode_top (engine.py:793)
    out += [op32("bn_fwd_stats", "enc_top", T, B, 128), op32("bn_act", "enc_top", T, B, 128, 2)]
    G = S + 1
    N, H = G * B, 4
    out.append(gemm32("dec-1", N, 16 * 512, 128, b_mn=True, bias=True))                              # decode_head (engine.py:1008)
    out += [op32("bn_fwd_stats", "dec-1", G, B * 16, 512), op32("bn_act", "dec-1", G, B * 16, 512, 1)]
    for k, stage in enumerate(DEC):
        for j, (cin, cout) in enumerate(stage):
            if j == 0:
                H *= 2
                C = cin // 2
                _conv3_fwd32(out, f"dec{k}.0.S", nskip * B, H, C, cout)                                 # :183
                _conv3_fwd32(out, f"dec{k}.0.D", N, H, C, cout, bias=False, add_groups=G)             # :185
            else:
                _conv3_fwd32(out, f"dec{k}.{j}", N, H, cin, cout)                                       # :189
            out += [op32("bn_fwd_stats", f"dec{k}.{j}", G, B * H * H, cout), op32("bn_act", f"dec{k}.{j}", G, B * H * H, cout, 1)]
    ldl = up8(9 * nc)
    out.append(gemm32("dec_last", N * W0 * W0, ldl, 64, b_mn=True))                                    # :198
    out.append(op32("col2im3", "dec_last", N, W0, nc, ldl, True))                                      # :200
    out.append(op32("sigmoid_mse", "loss", G, B * nc * W0 * W0))                                       # losses_fwd (engine.py:1026)
    return out


def _decoder_backward32(out, DEC, Gn, B, nskip, W0, nc, want_wgrad, want_skip, tag):
    """TrainEngineVGG.decoder_backward (engine_vgg.py:207-272) on the explicit path, then decode_head_backward (engine.py:1130)."""
    N = Gn * B
    ldl = up8(9 * nc)
    M = N * W0 * W0
    out.append(op32("im2col3", f"{tag}dec_last dcol", N, W0, nc, ldl, 1))                              # :220
    out.append(gemm32(f"{tag}dec_last dgrad", M, 64, ldl))                                              # :223
    if want_wgrad:
        out.append(op32("colsum", f"{tag}dec_last bias grad", M, nc, nc))                              # :225
        out.append(gemm32(f"{tag}dec_last wgrad", 64, ldl, M, a_mn=True, b_mn=True, lda=64, ldb=ldl))  # :227
    for k in range(len(DEC) - 1, -1, -1):
        H = 8 << k
        for j in range(len(DEC[k]) - 1, -1, -1):
            cin, cout = DEC[k][j]
            nm = f"{tag}dec{k}.{j}"
            out.append(op32("bn_bwd", nm, Gn, B * H * H, cout, 1))                                     # :237
            if want_wgrad:
                out.append(op32("bn_param_grad", nm, Gn, cout))                                        # :239
            if j == 0:
                C = cin // 2
                _conv3_dgrad32(out, f"{nm}.D", N, H, cout, C)                                           # :245
                if want_wgrad:
                    _conv3_wgrad32(out, f"{nm}.D", N, H, cout, C)                                       # :248
                if want_skip:
                    out.append(op32("group_sum", f"{nm} skip sum", Gn, nskip, B * H * H * cout))       # :251
                    _conv3_dgrad32(out, f"{nm}.S", nskip * B, H, cout, C)                               # :253
                    if want_wgrad:
                        _conv3_wgrad32(out, f"{nm}.S", nskip * B, H, cout, C)                           # :256
            else:
                _conv3_dgrad32(out, nm, N, H, cout, cin)                                                # :266
                if want_wgrad:
                    _conv3_wgrad32(out, nm, N, H, cout, cin)                                            # :269
    out.append(op32("bn_bwd", f"{tag}dec-1", Gn, B * 16, 512, 1))                                      # engine.py:1140
    if want_wgrad:
        out.append(op32("bn_param_grad", f"{tag}dec-1", Gn, 512))
        out.append(gemm32(f"{tag}dec-1 wgrad", 128, 16 * 512, N, a_mn=True, b_mn=True))
    out.append(gemm32(f"{tag}dec-1 dgrad", N, 128, 16 * 512))


def _backward32(T, B, S, nskip, W0, nc, has_cpc):
    """decoder_backward(0, S), the CPC decoder_backward(S, S + 1) and encoder_backward (engine_vgg.py:274-305), in the order the
    serial fp32 step enqueues them (engine.py:684-688)."""
    ENC, DEC = vgg_tables(W0)
    out = []
    _decoder_backward32(out, DEC, S, B, nskip, W0, nc, True, True, "")
    if has_cpc:
        _decoder_backward32(out, DEC, 1, B, nskip, W0, nc, False, False, "cpc ")
    N = T * B
    out += [op32("bn_bwd", "enc_top", T, B, 128, 2), op32("bn_param_grad", "enc_top", T, 128),        # encode_top_backward
            gemm32("enc_top wgrad", 128, 16 * 512, N, a_mn=True, b_mn=True), gemm32("enc_top dgrad", N, 16 * 512, 128, b_mn=True)]
    for i in range(len(ENC) - 1, -1, -1):
        H = W0 >> i
        out.append(op32("add_indexed", f"enc{i} skip grad", nskip, B * H * H * ENC[i][-1][1]))          # :290
        for j in range(len(ENC[i]) - 1, -1, -1):
            cin, cout = ENC[i][j]
            cin = nc if cin is None else cin
            nm = f"enc{i}.{j}"
            out += [op32("bn_bwd", nm, T, B * H * H, cout, 1), op32("bn_param_grad", nm, T, cout)]   # :296-297
            _conv3_wgrad32(out, nm, N, H, cout, cin)                                                    # :300
            if i > 0 or j > 0:
                _conv3_dgrad32(out, nm, N, H, cout, cin)                                                # :304
    return out


def launch_key(L):
    """What a conv_gemm launch is, as the launch-list test compares it: kind, N, H, Ck, Cn, Cm, bias, addend dtype (the bf16
    skip half), images per group, fused statistics."""
    if L["kind"] == 4:
        return (4, L["N"], L["H"], 0, L["Cn"], L["Cm"], False, None, 0, False)
    return (L["kind"], L["N"], L["H"], L["Ck"], L["Cn"], 0, L["bias"], torch.bfloat16 if L["addend"] else None, L["ipg"],
            L["stat"] is not None)


def row_cooperative(c_dtype, stat, accumulate, addend_dtype):
    """The epilogue of kinds 0 / 3 / 5 stores whole bf16 rows cooperatively (conv_gemm.cu, `row_major_store`)."""
    return c_dtype == torch.bfloat16 and not stat and not accumulate and addend_dtype in (None, torch.bfloat16)


def variant(kind, Ck, Cn, stat, addend_dtype, c_dtype, accumulate=False, swap=False):
    """The code path a conv_gemm launch takes, as the coverage assertions name it."""
    if kind == 4:
        return ("k4", "swap" if swap else "noswap")
    return (f"k{kind}", "bres" if (Ck == 64 and Cn == 64) else "bn128" if Cn > 64 else "bn64", "stat" if stat else "-",
            {None: "-", torch.bfloat16: "add_bf16", torch.float32: "add_f32"}[addend_dtype],
            "rowcoop" if row_cooperative(c_dtype, stat, accumulate, addend_dtype) else "perrow")


# ------------------------------------------------------------------ kinds 3 / 5: per-(image, channel) sums

def _window_sums(x, sgn):
    """[n, 3, 3, C] float64: sum over the output pixels of x at the tap's offset sgn * (kh - 1, kw - 1), zero padding."""
    H, W = x.shape[1], x.shape[2]

    def rng(d, L):   # source rows r = p + d for output rows p in [0, L)
        return max(0, d), min(L, L + d)
    cols = torch.stack([x[:, :, slice(*rng(sgn * (kw - 1), W))].sum(2) for kw in range(3)], 2)       # [n, H, 3, C]
    return torch.stack([cols[:, slice(*rng(sgn * (kh - 1), H))].sum(1) for kh in range(3)], 1)       # [n, 3, 3, C]


def conv3_sums64(kind, a, b, N, H, Ck, Cn, bias=None, addend=None, add_idx=None):
    """(ref, absref) [N, Cn] float64: sum over pixels of the kind-3 (kind 5: mirrored taps) output
    sum_{tap,ck} w[c,tap,ck] * window_sum(x)[tap,ck] + HW bias[c] + sum_p addend[src(n), p, c], and the same over |.|."""
    sgn = -1 if kind == 5 else 1
    w = b.double().view(Cn, 3, 3, Ck)
    wa = w.abs()
    per = max(1, CHUNK // (H * H * Ck))
    ref = torch.empty(N, Cn, dtype=torch.float64, device=a.device)
    absref = torch.empty_like(ref)
    for n0 in range(0, N, per):
        x = a[n0:n0 + per].double()
        ref[n0:n0 + per] = torch.einsum("nabk,cabk->nc", _window_sums(x, sgn), w)
        absref[n0:n0 + per] = torch.einsum("nabk,cabk->nc", _window_sums(x.abs_(), sgn), wa)
        del x
    if bias is not None:
        ref += H * H * bias.double()
        absref += H * H * bias.double().abs()
    if addend is not None:
        s = addend.double().sum((1, 2)) if addend.numel() <= CHUNK else torch.cat(
            [addend[i:i + 64].double().sum((1, 2)) for i in range(0, addend.shape[0], 64)])
        sa = addend.double().abs().sum((1, 2)) if addend.numel() <= CHUNK else torch.cat(
            [addend[i:i + 64].double().abs().sum((1, 2)) for i in range(0, addend.shape[0], 64)])
        ref += s[add_idx]
        absref += sa[add_idx]
    return ref, absref


def out_sums(out, H):
    """(sum, sum of |.|) over the pixels of each image of an NHWC output, float64, in chunks."""
    N, Cn = out.shape[0], out.shape[-1]
    per = max(1, CHUNK // (H * H * Cn))
    s = torch.cat([out[i:i + per].double().sum((1, 2)) for i in range(0, N, per)])
    sa = torch.cat([out[i:i + per].double().abs().sum((1, 2)) for i in range(0, N, per)])
    return s, sa


def check_conv3_sums(out, kind, a, b, N, H, Ck, Cn, bias=None, addend=None, add_idx=None, name=""):
    """Every tile of the output contributes: per-(image, channel) sums within alpha * sum|terms| + beta * sum|out|.

    The output-rounding term beta * sum|out| grows with H W: at 64x64 with a bf16 output it is about 16 times one element's
    magnitude, the size of the error one wrong 128-row tile makes in an image's sum.  So this check reliably sees every
    tile of the smaller maps; at 64x64 it sees gross errors, and the element-wise slices carry the rest."""
    ref, absref = conv3_sums64(kind, a, b, N, H, Ck, Cn, bias, addend, add_idx)
    got, gabs = out_sums(out, H)
    diff = (got - ref).abs()
    bound = alpha_for(9 * Ck) * absref + BETA[out.dtype] * gabs
    ratio = torch.where(bound > 0, diff / bound.clamp_min(1e-300), torch.where(diff > 0, torch.inf, 0.0))
    worst = ratio.max().item()
    if not worst <= 1.0:
        n, c = (int(i) for i in torch.unravel_index(ratio.argmax(), ratio.shape))
        raise AssertionError(f"{name}: per-(image, channel) sums: {int((ratio > 1).sum())}/{ratio.numel()} out of bound, worst "
                             f"{worst:.3g} at image {n} channel {c} (got {got[n, c].item():.6g}, ref {ref[n, c].item():.6g})")
    print(f"[bound] {name} image/channel sums: worst error/bound {worst:.3g}")
    return worst


def conv3_ref64_elem(kind, a, b, H, Ck, Cn, bias=None, addend_rows=None):
    """Element-wise float64 reference (and magnitude) of kind 3 / 5 on the images of `a`; addend_rows: the addend images
    each image reads."""
    x = a.double().permute(0, 3, 1, 2)
    w = b.double().view(Cn, 3, 3, Ck)
    if kind == 3:
        run = lambda x_, w_: F.conv2d(x_, w_.permute(0, 3, 1, 2), padding=1)
    else:
        run = lambda x_, w_: F.conv_transpose2d(x_, w_.permute(3, 0, 1, 2), padding=1)
    ref = run(x, w).permute(0, 2, 3, 1)
    absref = run(x.abs(), w.abs()).permute(0, 2, 3, 1)
    if bias is not None:
        ref = ref + bias.double()
        absref = absref + bias.double().abs()
    if addend_rows is not None:
        ref = ref + addend_rows.double()
        absref = absref + addend_rows.double().abs()
    return ref, absref


# ------------------------------------------------------------------ fused statistics

def check_stat_rows(part, out, N, H, Cn, name=""):
    """Every partial row [tile, Cn, (sum, sum of squares)] against the float64 sums of the (up to 128) stored rows it covers,
    in tile-aligned image chunks (rows_by_tile pads the rows past the end with zeros)."""
    HW = H * H
    unit = max(1, 128 // HW)
    per = max(unit, CHUNK // (HW * Cn) // unit * unit)
    worst = 0.0
    for n0 in range(0, N, per):
        n = min(per, N - n0)
        rows = rows_by_tile(out[n0:n0 + n], 3, n, H, Cn, cdiv(n * HW, 128))
        t0 = n0 * HW // 128
        p = part[t0:t0 + rows.shape[0]]
        sq = rows * rows
        for j, (val, mag) in enumerate(((rows.sum(1), rows.abs().sum(1)), (sq.sum(1), sq.sum(1)))):
            worst = max(worst, assert_within(p[:, :, j], val, mag, 0, torch.float32, alpha=A_STAT, quiet=True,
                                             name=f"{name} stat rows from tile {t0} {'sum' if j == 0 else 'sumsq'}"))
        del rows, sq
    print(f"[bound] {name} statistics rows ({cdiv(N * HW, 128)} tiles): worst error/bound {worst:.3g}")
    return worst


# ------------------------------------------------------------------ kind 4

def wgrad_ref64(a, b, N, H, Cm, Cn):
    """g[Cm, (tap, Cn)] = sum_pix a[pix, Cm]^T b[pix + (kh-1, kw-1), Cn] in float64 (and over |.|), image chunk by chunk."""
    ref = torch.zeros(Cm, 9, Cn, dtype=torch.float64, device=a.device)
    absref = torch.zeros_like(ref)
    per = max(1, CHUNK // (H * H * max(Cm, Cn)))
    for n0 in range(0, N, per):
        x = a[n0:n0 + per].double().reshape(-1, Cm)
        bp = F.pad(b[n0:n0 + per].double(), (0, 0, 1, 1, 1, 1))
        for mag in (False, True):
            xa = x.abs() if mag else x
            bpa = bp.abs() if mag else bp
            dst = absref if mag else ref
            for tap in range(9):
                kh, kw = divmod(tap, 3)
                dst[:, tap] += xa.t() @ bpa[:, kh:kh + H, kw:kw + H].reshape(-1, Cn)
        del x, bp
    return ref.view(Cm, 9 * Cn), absref.view(Cm, 9 * Cn)


# ------------------------------------------------------------------ vgg.cu data movement (exact statements, in image chunks)

IMG_CHUNK = 256


def windows(x, N, H, W, C):
    """The four values of every 2x2 window in row-major order: [N, H/2, W/2, C] views."""
    v = x.reshape(N, H // 2, 2, W // 2, 2, C)
    return [v[:, :, 0, :, 0], v[:, :, 0, :, 1], v[:, :, 1, :, 0], v[:, :, 1, :, 1]]


def _first_max(wins):
    """Window maximum and the index of its first occurrence in row-major order (torch's max_pool2d tie rule: -0 == +0)."""
    best = torch.zeros(wins[0].shape, dtype=torch.int64, device=wins[0].device)
    bv = wins[0]
    for k in (1, 2, 3):
        upd = wins[k] > bv
        best = torch.where(upd, k, best)
        bv = torch.where(upd, wins[k], bv)
    return bv, best


def check_maxpool(x, y, dy, dx, N, H, W, C, name):
    """maxpool2_fwd output y (if given) equals the window maximum; maxpool2_bwd output dx (if given) holds dy at each
    window's first maximum and zeros elsewhere.  x, y, dy, dx: flat or shaped NHWC tensors."""
    x = x.reshape(-1)[:N * H * W * C].view(N, H, W, C)
    for n0 in range(0, N, IMG_CHUNK):
        n = min(IMG_CHUNK, N - n0)
        bv, best = _first_max(windows(x[n0:n0 + n], n, H, W, C))
        q = n0 * (H // 2) * (W // 2) * C
        if y is not None:
            assert torch.equal(y.reshape(-1)[q:q + bv.numel()].view_as(bv), bv), f"{name} maxpool2_fwd images [{n0}, ..)"
        if dx is not None:
            g = dy.reshape(-1)[q:q + bv.numel()].view_as(bv)
            got = windows(dx.reshape(-1)[n0 * H * W * C:(n0 + n) * H * W * C], n, H, W, C)
            for k in range(4):
                assert torch.equal(got[k], torch.where(best == k, g, torch.zeros_like(g))), \
                    f"{name} maxpool2_bwd images [{n0}, ..): not the first maximum's gradient"


def check_upsample_fwd(x, y, N, H, W, C, name):
    x = x.reshape(-1)[:N * H * W * C].view(N, H, W, C)
    for n0 in range(0, N, IMG_CHUNK):
        ref = x[n0:n0 + IMG_CHUNK].repeat_interleave(2, 1).repeat_interleave(2, 2)
        q = n0 * 4 * H * W * C
        assert torch.equal(y.reshape(-1)[q:q + ref.numel()].view_as(ref), ref), f"{name} upsample2_fwd images [{n0}, ..)"


def check_upsample_bwd(dy, dx, N, H, W, C, name):
    """dx (N x H x W) equals torch's fp32 (a + b) + (c + d) of each 2x2 window of dy, rounded once to dx's dtype, and lies
    within one rounding of the float64 sum.  Returns the worst error/bound ratio against float64."""
    worst = 0.0
    for n0 in range(0, N, IMG_CHUNK):
        n = min(IMG_CHUNK, N - n0)
        q = n0 * 4 * H * W * C
        a, b, c, d = (v.float() for v in windows(dy.reshape(-1)[q:q + n * 4 * H * W * C], n, 2 * H, 2 * W, C))
        got = dx.reshape(-1)[n0 * H * W * C:(n0 + n) * H * W * C].view(n, H, W, C)
        assert torch.equal(got, ((a + b) + (c + d)).to(dx.dtype)), f"{name} upsample2_bwd images [{n0}, ..): not (a+b)+(c+d)"
        ref = (a.double() + b.double()) + (c.double() + d.double())
        mag = a.double().abs() + b.double().abs() + c.double().abs() + d.double().abs()
        worst = max(worst, bound_check(got, ref, 2.0 ** -23 * mag + BETA[dx.dtype] * ref.abs(), f"{name} upsample2_bwd vs float64"))
    return worst


def im2col3_ref(x, N, H, W, C, sgn, ld):
    """col[(n,y,x), tap*C + c] = x[n, y + sgn*(kh-1), x + sgn*(kw-1), c] (zero outside the map); columns [9C, ld) zero."""
    xp = F.pad(x.reshape(N, H, W, C), (0, 0, 1, 1, 1, 1))
    cols = []
    for tap in range(9):
        kh, kw = divmod(tap, 3)
        dh, dw = sgn * (kh - 1), sgn * (kw - 1)
        cols.append(xp[:, 1 + dh:1 + dh + H, 1 + dw:1 + dw + W])
    return F.pad(torch.cat(cols, -1).reshape(N * H * W, 9 * C), (0, ld - 9 * C))


def check_im2col3(x, col, N, H, W, C, ld, sgn, name):
    x = x.reshape(-1)[:N * H * W * C].view(N, H, W, C)
    col = col.reshape(-1)[:N * H * W * ld].view(N * H * W, ld)
    for n0 in range(0, N, IMG_CHUNK):
        n = min(IMG_CHUNK, N - n0)
        assert torch.equal(col[n0 * H * W:(n0 + n) * H * W], im2col3_ref(x[n0:n0 + n], n, H, W, C, sgn, ld)), \
            f"{name} im2col3 sgn={sgn} ld={ld} images [{n0}, ..)"


def check_col2im3(col, y, N, H, W, C, ld, bias, name):
    """y[p] = bias + sum_tap col[p - (kh-1, kw-1), tap] within 9 fp32 adds and one output rounding; returns the worst ratio."""
    col = col.reshape(-1)[:N * H * W * ld].view(N, H, W, ld)
    y = y.reshape(-1)[:N * H * W * C].view(N, H, W, C)
    worst = 0.0
    for n0 in range(0, N, IMG_CHUNK):
        n = min(IMG_CHUNK, N - n0)
        cv = F.pad(col[n0:n0 + n].double()[..., :9 * C], (0, 0, 1, 1, 1, 1))
        ref = torch.zeros(n, H, W, C, dtype=torch.float64, device=col.device)
        mag = torch.zeros_like(ref)
        if bias is not None:
            ref += bias.double()
            mag += bias.double().abs()
        for tap in range(9):
            kh, kw = divmod(tap, 3)
            t = cv[:, 2 - kh:2 - kh + H, 2 - kw:2 - kw + W, tap * C:(tap + 1) * C]
            ref += t
            mag += t.abs()
        worst = max(worst, bound_check(y[n0:n0 + n], ref, 9 * 2.0 ** -24 * mag + BETA[y.dtype] * ref.abs(), f"{name} col2im3 images [{n0}, ..)"))
    return worst


def check_gather_add(dst, dst0, src, grp_src, G, n, name=""):
    """gather_add: dst[g] = dst0[g] + src[grp_src[g]] with one rounding to dst's dtype (a bf16 destination rounds twice: one
    bf16 ulp), group by group against float64.  Returns the worst ratio."""
    srcl = grp_src.tolist()[:G]
    rel = 2.0 ** -7 if dst.dtype == torch.bfloat16 else 2.0 ** -24
    dv, d0, sv = dst.reshape(-1)[:G * n].view(G, n), dst0.reshape(-1)[:G * n].view(G, n), src.reshape(-1)
    worst = 0.0
    for g in range(G):
        ref = d0[g].double() + sv[srcl[g] * n:(srcl[g] + 1) * n].double()
        worst = max(worst, bound_check(dv[g], ref, rel * ref.abs(), f"{name}: gather_add group {g}"))
    return worst


# ------------------------------------------------------------------ launch checks (vgg_64 and vgg_128 shapes)

def run_conv(K, sms, L, cdt, seed, label=""):
    """Launch kind 3 / 5 as L describes (forward_launches / backward_launches entry, or a part-B case) on seeded operands
    and run checks 1-4 of the launch list.  Returns the variant it exercised."""
    kind, N, H, Ck, Cn, B = L["kind"], L["N"], L["H"], L["Ck"], L["Cn"], L["B"]
    HW = H * H
    name = f"{label}{L['name']} kind {kind} N={N} {H}x{H} {Ck}->{Cn} out={str(cdt)[6:]}"
    torch.manual_seed(seed)
    a = randn(N, H, H, Ck, scale=0.5)
    b = randn(Cn, 9 * Ck, scale=1.0 / math.sqrt(9 * Ck))
    bias = randn(Cn, dtype=torch.float32) if L["bias"] else None
    add = src = idx = None
    ipg = L["ipg"]
    if L["addend"]:
        nsrc = L.get("nsrc", 1)
        G = cdiv(N, ipg)
        src = torch.tensor([(g + 1) % nsrc for g in range(G)], dtype=torch.int32, device="cuda")
        idx = addend_index(src.tolist(), ipg, N)
        add = randn(nsrc * ipg, H, H, Cn)
    st = L["stat"]
    s = conv_tiles(kind, N, H, H, Ck, Cn, 0, sms)
    part = torch.full((s.tiles_m, Cn, 2), NAN, device="cuda") if st is not None else None
    out = torch.full((N, H, H, Cn), NAN, device="cuda", dtype=cdt)
    K.conv_gemm(kind, a, b, out, N, H, H, Ck, Cn, bias=bias, addend=add, grp_src=src, imgs_per_group=ipg, stat_partial=part)
    torch.cuda.synchronize()
    assert not torch.isnan(out).any(), f"{name}: unwritten output elements"
    # 1 + 2: float64 and bit-identity on slices of the first, middle and last round
    worst = 0.0
    for i0, i1 in slices_with_boundary(N, HW, s, sms, max(1, ipg or B)):
        arows = add[idx[i0:i1]] if add is not None else None
        ref, absref = conv3_ref64_elem(kind, a[i0:i1], b, H, Ck, Cn, bias, arows)
        worst = max(worst, assert_within(out[i0:i1], ref, absref, 9 * Ck, cdt, quiet=True, name=f"{name} images [{i0}, {i1})",
                                         locate=lambda ix, i0=i0: s.where(0, ((i0 + ix[0]) * HW + ix[1] * H + ix[2]) // 128, ix[3] // s.BN)))
        del ref, absref
        sub = conv_tiles(kind, i1 - i0, H, H, Ck, Cn, 0, sms)
        assert sub.tiles <= sms
        o = torch.empty(i1 - i0, H, H, Cn, device="cuda", dtype=cdt)
        p = torch.full((sub.tiles_m, Cn, 2), NAN, device="cuda") if st is not None else None
        kw = {}
        if add is not None:   # the same addend rows, one group per image
            kw = dict(addend=arows.contiguous(), grp_src=torch.arange(i1 - i0, dtype=torch.int32, device="cuda"), imgs_per_group=1)
        K.conv_gemm(kind, a[i0:i1], b, o, i1 - i0, H, H, Ck, Cn, bias=bias, stat_partial=p, **kw)
        assert torch.equal(o, out[i0:i1]), f"{name}: images [{i0}, {i1}) differ from a launch of just those images"
        if p is not None:
            t0 = i0 * HW // 128
            assert torch.equal(p, part[t0:t0 + p.shape[0]]), f"{name}: statistics rows of images [{i0}, {i1}) differ"
        del o, p, arows
    print(f"[bound] {name} slices: worst error/bound {worst:.3g}")
    # 3: every tile, through the per-(image, channel) sums
    check_conv3_sums(out, kind, a, b, N, H, Ck, Cn, bias, add, idx, name=name)
    # 4: statistics rows and the finalize per BatchNorm group
    if st is not None:
        check_stat_rows(part, out, N, H, Cn, name=name)
        check_finalize_vs_output(K, part, st["parts_per_group"], out, N // B, B * HW, Cn, name=name)
    v = variant(kind, Ck, Cn, st is not None, add.dtype if add is not None else None, cdt)
    del a, b, out, part, add
    release()
    return v


def distinct_convs(launches):
    """The first launch of each distinct kind-3 / kind-5 shape of a list."""
    seen, out = set(), []
    for L in launches:
        if L["kind"] == 4:
            continue
        key = (L["kind"], L["N"], L["H"], L["Ck"], L["Cn"], L["bias"], L["addend"], L["stat"] is not None)
        if key not in seen:
            seen.add(key)
            out.append(L)
    return out


def encoder_first(backward):
    """A backward list with the encoder's launches first, in layer order (the engine runs them last, in reverse): each shape
    is then represented by its longest launch (all T B frames) under the encoder layer's name."""
    enc = [L for L in backward if L["name"].startswith("enc")]
    return enc[::-1] + [L for L in backward if not L["name"].startswith("enc")]


def wgrad_classes(launches):
    """The first kind-4 launch of each (map size, swapped roles) class of a backward list, encoder launches first."""
    sms_ = sm_count() if torch.cuda.is_available() else 132
    seen, out = set(), []
    for L in encoder_first(launches):
        if L["kind"] != 4:
            continue
        s = conv_tiles(4, L["N"], L["H"], L["H"], 0, L["Cn"], L["Cm"], sms_)
        if (L["H"], s.swap) not in seen:
            seen.add((L["H"], s.swap))
            out.append(L)
    return out


def run_wgrad(K, sms, L):
    """A kind-4 launch as L describes.  Zero-mean operands would cancel: over K = N H W the worst-case accumulation bound is
    larger than the result itself.  So (1) 0 / 1 operands, whose fp32 sums are exact integers: the result must equal float64
    bit for bit, and one lost 64-pixel block or split changes it; (2) real operands that do not cancel (one positive, one of
    mean 1/2), so that the bound is a small fraction of the value."""
    N, H, Cm, Cn = L["N"], L["H"], L["Cm"], L["Cn"]
    s = conv_tiles(4, N, H, H, 0, Cn, Cm, sms)
    name = f"wgrad {L['name']} {H}x{H} {Cm}x{Cn} swap={s.swap} splits={s.splits}"
    torch.manual_seed(22)
    a, b = binary01((N, H, H, Cm)), binary01((N, H, H, Cn))
    out = torch.full((Cm, 9 * Cn), NAN, device="cuda")
    K.conv_gemm(4, a, b, out, N, H, H, 0, Cn, Cm=Cm)
    assert_exact(out, wgrad_ref64(a, b, N, H, Cm, Cn)[0], N * H * H, name + " 0/1 operands")
    a = torch.rand(N, H, H, Cm, device="cuda").bfloat16()
    b = randn(N, H, H, Cn, scale=0.5) + 0.5
    K.conv_gemm(4, a, b, out, N, H, H, 0, Cn, Cm=Cm)
    ref, absref = wgrad_ref64(a, b, N, H, Cm, Cn)
    keff = s.kb_per_split * 64 + 16 * s.splits
    assert (ref.abs() >= 0.5 * absref).all()
    assert_within(out, ref, absref, keff, torch.float32, name=f"{name} K={N * H * H} non-cancelling operands")
    del a, b, out, ref, absref
    release()


def run_end_gemms(K, M):
    """The explicit GEMMs of the 3-channel ends over M pixels: the first encoder layer ([M, 32] x [64, 32] after im2col3) and
    the last decoder layer ([M, 64] x [64, 32], MN-major weight), and the [64, 32] weight gradient with K = M that both the
    first layer (dy^T col) and the last layer (x^T dcol, row pitch up8(27) = 32) launch."""
    torch.manual_seed(23)
    col = randn(M, 32)
    col[:, 27:] = 0
    w = randn(64, 32, scale=0.3)
    bias = randn(64, dtype=torch.float32)
    out = torch.full((M, 64), NAN, device="cuda", dtype=torch.bfloat16)
    K.gemm(col, w, out, M, 64, 32, bias=bias)
    for r0 in range(0, M, 1 << 21):
        r1 = min(M, r0 + (1 << 21))
        ref, absref = gemm_ref64(col[r0:r1], w, r1 - r0, 64, 32, False, False, 32, 32, bias=bias)
        assert_within(out[r0:r1], ref, absref, 32, torch.bfloat16, quiet=r0 > 0, name=f"enc first layer GEMM rows {r0}")
    a = randn(M, 64)
    wl = randn(64, 32, scale=0.2)
    colT = torch.full((M, 32), NAN, device="cuda", dtype=torch.bfloat16)
    K.gemm(a, wl, colT, M, 32, 64, b_mn=True)
    for r0 in range(0, M, 1 << 21):
        r1 = min(M, r0 + (1 << 21))
        ref, absref = gemm_ref64(a[r0:r1], wl, r1 - r0, 32, 64, False, True, 64, 32)
        assert_within(colT[r0:r1], ref, absref, 64, torch.bfloat16, quiet=r0 > 0, name=f"dec last layer GEMM rows {r0}")
    del col, out, a, colT
    # the first layer's weight gradient, K = M: exact on 0 / 1 operands, and within the bound on operands that do not cancel
    s = gemm_tc_tiles(64, 32, M, sm_count())
    name = f"enc first layer weight gradient K={M} splits={s.splits}"
    dy, col = binary01((M, 64)), binary01((M, 32))
    gw = torch.full((64, 32), NAN, device="cuda")
    K.set_gemm_impl("tc")
    try:
        K.gemm(dy, col, gw, 64, 32, M, a_mn=True, b_mn=True, lda=64, ldb=32)
        assert_exact(gw, gemm_ref64(dy, col, 64, 32, M, True, True, 64, 32)[0], M, name + " 0/1 operands")
        dy = torch.rand(M, 64, device="cuda").bfloat16()
        col = randn(M, 32, scale=0.5) + 0.5
        K.gemm(dy, col, gw, 64, 32, M, a_mn=True, b_mn=True, lda=64, ldb=32)
    finally:
        K.set_gemm_impl("auto")
    ref, absref = gemm_ref64(dy, col, 64, 32, M, True, True, 64, 32)
    assert (ref.abs() >= 0.5 * absref).all()
    assert_within(gw, ref, absref, s.kb_per_split * 64 + 16 * s.splits, torch.float32, name=name)
    del dy, col
    release()


def misaligned_like(n, dtype):
    """A flat tensor of n elements whose data pointer is not 16-byte aligned (forces the scalar kernels)."""
    return torch.empty(n + 1, device="cuda", dtype=dtype)[1:]


def run_maxpool(K, N, H, C, dtype, label):
    """maxpool2_fwd / maxpool2_bwd on an N x H x H x C map with planted ties: equal pairs, four equal values, and -0 / +0.
    The gradient goes to the first maximum in row-major order; the scalar paths equal the vector ones."""
    torch.manual_seed(26)
    x = randn(N, H, H, C, dtype=dtype)
    w = windows(x, N, H, H, C)
    # ties, on every 7th / 11th / 13th window channel
    w[1][..., 0::7].copy_(w[0][..., 0::7])                        # pair (0, 1)
    w[3][..., 3::11].copy_(w[2][..., 3::11])                      # pair (2, 3)
    for k in (1, 2, 3):
        w[k][:, ::5, :, 5::13].copy_(w[0][:, ::5, :, 5::13])      # four equal
    w[0][:, 1::5, :, 6::13] = -0.0                                 # -0 then +0, the others negative
    w[1][:, 1::5, :, 6::13] = 0.0
    w[2][:, 1::5, :, 6::13] = -1.0
    w[3][:, 1::5, :, 6::13] = -2.0
    del w
    y = torch.empty(N, H // 2, H // 2, C, device="cuda", dtype=dtype)
    K.maxpool2_fwd(x, y, N, H, H, C)
    ys = misaligned_like(y.numel(), dtype).view_as(y)
    K.maxpool2_fwd(x, ys, N, H, H, C)
    dy = randn(N, H // 2, H // 2, C, dtype=dtype)
    dx = torch.empty_like(x)
    K.maxpool2_bwd(x, dy, dx, N, H, H, C)
    dxs = misaligned_like(x.numel(), dtype).view_as(x)
    K.maxpool2_bwd(x, dy, dxs, N, H, H, C)
    check_maxpool(x, y, dy, dx, N, H, H, C, f"{label} {dtype}")
    for n0 in range(0, N, 256):
        sl = slice(n0, n0 + 256)
        assert torch.equal(ys[sl], y[sl]) and torch.equal(dxs[sl], dx[sl]), f"scalar and vector paths differ, images [{n0}, ..)"
    print(f"[exact] maxpool2 fwd/bwd {dtype} N={N} {H}x{H}x{C}: exact, scalar == vector")
    del x, y, ys, dy, dx, dxs
    release()


def run_upsample(K, N, H, C, dtype, label):
    """upsample2_fwd / upsample2_bwd from an N x H x H x C map: forward exact; backward bit for bit against torch's fp32
    (a + b) + (c + d) and within one rounding of float64; the scalar paths equal the vector ones."""
    torch.manual_seed(27)
    x = randn(N, H, H, C, dtype=dtype)
    u = torch.empty(N, 2 * H, 2 * H, C, device="cuda", dtype=dtype)
    K.upsample2_fwd(x, u, N, H, H, C)
    us = misaligned_like(u.numel(), dtype).view_as(u)
    K.upsample2_fwd(x, us, N, H, H, C)
    check_upsample_fwd(x, u, N, H, H, C, f"{label} {dtype}")
    for n0 in range(0, N, 256):
        assert torch.equal(us[n0:n0 + 256], u[n0:n0 + 256]), f"upsample2_fwd scalar and vector paths differ, images [{n0}, ..)"
    del us
    dy = u.normal_()   # the 64x64 gradient map, reusing the upsampled buffer
    dx = torch.empty(N, H, H, C, device="cuda", dtype=dtype)
    K.upsample2_bwd(dy, dx, N, H, H, C)
    dxs = misaligned_like(dx.numel(), dtype).view_as(dx)
    K.upsample2_bwd(dy, dxs, N, H, H, C)
    worst = check_upsample_bwd(dy, dx, N, H, H, C, f"{label} {dtype}")
    for n0 in range(0, N, 256):
        assert torch.equal(dxs[n0:n0 + 256], dx[n0:n0 + 256]), f"upsample2_bwd scalar and vector paths differ, images [{n0}, ..)"
    print(f"[bound] upsample2 {dtype} N={N} {H}x{H}x{C}: fwd exact, bwd bit-exact, worst error/bound vs float64 {worst:.3g}")
    del x, u, dy, dx, dxs
    release()


def run_im2col3_col2im3(K, N, H, dtype, label):
    """The 3-channel ends on N frames of H x H x 3: im2col3's row32 path (ld = 32) against the generic one (ld = 40) and an
    exact statement for both tap signs, pad columns zero; col2im3 within 9 fp32 adds and one rounding."""
    C = 3
    torch.manual_seed(28)
    x = randn(N, H, H, C, dtype=dtype)
    for sgn in (1, -1):
        c32 = torch.full((N * H * H, 32), 7.0, device="cuda", dtype=dtype)
        c40 = torch.full((N * H * H, 40), 7.0, device="cuda", dtype=dtype)
        K.im2col3(x, c32, N, H, H, C, 32, sgn)
        K.im2col3(x, c40, N, H, H, C, 40, sgn)
        check_im2col3(x, c40, N, H, H, C, 40, sgn, f"{label} generic {dtype}")
        check_im2col3(x, c32, N, H, H, C, 32, sgn, f"{label} row32 {dtype}")
        del c32, c40
    ld = 32
    col = randn(N * H * H, ld, dtype=dtype)
    bias = randn(C, dtype=torch.float32)
    y = torch.full((N, H, H, C), NAN, device="cuda", dtype=dtype)
    K.col2im3(col, y, N, H, H, C, ld, bias=bias)
    worst = check_col2im3(col, y, N, H, H, C, ld, bias, f"{label} {dtype}")
    print(f"[bound] im2col3 exact (row32 == generic), col2im3 {dtype}: worst error/bound {worst:.3g}")
    del x, col, y
    release()


def run_skip_index(K, G, B, H, C, dtype, gather):
    """(gather: gather_add,) group_sum and add_indexed over G groups of B images of H x H x C, three distinct skip sources."""
    nsrc = 3
    n = B * H * H * C
    src = torch.tensor([(g + 1) % nsrc for g in range(G)], dtype=torch.int32, device="cuda")
    srcl = src.tolist()
    torch.manual_seed(29)
    big = randn(G * n, dtype=dtype)
    if gather:
        small = randn(nsrc * n, dtype=torch.float32)
        dst0 = big.clone()
        # gather_add: dst[g] += src[grp_src[g]] (fp32 addend); a bf16 destination rounds twice (fp32, then bf16): one bf16 ulp
        K.gather_add(big, small, src, G, n)
        worst = 0.0
        for g in range(G):
            ref = dst0[g * n:(g + 1) * n].double() + small[srcl[g] * n:(srcl[g] + 1) * n].double()
            rel = 2.0 ** -7 if dtype == torch.bfloat16 else 2.0 ** -23
            worst = max(worst, bound_check(big[g * n:(g + 1) * n], ref, rel * ref.abs(), f"gather_add group {g}"))
        print(f"[bound] gather_add {dtype} G={G} n={n}: worst error/bound {worst:.3g}")
        del dst0, small
    # group_sum: out[f] = sum over the groups reading source f (fp32 in group order, one output rounding)
    out = torch.full((nsrc * n,), NAN, device="cuda", dtype=dtype)
    K.group_sum(big, out, src, G, nsrc, n)
    worst = 0.0
    for f in range(nsrc):
        for j0 in range(0, n, 1 << 24):
            j1 = min(n, j0 + (1 << 24))
            gs = [g for g in range(G) if srcl[g] == f]
            ref = sum(big[g * n + j0:g * n + j1].double() for g in gs)
            mag = sum(big[g * n + j0:g * n + j1].double().abs() for g in gs)
            worst = max(worst, bound_check(out[f * n + j0:f * n + j1], ref, len(gs) * 2.0 ** -24 * mag + BETA[dtype] * ref.abs(),
                                            f"group_sum source {f}"))
    print(f"[bound] group_sum {dtype}: worst error/bound {worst:.3g}")
    # add_indexed: dst[dst_idx[f]] += src[f]; the other groups untouched
    dst_idx = torch.tensor([2, 0, 1], dtype=torch.int32, device="cuda")
    dst0 = big.clone()
    K.add_indexed(big, out, dst_idx, nsrc, n)
    worst = 0.0
    for f, d in enumerate(dst_idx.tolist()):
        ref = dst0[d * n:(d + 1) * n].double() + out[f * n:(f + 1) * n].double()
        worst = max(worst, bound_check(big[d * n:(d + 1) * n], ref, BETA[dtype] * ref.abs(), f"add_indexed {f} -> {d}"))
    assert torch.equal(big[nsrc * n:], dst0[nsrc * n:]), "add_indexed wrote outside its destination groups"
    print(f"[bound] add_indexed {dtype}: worst error/bound {worst:.3g}")
    del big, dst0, out
    release()


# ------------------------------------------------------------------ the audited step

AUDIT_CASES = [("bench_options", BENCH_OPT), ("skip_lfs", SKIP_OPT)]


class VggAudit(AuditKernels):
    """AuditKernels for a vgg step: also its convolutions (kinds 3, 4, 5), the 3-channel ends, pooling and upsampling, the
    fp32 skip gather and the BatchNorm finalize."""
    PRINT_RECORDS = True

    # ---- convolutions
    def conv_gemm(self, kind, a, b, c, N, H, W, Ck, Cn, Cm=0, ldb=None, ldc=None, bias=None, addend=None, grp_src=None,
                  imgs_per_group=0, accumulate=False, stat_partial=None, eval_scale=None, eval_shift=None, act=0):
        assert kind in (3, 4, 5) and H == W and eval_scale is None, f"unexpected conv_gemm launch kind {kind} in a vgg step"
        torch.cuda.synchronize()
        c0 = c.clone() if accumulate else None
        self._sync("conv_gemm", kind, a, b, c, N, H, W, Ck, Cn, Cm, ldb, ldc, bias, addend, grp_src, imgs_per_group, accumulate,
                   stat_partial, eval_scale, eval_shift, act)
        if kind == 4:
            s = conv_tiles(4, N, H, W, 0, Cn, Cm, self._sms)
            npx = N * H * W
            ref, absref = wgrad_ref64(a.view(-1)[:npx * Cm].view(N, H, W, Cm), b.view(-1)[:npx * Cn].view(N, H, W, Cn), N, H, Cm, Cn)
            if c0 is not None:
                ref += c0.view(-1)[:Cm * 9 * Cn].view(Cm, 9 * Cn).double()
                absref += c0.view(-1)[:Cm * 9 * Cn].view(Cm, 9 * Cn).double().abs()
            got = c.view(-1)[:Cm * 9 * Cn].view(Cm, 9 * Cn)
            w = assert_within(got, ref, absref, s.kb_per_split * 64 + 16 * s.splits, torch.float32, quiet=True,
                              name=f"audit kind 4 N={N} {H}x{W} {Cm}x{Cn}")
            # the step's gradients cancel over these K, so the bound above is loose; the same launch on the 0 / 1 pattern of
            # its operands (x > 0) must be exact
            a01 = (a.view(-1)[:npx * Cm] > 0).bfloat16().view(N, H, W, Cm)
            b01 = (b.view(-1)[:npx * Cn] > 0).bfloat16().view(N, H, W, Cn)
            probe = torch.full((Cm, 9 * Cn), NAN, device=c.device)
            super().conv_gemm(4, a01, b01, probe, N, H, W, 0, Cn, Cm=Cm)
            assert_exact(probe, wgrad_ref64(a01, b01, N, H, Cm, Cn)[0], npx, f"audit kind 4 N={N} {H}x{W} {Cm}x{Cn} 0/1 probe")
            self._rec(f"conv_gemm kind 4 N={N} {H}x{W} {Cm}x{Cn}", variant(4, 0, Cn, False, None, c.dtype, swap=s.swap), w)
            return
        assert not accumulate
        x = a.view(-1)[:N * H * W * Ck].view(N, H, W, Ck)
        wt = b.view(-1)[:Cn * 9 * Ck].view(Cn, 9 * Ck)
        out = c.view(-1)[:N * H * W * Cn].view(N, H, W, Cn)
        add, idx = self._addend(addend, grp_src, imgs_per_group, N, H, Cn) if addend is not None else (None, None)
        nm = f"conv_gemm kind {kind} N={N} {H}x{W} {Ck}->{Cn}"
        w = check_conv3_sums(out, kind, x, wt, N, H, Ck, Cn, bias, add, idx, name="audit " + nm)
        for i0 in sorted({0, N // 2, N - 1}):   # three images element-wise
            ref, absref = conv3_ref64_elem(kind, x[i0:i0 + 1], wt, H, Ck, Cn, bias, add[idx[i0:i0 + 1]] if add is not None else None)
            w = max(w, assert_within(out[i0:i0 + 1], ref, absref, 9 * Ck, out.dtype, quiet=True, name=f"audit {nm} image {i0}"))
        if stat_partial is not None:
            tiles = cdiv(N * H * W, 128)
            w = max(w, check_stat_rows(stat_partial.view(-1)[:tiles * Cn * 2].view(tiles, Cn, 2), out, N, H, Cn, name="audit " + nm))
        self._rec(nm, variant(kind, Ck, Cn, stat_partial is not None, addend.dtype if addend is not None else None, c.dtype), w)

    # ---- 3-channel ends
    def im2col3(self, x, col, N, H, W, C, ld, sgn=1):
        self._sync("im2col3", x, col, N, H, W, C, ld, sgn)
        check_im2col3(x, col, N, H, W, C, ld, sgn, "audit")
        self._rec(f"im2col3 N={N} C={C} ld={ld}", ("im2col3", "row32" if ld == 32 and C in (1, 3) else "generic", sgn), 0.0)

    def col2im3(self, col, y, N, H, W, C, ld, bias=None):
        self._sync("col2im3", col, y, N, H, W, C, ld, bias)
        self._rec(f"col2im3 N={N}", ("col2im3",), check_col2im3(col, y, N, H, W, C, ld, bias, "audit"))

    # ---- pooling / upsampling
    def maxpool2_fwd(self, x, y, N, H, W, C):
        self._sync("maxpool2_fwd", x, y, N, H, W, C)
        check_maxpool(x, y, None, None, N, H, W, C, "audit")
        self._rec(f"maxpool2_fwd N={N} {H}x{W}x{C}", ("maxpool2_fwd",), 0.0)

    def maxpool2_bwd(self, x, dy, dx, N, H, W, C):
        self._sync("maxpool2_bwd", x, dy, dx, N, H, W, C)
        check_maxpool(x, None, dy, dx, N, H, W, C, "audit")
        self._rec(f"maxpool2_bwd N={N} {H}x{W}x{C}", ("maxpool2_bwd",), 0.0)

    def upsample2_fwd(self, x, y, N, H, W, C):
        self._sync("upsample2_fwd", x, y, N, H, W, C)
        check_upsample_fwd(x, y, N, H, W, C, "audit")
        self._rec(f"upsample2_fwd N={N} {H}x{W}x{C}", ("upsample2_fwd",), 0.0)

    def upsample2_bwd(self, dy, dx, N, H, W, C):
        self._sync("upsample2_bwd", dy, dx, N, H, W, C)
        self._rec(f"upsample2_bwd N={N} {H}x{W}x{C}", ("upsample2_bwd",), check_upsample_bwd(dy, dx, N, H, W, C, "audit"))

    # ---- the fp32 skip gather and the BatchNorm finalize
    def gather_add(self, dst, src, grp_src, G, n):
        torch.cuda.synchronize()
        d0 = dst.view(-1)[:G * n].clone()
        self._sync("gather_add", dst, src, grp_src, G, n)
        srcl = grp_src.tolist()
        ref = d0.double().view(G, n) + src.view(-1).double().view(-1, n)[srcl[:G]]
        rel = 2.0 ** -7 if dst.dtype == torch.bfloat16 else 2.0 ** -23
        self._rec(f"gather_add G={G}", ("gather_add",), bound_check(dst.view(-1)[:G * n].view(G, n), ref, rel * ref.abs(), "audit gather_add"))

    def bn_fwd_finalize_tiles(self, partial, parts_per_group, ldp, fold, G, R, C, gamma, beta, mean, invstd, var_unb, scale,
                              shift, eps=1e-5):
        self._sync("bn_fwd_finalize_tiles", partial, parts_per_group, ldp, fold, G, R, C, gamma, beta, mean, invstd, var_unb, scale,
                   shift, eps)
        assert fold == 1 and ldp == C
        p = partial.view(-1)[:G * parts_per_group * C * 2].view(G, parts_per_group, C, 2).double()
        s1, s2, m1 = p[..., 0].sum(1), p[..., 1].sum(1), p[..., 0].abs().sum(1)
        # the kernel's own operands are exact here: only the float64 combine order and the fp32 outputs differ
        w = 0.0
        for got, (ref, _), nm in zip((mean, invstd, var_unb, scale, shift), finalize_ref(s1, s2, m1, R, gamma, beta, eps, 0.0),
                                     ("mean", "invstd", "var_unbiased", "scale", "shift")):
            g = got.view(-1)[:G * C].view(G, C)
            mag = ref.abs() if nm != "shift" else beta.double().abs() + (s1 / R * scale.view(-1)[:G * C].view(G, C).double()).abs()
            if nm == "mean":
                mag = mag + 2.0 ** -30 * m1 / R
            w = max(w, bound_check(g, ref, 2.0 ** -20 * mag + 1e-30, f"audit finalize {nm}"))
        self._rec(f"bn_fwd_finalize_tiles G={G} C={C}", ("bn_fwd_finalize_tiles",), w)


def vgg_cfg(W0):
    return dict(g_dim=128, z_dim=10, rnn_size=256, channels=3, image_width=W0, backbone="vgg", predictor_rnn_layers=2,
                posterior_rnn_layers=1, prior_rnn_layers=1)


def audit_vgg_step(name, optkw, T, B, W0):
    """One eager bf16 vgg step (vgg_64 or vgg_128 by W0) with every launch checked as it runs (launch_audit.audit_step): every
    path of the derived launch list must occur, and every decoder stage entry reads, for decoder call s, the skip frame the
    reference's schedule names (models/p2p_model.py).  Returns the plain step's results."""
    def expect(plan):
        fwd = forward_launches(T, B, plan.S, plan.nskip, W0)
        want = set()
        for L in fwd + backward_launches(T, B, plan.S, plan.nskip, W0, plan.has_cpc):
            if L["kind"] == 4:
                want.add(variant(4, 0, L["Cn"], False, None, torch.float32, swap=conv_tiles(4, L["N"], L["H"], L["H"], 0, L["Cn"], L["Cm"], sm_count()).swap))
            else:
                want.add(variant(L["kind"], L["Ck"], L["Cn"], L["stat"] is not None, torch.bfloat16 if L["addend"] else None, torch.bfloat16))
        want |= {("maxpool2_fwd",), ("maxpool2_bwd",), ("upsample2_fwd",), ("upsample2_bwd",), ("group_sum",), ("add_indexed",),
                 ("bn_fwd_finalize_tiles",), ("col2im3",), ("im2col3", "row32", 1)}
        for v in [("k3", "bres", "-", "add_bf16", "rowcoop"), ("k3", "bn128", "stat", "add_bf16", "perrow"), ("k4", "swap"),
                  ("k4", "noswap"), ("k3", "bn128", "-", "-", "rowcoop"), ("k5", "bres", "-", "-", "rowcoop")]:
            assert v in want, f"the derived launch list lost {v}"
        return want, [plan.skip_src] * sum(1 for L in fwd if L["addend"])
    audit = VggAudit("cuda")
    _, plain = audit_step(TrainEngineVGG, vgg_cfg(W0), optkw, T, B, audit, expect, f"{name} {W0}x{W0}")
    assert any(v[0] == "gemm" for v in audit.seen)
    return plain
