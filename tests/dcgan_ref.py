"""The dcgan_64 / dcgan_128 training step's kernel launches, derived from the engine's rules, and the float64 statements the
launch tests check them against (tests/test_dcgan_launches_gpu.py).

`forward_launches` / `backward_launches` walk the dcgan stacks the way TrainEngine.encode / decode / decoder_backward /
encoder_backward do (engine.py line numbers beside each rule) and ask the engine's own rules (implicit_shape, TrainEngine.stat_buf
with BN_FUSE_MIN) which layers take the implicit GEMM and which get fused BatchNorm statistics, so the list follows the engine
when it changes.  Each entry is a dict with `op`:
  * "conv_gemm": kind, N, H (small map), Ck, Cn, Cm, bias, addend (dtype or None), ipg (images per addend group), nsrc, stat
    (TrainEngine.stat_buf's dict or None) and variant (the epilogue / tile path it takes);
  * "gemm": M, N, K, a_mn, b_mn, bias (the bf16 GEMMs of the dcgan stacks);
  * a BatchNorm entry point ("bn_fwd_stats", "bn_fwd_finalize_tiles", "bn_act", "bn_bwd", "bn_bwd_group_sum",
    "bn_bwd_wgrad_c1", "bn_param_grad"): G, R, C, act, F (skip sources) and dout (the reduce pass also sums a 64 -> 1 layer's
    weight gradient).
`key(L)` is what a recording of the step is compared on.

precision "fp32" derives the launches of the fp32 step instead (TrainEngine.implicit, bd, fuse_stats, fuse_last, bn_skip_sums,
bn_wgrad_c1 off): im2col / col2im, the gemm_simt GEMMs with their pitches, the unfused BatchNorm passes, the group_sum of the
decoder's dcol, add_indexed, colsum and sigmoid_mse, as launch_audit.gemm32 / op32 entries whose `key` is what
launch_audit.fp32_call_key logs for the call (tests/test_dcgan_fp32_launches_gpu.py, tests/test_fp32_launch_lists_cpu.py).

The float64 checkers work in image chunks (ref64.CHUNK elements) so that references of C2-sized tensors stay a few GiB.
"""
import types

import torch
import torch.nn.functional as F

from p2pvg_b200.engine import BN_FUSE_MIN, TrainEngine
from p2pvg_b200.layouts import implicit_shape
from tests.launch_audit import gemm32, op32
from tests.lstm_schedule import gamma
from tests.ref64 import A_STAT, CHUNK, bound_check
from tests.tc_schedule import BETA, alpha_for, assert_within, box_for, cdiv, conv_ref64, rows_by_tile
from tests.vgg_ref import row_cooperative

ACT_LRELU, ACT_TANH = 1, 2
G_DIM = 128


def chans(W0):
    """TrainEngine.__init__ (engine.py:161)."""
    return [64, 128, 256, 512] if W0 == 64 else [64, 128, 256, 512, 512]


def _stat_rule(rows, phases, C, rows_per_group, kred):
    """TrainEngine.stat_buf (engine.py:816-824) on a stand-in engine: None, or its dict without the buffer."""
    assert BN_FUSE_MIN == 2048 * 128
    stub = types.SimpleNamespace(fuse_stats=True, fbuf=lambda tag, n: None)
    return TrainEngine.stat_buf(stub, "", rows, phases, C, rows_per_group, kred=kred)


def conv_variant(kind, Cn, stat, addend_dtype, H, c_dtype=torch.bfloat16, eval_epi=False, accumulate=False):
    """The code path of a kind-0 / kind-2 launch: tile rows (conv_gemm.cu:575, 256 for kind 2 with 64 output channels, no
    statistics or eval epilogue and a map 256-pixel boxes tile), tile width, statistics, addend dtype and the store path
    (conv_gemm.cu:244: row-cooperative for plain bf16 outputs and bf16 addends)."""
    if kind == 1:
        return ("k1",)
    bm = 256 if kind == 2 and Cn == 64 and not stat and not eval_epi and box_for(256, H, H) else 128
    return (f"k{kind}", f"{bm}x{128 if Cn > 64 else 64}", "stat" if stat else "-",
            {None: "-", torch.bfloat16: "add_bf16", torch.float32: "add_f32"}[addend_dtype],
            "rowcoop" if row_cooperative(c_dtype, stat, accumulate, addend_dtype) and not eval_epi else "perrow")


def _conv(name, kind, N, H, Ck, Cn, Cm=0, bias=False, addend=None, ipg=0, nsrc=0, stat=None, B=0):
    v = conv_variant(kind, Cn, stat is not None, addend, H)
    return dict(op="conv_gemm", name=name, kind=kind, N=N, H=H, Ck=Ck, Cn=Cn, Cm=Cm, bias=bias, addend=addend, ipg=ipg, nsrc=nsrc,
                stat=stat, B=B, variant=v)


def _gemm(name, M, N, K, a_mn=False, b_mn=False, bias=False):
    return dict(op="gemm", name=name, M=M, N=N, K=K, a_mn=a_mn, b_mn=b_mn, bias=bias)


def _bn(op, name, G, R=None, C=None, act=None, F=None, dout=False):
    return dict(op=op, name=name, G=G, R=R, C=C, act=act, F=F, dout=dout)


def key(L):
    """What a recorded call is compared on (an fp32 entry: launch_audit.fp32_call_key of the call)."""
    if "key" in L:
        return L["key"]
    if L["op"] == "conv_gemm":
        return ("conv_gemm", L["kind"], L["N"], L["H"], L["Ck"], L["Cn"], L["Cm"], L["bias"], L["addend"], L["ipg"],
                L["stat"] is not None)
    if L["op"] == "gemm":
        return ("gemm", L["M"], L["N"], L["K"], L["a_mn"], L["b_mn"], L["bias"])
    return (L["op"], L["G"], L["R"], L["C"], L["act"], L["F"], L["dout"])


def _bn_forward(out, name, G, R, C, act, stat):
    """TrainEngine.bn_forward (engine.py:838-843)."""
    if stat is not None:
        out.append(_bn("bn_fwd_finalize_tiles", name, G, R, C))
    else:
        out.append(_bn("bn_fwd_stats", name, G, R, C))
    out.append(_bn("bn_act", name, G, R, C, act))


def _stack(nc, W0):
    ch = chans(W0)
    n = len(ch)
    # pack_weights (engine.py:331, :346): block-diagonal copies for the 1- / 3-channel ends whose 16 nc is not a multiple of 64
    return ch, n, (16 * nc) % 64 != 0


def forward_launches(T, B, S, nskip, nc, W0, precision="bf16"):
    """encode (engine.py:761-800) then decode (engine.py:944-1004), in engine order.  precision "fp32": the fp32 step's
    launches (_forward32), entries with op32 / gemm32 keys."""
    if precision == "fp32":
        return _forward32(T, B, S, nskip, nc, W0)
    ch, n, bd = _stack(nc, W0)
    out = []
    N = T * B
    H = W0
    for l in range(n):
        cin = nc if l == 0 else ch[l - 1]
        cout = ch[l]
        Ho = H // 2
        M = N * Ho * Ho
        if implicit_shape(cin, cout):                                         # :777-782
            st = _stat_rule(M, 1, cout, B * Ho * Ho, 16 * cin)
            out.append(_conv(f"enc{l}", 0, N, Ho, cin, cout, bias=True, stat=st, B=B))
        elif l == 0 and bd:                                                   # :786-787
            out.append(_gemm("enc0.bd", M // 4, 4 * cout, 64 * cin, bias=True))
            st = None
        else:
            out.append(_gemm(f"enc{l}", M, cout, 16 * cin, bias=True))
            st = None
        _bn_forward(out, f"enc{l}", T, B * Ho * Ho, cout, ACT_LRELU, st)
        H = Ho
    out.append(_gemm("enc_final", N, G_DIM, 16 * ch[-1], bias=True))       # :798
    _bn_forward(out, "enc_final", T, B, G_DIM, ACT_TANH, None)
    G = S + 1
    N = G * B
    out.append(_gemm("dec-1", N, 16 * ch[-1], G_DIM, b_mn=True, bias=True))   # :958
    _bn_forward(out, "dec-1", G, B * 16, ch[-1], ACT_LRELU, None)
    Hi = 4
    for k in range(n):
        cd = ch[n - 1 - k]
        cout = ch[n - 2 - k] if k < n - 1 else nc
        Md, Ms = N * Hi * Hi, nskip * B * Hi * Hi
        st = None
        if implicit_shape(cd, cout):                                          # :974-983
            out.append(_conv(f"dec{k}.S", 2, nskip * B, Hi, cd, cout, bias=True, B=B))
            st = _stat_rule(Md, 4, cout, B * Hi * Hi, 4 * cd) if k < n - 1 else None
            out.append(_conv(f"dec{k}.D", 2, N, Hi, cd, cout, addend=torch.bfloat16, ipg=B, nsrc=nskip, stat=st, B=B))
        elif k == n - 1 and bd:                                               # :987-989; the last layer: convt_c1_loss
            out.append(_gemm("dec_last.bdD", Md // 4, 64 * cout, 4 * cd, b_mn=True))
            out.append(_gemm("dec_last.bdS", Ms // 4, 64 * cout, 4 * cd, b_mn=True))
        else:
            out.append(_gemm(f"dec{k}.D", Md, 16 * cout, cd, b_mn=True))
            out.append(_gemm(f"dec{k}.S", Ms, 16 * cout, cd, b_mn=True))
        if k < n - 1:
            _bn_forward(out, f"dec{k}", G, B * 4 * Hi * Hi, cout, ACT_LRELU, st)
        Hi *= 2
    return out


def _decoder_backward(out, g0, g1, B, nskip, nc, W0, want_wgrad, want_skip, tag):
    """TrainEngine.decoder_backward (engine.py:1032-1148)."""
    ch, n, bd = _stack(nc, W0)
    Gn = g1 - g0
    N = Gn * B
    imp = [implicit_shape(ch[n - 1 - k], ch[n - 2 - k] if k < n - 1 else nc) for k in range(n)]
    cd_last = ch[0]
    # :1044-1045: a 64 -> 1 last layer's D-half weight gradient is summed in the previous stage's BatchNorm reduce pass
    wg_last = want_wgrad and want_skip and n >= 2 and nc == 1 and cd_last == 64 and not imp[n - 1] and imp[n - 2]
    deferred = False
    Hi = 4 << (n - 1)
    for k in range(n - 1, -1, -1):
        cd = ch[n - 1 - k]
        cout = ch[n - 2 - k] if k < n - 1 else nc
        Md, Ms = N * Hi * Hi, nskip * B * Hi * Hi
        Ho = 2 * Hi
        nm = f"{tag}dec{k}"
        fused_skip = want_skip and imp[k] and k < n - 1                       # :1055-1056 (bn_skip_sums)
        if k < n - 1:
            if fused_skip:                                                    # :1061-1068
                out.append(_bn("bn_bwd_group_sum", nm, Gn, B * Ho * Ho, cout, ACT_LRELU, F=nskip, dout=deferred))
                deferred = False
            else:
                out.append(_bn("bn_bwd", nm, Gn, B * Ho * Ho, cout, ACT_LRELU))
            if want_wgrad:
                out.append(_bn("bn_param_grad", nm, Gn, C=cout))
        if imp[k]:                                                            # :1085-1101
            if want_wgrad:
                out.append(_conv(f"{nm} wgrad D", 1, N, Hi, 0, cout, Cm=cd))
            if want_skip:
                out.append(_conv(f"{nm} dgrad S", 0, nskip * B, Hi, cout, cd))
                if want_wgrad:
                    out.append(_conv(f"{nm} wgrad S", 1, nskip * B, Hi, 0, cout, Cm=cd))
            out.append(_conv(f"{nm} dgrad D", 0, N, Hi, cout, cd))
        else:                                                                 # :1103-1126
            bdl = k == n - 1 and bd
            out.append(_gemm(f"{nm} dgrad D", Md // 4, 4 * cd, 64 * cout) if bdl else _gemm(f"{nm} dgrad D", Md, cd, 16 * cout))
            if want_wgrad and not (wg_last and k == n - 1):
                out.append(_gemm(f"{nm} wgrad D", cd, 16 * cout, Md, a_mn=True, b_mn=True))
            if want_skip:
                out.append(_gemm(f"{nm} dgrad S", Ms // 4, 4 * cd, 64 * cout) if bdl else _gemm(f"{nm} dgrad S", Ms, cd, 16 * cout))
                if want_wgrad:
                    out.append(_gemm(f"{nm} wgrad S", cd, 16 * cout, Ms, a_mn=True, b_mn=True))
            deferred = wg_last and k == n - 1
        Hi //= 2
    ctop = ch[-1]                                                             # :1129-1148
    out.append(_bn("bn_bwd", f"{tag}dec-1", Gn, B * 16, ctop, ACT_LRELU))
    if want_wgrad:
        out.append(_bn("bn_param_grad", f"{tag}dec-1", Gn, C=ctop))
        out.append(_gemm(f"{tag}dec-1 wgrad", G_DIM, 16 * ctop, N, a_mn=True, b_mn=True))
    out.append(_gemm(f"{tag}dec-1 dgrad", N, G_DIM, 16 * ctop))


def backward_launches(T, B, S, nskip, nc, W0, has_cpc=True, precision="bf16"):
    """backward_decoder (engine.py:1236), the CPC chain of backward_prior (:1355) and encoder_backward (:1286-1344), in the
    order the step enqueues them (engine.py:679-696, mode A).  precision "fp32": _backward32."""
    if precision == "fp32":
        return _backward32(T, B, S, nskip, nc, W0, has_cpc)
    ch, n, bd = _stack(nc, W0)
    out = []
    _decoder_backward(out, 0, S, B, nskip, nc, W0, True, True, "")
    if has_cpc:
        _decoder_backward(out, S, S + 1, B, nskip, nc, W0, False, False, "cpc ")
    N = T * B
    ctop = ch[-1]
    out.append(_bn("bn_bwd", "enc_final", T, B, G_DIM, ACT_TANH))
    out.append(_bn("bn_param_grad", "enc_final", T, C=G_DIM))
    out.append(_gemm("enc_final wgrad", G_DIM, 16 * ctop, N, a_mn=True, b_mn=True))
    out.append(_gemm("enc_final dgrad", N, 16 * ctop, G_DIM, b_mn=True))
    H = W0 >> (n - 1)
    for l in range(n - 1, -1, -1):
        cin = nc if l == 0 else ch[l - 1]
        cout = ch[l]
        Ho = H // 2
        M = N * Ho * Ho
        if l == 0 and cin == 1 and cout == 64:                               # :1319-1326 (bn_wgrad_c1)
            out.append(_bn("bn_bwd_wgrad_c1", f"enc{l}", T, B * Ho * Ho, 64, ACT_LRELU))
            out.append(_bn("bn_param_grad", f"enc{l}", T, C=cout))
            continue
        out.append(_bn("bn_bwd", f"enc{l}", T, B * Ho * Ho, cout, ACT_LRELU))
        out.append(_bn("bn_param_grad", f"enc{l}", T, C=cout))
        imp = implicit_shape(cin, cout)
        if imp:
            out.append(_conv(f"enc{l} wgrad", 1, N, Ho, 0, cin, Cm=cout))
        else:
            out.append(_gemm(f"enc{l} wgrad", cout, 16 * cin, M, a_mn=True, b_mn=True))
        if l > 0:
            out.append(_conv(f"enc{l} dgrad", 2, N, Ho, cout, cin) if imp else _gemm(f"enc{l} dgrad", M, 16 * cin, cout, b_mn=True))
        H *= 2
    return out


def step_launches(T, B, S, nskip, nc, W0, has_cpc=True, precision="bf16"):
    return forward_launches(T, B, S, nskip, nc, W0, precision) + backward_launches(T, B, S, nskip, nc, W0, has_cpc, precision)


# ------------------------------------------------------------------ the fp32 step's launches

def _bn_forward32(out, name, G, R, C, act):
    """TrainEngine.bn_forward (engine.py:838-840) without fused statistics."""
    out += [op32("bn_fwd_stats", name, G, R, C), op32("bn_act", name, G, R, C, act)]


def _forward32(T, B, S, nskip, nc, W0):
    """encode (engine.py:750-784) and decode (:941-1011) with TrainEngine.implicit, bd and fuse_last off (act_dtype fp32,
    engine.py:207-215): every 4x4 convolution is im2col -> gemm_simt, every transposed one gemm_simt -> col2im."""
    ch, n = chans(W0), len(chans(W0))
    out = []
    N, H = T * B, W0
    for l in range(n):
        cin, cout = (nc if l == 0 else ch[l - 1]), ch[l]
        Ho = H // 2
        out.append(op32("im2col", f"enc{l}", N, H, cin))                                       # :774
        out.append(gemm32(f"enc{l}", N * Ho * Ho, cout, 16 * cin, bias=True))                   # :778
        _bn_forward32(out, f"enc{l}", T, B * Ho * Ho, cout, ACT_LRELU)                          # :779
        H = Ho
    out.append(gemm32("enc_top", N, G_DIM, 16 * ch[-1], bias=True))                             # encode_top :793
    _bn_forward32(out, "enc_top", T, B, G_DIM, ACT_TANH)
    G = S + 1
    N = G * B
    out.append(gemm32("dec-1", N, 16 * ch[-1], G_DIM, b_mn=True, bias=True))                    # decode_head :1008
    _bn_forward32(out, "dec-1", G, B * 16, ch[-1], ACT_LRELU)
    Hi = 4
    for k in range(n):
        cd, cout = ch[n - 1 - k], (ch[n - 2 - k] if k < n - 1 else nc)
        out.append(gemm32(f"dec{k}.D", N * Hi * Hi, 16 * cout, cd, b_mn=True))                  # :977
        out.append(gemm32(f"dec{k}.S", nskip * B * Hi * Hi, 16 * cout, cd, b_mn=True))          # :978
        out.append(op32("col2im", f"dec{k}", N, Hi, cout, True, True, B))                       # :983
        if k < n - 1:
            _bn_forward32(out, f"dec{k}", G, B * 4 * Hi * Hi, cout, ACT_LRELU)                 # :987
        Hi *= 2
    out.append(op32("sigmoid_mse", "loss", G, B * nc * W0 * W0))                                # losses_fwd :1026
    return out


def _decoder_backward32(out, Gn, B, nskip, nc, W0, want_wgrad, want_skip, tag):
    """TrainEngine.decoder_backward (engine.py:1032-1128) on the explicit path (implicit, bn_skip_sums off), then
    decode_head_backward (:1130-1154)."""
    ch, n = chans(W0), len(chans(W0))
    N = Gn * B
    Hi = 4 << (n - 1)
    for k in range(n - 1, -1, -1):
        cd, cout = ch[n - 1 - k], (ch[n - 2 - k] if k < n - 1 else nc)
        Md, Ms, Ho = N * Hi * Hi, nskip * B * Hi * Hi, 2 * Hi
        nm = f"{tag}dec{k}"
        if k < n - 1:
            out.append(op32("bn_bwd", nm, Gn, B * Ho * Ho, cout, ACT_LRELU))                   # :1073
            if want_wgrad:
                out.append(op32("bn_param_grad", nm, Gn, cout))                                 # :1075
        elif want_wgrad:
            out.append(op32("colsum", f"{nm} bias grad", N * Ho * Ho, cout, cout))              # :1078
        out.append(op32("im2col", f"{nm} dcol", N, Ho, cout))                                   # :1104
        out.append(gemm32(f"{nm} dgrad D", Md, cd, 16 * cout))                                  # :1109
        if want_wgrad:
            out.append(gemm32(f"{nm} wgrad D", cd, 16 * cout, Md, a_mn=True, b_mn=True))        # :1111
        if want_skip:
            out.append(op32("group_sum", f"{nm} dcol skip sum", Gn, nskip, B * Hi * Hi * 16 * cout))   # :1114
            out.append(gemm32(f"{nm} dgrad S", Ms, cd, 16 * cout))                              # :1119
            if want_wgrad:
                out.append(gemm32(f"{nm} wgrad S", cd, 16 * cout, Ms, a_mn=True, b_mn=True))    # :1122
        Hi //= 2
    ctop = ch[-1]
    out.append(op32("bn_bwd", f"{tag}dec-1", Gn, B * 16, ctop, ACT_LRELU))                      # :1140
    if want_wgrad:
        out.append(op32("bn_param_grad", f"{tag}dec-1", Gn, ctop))                              # :1143
        out.append(gemm32(f"{tag}dec-1 wgrad", G_DIM, 16 * ctop, N, a_mn=True, b_mn=True))      # :1146
    out.append(gemm32(f"{tag}dec-1 dgrad", N, G_DIM, 16 * ctop))                                # :1150


def encode_top_backward32(out, T, B, ctop=512):
    """TrainEngine.encode_top_backward (engine.py:1337-1355), fp32: dy is dH itself."""
    N = T * B
    out.append(op32("bn_bwd", "enc_top", T, B, G_DIM, ACT_TANH))
    out.append(op32("bn_param_grad", "enc_top", T, G_DIM))
    out.append(gemm32("enc_top wgrad", G_DIM, 16 * ctop, N, a_mn=True, b_mn=True))
    out.append(gemm32("enc_top dgrad", N, 16 * ctop, G_DIM, b_mn=True))


def _backward32(T, B, S, nskip, nc, W0, has_cpc):
    """backward_decoder's decoder_backward(0, S) (engine.py:1242), backward_prior's CPC decoder_backward(S, S + 1) (:1366) and
    encoder_backward (:1292-1335) with bn_wgrad_c1 off, in the order the serial fp32 step enqueues them (:684-688)."""
    ch, n = chans(W0), len(chans(W0))
    out = []
    _decoder_backward32(out, S, B, nskip, nc, W0, True, True, "")
    if has_cpc:
        _decoder_backward32(out, 1, B, nskip, nc, W0, False, False, "cpc ")
    encode_top_backward32(out, T, B, ch[-1])
    N = T * B
    H = W0 >> (n - 1)
    for l in range(n - 1, -1, -1):
        cin, cout = (nc if l == 0 else ch[l - 1]), ch[l]
        Ho = H // 2
        M = N * Ho * Ho
        out.append(op32("add_indexed", f"enc{l} skip grad", nskip, B * Ho * Ho * cout))         # :1307
        out.append(op32("bn_bwd", f"enc{l}", T, B * Ho * Ho, cout, ACT_LRELU))                  # :1318
        out.append(op32("bn_param_grad", f"enc{l}", T, cout))                                   # :1319
        out.append(gemm32(f"enc{l} wgrad", cout, 16 * cin, M, a_mn=True, b_mn=True))           # :1325
        if l > 0:
            out.append(gemm32(f"enc{l} dgrad", M, 16 * cin, cout, b_mn=True))                   # :1333
            out.append(op32("col2im", f"enc{l} dx", N, Ho, cin, False, False, 0))               # :1334
        H *= 2
    return out


# ------------------------------------------------------------------ the explicit lowering (conv_lower.cu)

def im2col_ref(x, N, H, C):
    """col[(n, oy, ox), (kh, kw, c)] = x[n, 2 oy - 1 + kh, 2 ox - 1 + kw, c], zero outside the map (conv_lower.cu:32)."""
    Ho = H // 2
    xp = F.pad(x.reshape(N, H, H, C), (0, 0, 1, 1, 1, 1))
    taps = [xp[:, kh:kh + 2 * Ho:2, kw:kw + 2 * Ho:2] for kh in range(4) for kw in range(4)]
    return torch.stack(taps, 3).reshape(N * Ho * Ho, 16 * C)


def check_im2col(x, col, N, H, C, name=""):
    """im2col bit-exact against the gather reference, image chunk by image chunk."""
    Ho = H // 2
    rows = Ho * Ho
    x = x.reshape(-1)[:N * H * H * C].view(N, H * H * C)
    col = col.reshape(-1)[:N * rows * 16 * C].view(N, rows * 16 * C)
    per = max(1, CHUNK // (rows * 16 * C))
    for n0 in range(0, N, per):
        n = min(per, N - n0)
        assert torch.equal(col[n0:n0 + n].reshape(n * rows, 16 * C), im2col_ref(x[n0:n0 + n], n, H, C)), \
            f"{name}: im2col N={N} {H}x{H}x{C} differs from the gather in images [{n0}, {n0 + n})"


def check_col2im(y, col, N, Hi, C, bias=None, col2=None, grp_src=None, ipg=0, name=""):
    """col2im (conv_lower.cu:107-177): y[n, oy, ox] = bias + the (up to) four taps (kh, kw) with oy = 2 iy - 1 + kh,
    ox = 2 ix - 1 + kw of col[n, iy, ix] and, with col2, of col2 at image grp_src[n // ipg] * ipg + n % ipg; an fp32 chain
    from the bias, one rounding per tap add (at most 8), stored as it is.  Against float64, image chunk by image chunk.
    Returns the worst ratio."""
    from tests.launch_audit import addend_index
    Ho = 2 * Hi
    cv = col.reshape(-1)[:N * Hi * Hi * 16 * C].view(N, Hi, Hi, 4, 4, C)
    yv = y.reshape(-1)[:N * Ho * Ho * C].view(N, Ho, Ho, C)
    idx = None
    if col2 is not None:
        idx = addend_index(grp_src.tolist()[:cdiv(N, ipg)], ipg, N, col.device)
        c2v = col2.reshape(-1)[:(int(idx.max()) + 1) * Hi * Hi * 16 * C].view(-1, Hi, Hi, 4, 4, C)
    per = max(1, CHUNK // (Hi * Hi * 16 * C))
    worst = 0.0
    for n0 in range(0, N, per):
        n1 = min(N, n0 + per)
        c = cv[n0:n1].double()
        m = c.abs()
        if idx is not None:
            c2 = c2v[idx[n0:n1]].double()
            c, m = c + c2, m + c2.abs()
            del c2
        ref = torch.zeros(n1 - n0, Ho + 2, Ho + 2, C, dtype=torch.float64, device=col.device)
        mag = torch.zeros_like(ref)
        for kh in range(4):
            for kw in range(4):
                ref[:, kh:kh + Ho:2, kw:kw + Ho:2] += c[:, :, :, kh, kw]
                mag[:, kh:kh + Ho:2, kw:kw + Ho:2] += m[:, :, :, kh, kw]
        ref, mag = ref[:, 1:-1, 1:-1], mag[:, 1:-1, 1:-1]
        if bias is not None:
            ref = ref + bias.double()
            mag = mag + bias.double().abs()
        worst = max(worst, bound_check(yv[n0:n1], ref, gamma(8) * mag, f"{name}: col2im images [{n0}, {n1})"))
        del c, m, ref, mag
    return worst


# ------------------------------------------------------------------ kinds 0 / 2: per-(image, channel) sums

def _tap_rows(kind, H):
    """[4, n_in] 0 / 1: input row r is read by tap kh for how many output rows (kind 0: out y reads in 2y + kh - 1 of a 2H map;
    kind 2: in row i writes out 2i + kh - 1 of a 2H map)."""
    if kind == 0:
        m = torch.zeros(4, 2 * H, dtype=torch.float64)
        for kh in range(4):
            for y in range(H):
                r = 2 * y + kh - 1
                if 0 <= r < 2 * H:
                    m[kh, r] += 1
    else:
        m = torch.zeros(4, H, dtype=torch.float64)
        for kh in range(4):
            for i in range(H):
                if 0 <= 2 * i + kh - 1 < 2 * H:
                    m[kh, i] += 1
    return m


def conv4_sums64(kind, a, b, N, H, Ck, Cn, bias=None, addend=None, add_idx=None):
    """(ref, absref) [N, Cn] float64: sum over the output pixels of a kind-0 / kind-2 launch, from per-tap window sums of the
    input (O(N H W Ck)), plus bias and the addend rows each image reads."""
    rows = _tap_rows(kind, H).to(a.device)
    if kind == 0:
        w = b.double().view(Cn, 4, 4, Ck)
        eq = "nabk,cabk->nc"
        npix = H * H
    else:
        w = b.double().view(Ck, 4, 4, Cn)
        eq = "nabk,kabc->nc"
        npix = 4 * H * H
    wa = w.abs()
    Hin = a.shape[1]
    per = max(1, CHUNK // (Hin * Hin * Ck))
    ref = torch.empty(N, Cn, dtype=torch.float64, device=a.device)
    absref = torch.empty_like(ref)
    for n0 in range(0, N, per):
        x = a[n0:n0 + per].double()
        ws = torch.einsum("nrsk,ar,bs->nabk", x, rows, rows)
        ref[n0:n0 + per] = torch.einsum(eq, ws, w)
        ws = torch.einsum("nrsk,ar,bs->nabk", x.abs_(), rows, rows)
        absref[n0:n0 + per] = torch.einsum(eq, ws, wa)
        del x, ws
    if bias is not None:
        ref += npix * bias.double()
        absref += npix * bias.double().abs()
    if addend is not None:
        s = torch.cat([addend[i:i + 16].double().sum((1, 2)) for i in range(0, addend.shape[0], 16)])
        sa = torch.cat([addend[i:i + 16].double().abs().sum((1, 2)) for i in range(0, addend.shape[0], 16)])
        ref += s[add_idx]
        absref += sa[add_idx]
    return ref, absref


def out_sums(out):
    N = out.shape[0]
    per = max(1, CHUNK // (out[0].numel()))
    s = torch.cat([out[i:i + per].double().sum((1, 2)) for i in range(0, N, per)])
    sa = torch.cat([out[i:i + per].double().abs().sum((1, 2)) for i in range(0, N, per)])
    return s, sa


def check_conv4_sums(out, kind, a, b, N, H, Ck, Cn, bias=None, addend=None, add_idx=None, name=""):
    """Per-(image, channel) sums of the whole output within alpha * sum|terms| + beta * sum|out| (see vgg_ref.check_conv3_sums)."""
    ref, absref = conv4_sums64(kind, a, b, N, H, Ck, Cn, bias, addend, add_idx)
    got, gabs = out_sums(out)
    diff = (got - ref).abs()
    bound = alpha_for(16 * Ck) * absref + BETA[out.dtype] * gabs
    ratio = torch.where(bound > 0, diff / bound.clamp_min(1e-300), torch.where(diff > 0, torch.inf, 0.0))
    ratio = torch.nan_to_num(ratio, nan=torch.inf)
    worst = ratio.max().item()
    if not worst <= 1.0:
        n, c = (int(i) for i in torch.unravel_index(ratio.argmax(), ratio.shape))
        raise AssertionError(f"{name}: per-(image, channel) sums: {int((ratio > 1).sum())}/{ratio.numel()} out of bound, worst "
                             f"{worst:.3g} at image {n} channel {c} (got {got[n, c].item():.6g}, ref {ref[n, c].item():.6g})")
    print(f"[bound] {name} image/channel sums: worst error/bound {worst:.3g}")
    return worst


def conv4_ref64_elem(kind, a, b, H, Ck, Cn, bias=None, addend_rows=None):
    """Element-wise float64 reference (and magnitude) of kind 0 / 2 on the images of `a`."""
    ref, absref = conv_ref64(kind, a, b, a.shape[0], H, H, Ck, Cn)
    for e in (bias, addend_rows):
        if e is not None:
            ref = ref + e.double()
            absref = absref + e.double().abs()
    return ref, absref


def check_stat_rows(part, out, kind, N, H, Cn, name=""):
    """Every partial row [(tile, phase), Cn, (sum, sum of squares)] against the float64 sums of the stored rows it covers,
    in tile-aligned image chunks.  H: small map."""
    HW = H * H
    phases = 4 if kind == 2 else 1
    unit = max(1, 128 // HW)
    per = max(unit, CHUNK // (HW * phases * Cn) // unit * unit)
    worst = 0.0
    for n0 in range(0, N, per):
        n = min(per, N - n0)
        rows = rows_by_tile(out[n0:n0 + n], kind, n, H, Cn, cdiv(n * HW, 128))
        t0 = n0 * HW // 128 * phases
        p = part[t0:t0 + rows.shape[0]]
        sq = rows * rows
        for j, (val, mag) in enumerate(((rows.sum(1), rows.abs().sum(1)), (sq.sum(1), sq.sum(1)))):
            worst = max(worst, assert_within(p[:, :, j], val, mag, 0, torch.float32, alpha=A_STAT, quiet=True,
                                             name=f"{name} stat rows from {t0} {'sum' if j == 0 else 'sumsq'}"))
        del rows, sq
    print(f"[bound] {name} statistics rows ({part.shape[0]} rows): worst error/bound {worst:.3g}")
    return worst


# ------------------------------------------------------------------ kind 1

def wgrad4_ref64(a, b, N, H, Cm, Cn):
    """Kind-1 weight gradient g[Cm, (tap, Cn)] = sum_pix a_small[pix, Cm]^T gather_s2(b_big)[pix, tap, Cn] in float64 (and over
    |.|), image chunk by image chunk."""
    ref = torch.zeros(Cm, 16, Cn, dtype=torch.float64, device=a.device)
    absref = torch.zeros_like(ref)
    per = max(1, CHUNK // (4 * H * H * max(Cm, Cn)))
    for n0 in range(0, N, per):
        x = a[n0:n0 + per].double().reshape(-1, Cm)
        bp = F.pad(b[n0:n0 + per].double(), (0, 0, 1, 1, 1, 1))     # big map, one pixel of zero padding
        for mag in (False, True):
            xa, bpa, dst = (x.abs(), bp.abs(), absref) if mag else (x, bp, ref)
            for tap in range(16):
                kh, kw = divmod(tap, 4)
                dst[:, tap] += xa.t() @ bpa[:, kh:kh + 2 * H:2, kw:kw + 2 * H:2].reshape(-1, Cn)
        del x, bp
    return ref.view(Cm, 16 * Cn), absref.view(Cm, 16 * Cn)


# ------------------------------------------------------------------ BatchNorm, group by group

BN_MAXCHUNK = 64


def bn_chunks(R, C, vec=8):
    """choose_chunks (bn.cu:676-684): (chunks per group, rows per chunk) of the BatchNorm passes; vec = 8 for bf16."""
    lanes = max(1, 256 // (C // vec))
    want = cdiv(R, lanes * 16)
    nchunk = max(1, min(want, BN_MAXCHUNK))
    rpc = cdiv(R, nchunk)
    return cdiv(R, rpc), rpc


def check_wgrad_c1(dw, exact, absum, R, C, name):
    """The 64 x 16 weight gradient of bn_bwd_wgrad_c1 / the `dout` reduce of bn_bwd_group_sum.  Its bf16 operands (dx or y as
    stored, the tap of the 1-channel map) multiply exactly in fp32; each wpart entry is one block's fp32 MMA accumulator over
    the rows_per_chunk rows of its chunk (bn.cu:457-504, :512-584), and wgrad_partials_finalize_kernel (bn.cu:605) adds the
    entries in float64 and rounds once to fp32: |dw - exact| <= alpha_for(rows_per_chunk) * sum|terms| + 2^-22 |exact|."""
    _, rpc = bn_chunks(R, C)
    return assert_within(dw.view(C, 16), exact, absum, rpc, torch.float32, name=f"{name} (rows per chunk {rpc})")


def taps_1ch64(cin, Ho):
    """float64 [n, 16, Ho*Ho] 4x4 / stride-2 / pad-1 patches of the 1-channel maps cin [n, 2Ho, 2Ho], tap = kh*4 + kw."""
    n = cin.numel() // (4 * Ho * Ho)
    return F.unfold(cin.reshape(n, 1, 2 * Ho, 2 * Ho).double(), kernel_size=4, stride=2, padding=1)


def wgrad_c1_ref64(d, cin, Ho, C=64):
    """sum over rows of d[row, c] * tap[row, t] in float64 (and over |.|), image chunk by chunk: d [n, Ho*Ho, C] (bf16) and the
    1-channel map cin [n, 2Ho, 2Ho]."""
    n = cin.numel() // (4 * Ho * Ho)
    d = d.reshape(n, Ho * Ho, C)
    cin = cin.reshape(n, 4 * Ho * Ho)
    per = max(1, CHUNK // (Ho * Ho * C))
    ref = torch.zeros(C, 16, dtype=torch.float64, device=d.device)
    mag = torch.zeros_like(ref)
    for i in range(0, n, per):
        dd = d[i:i + per].double()
        t = taps_1ch64(cin[i:i + per], Ho)
        ref += torch.einsum("npc,ntp->ct", dd, t)
        mag += torch.einsum("npc,ntp->ct", dd.abs(), t.abs())
    return ref, mag
