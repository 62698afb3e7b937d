"""The vgg_64 and vgg_128 training steps' kernel launches, derived from the engine's layer tables, and the float64 statements
the launch tests check them against (tests/test_vgg_launches_gpu.py, tests/test_vgg128_launches_gpu.py).

`forward_launches` / `backward_launches` walk the backbone's layer tables (VGG_ENC / VGG_DEC for 64x64 frames, VGG_ENC_128 /
VGG_DEC_128 for 128x128) the way TrainEngineVGG.encode / decode / decoder_backward / encoder_backward do and ask the engine's
own rules (implicit_shape, TrainEngine.stat_buf with BN_FUSE_MIN) which launches take the implicit GEMM,
which get fused BatchNorm statistics and which carry the skip addend, so the list follows the engine when it changes.

The checkers work in image chunks so that float64 references of C3-sized tensors (up to 10^9 elements) stay a few GiB:
  * conv3_sums64: per-(image, channel) sums of a kind-3 / kind-5 output from per-tap window sums of the input, O(N H W Ck);
  * wgrad_ref64: the kind-4 weight gradient, accumulated over image chunks (9 float64 GEMMs per chunk);
  * stat rows / finalize: every fused statistics row against the float64 sums of the stored rows it covers, and the
    finalized BatchNorm statistics per group against float64 statistics of the stored output.
"""
import types

import torch
import torch.nn.functional as F

from p2pvg_b200.engine import TrainEngine
from p2pvg_b200.engine_vgg import VGG_DEC, VGG_DEC_128, VGG_ENC, VGG_ENC_128
from p2pvg_b200.layouts import implicit_shape
from tests.tc_schedule import BETA, alpha_for, assert_within, cdiv
from tests.test_tc_schedule_gpu import rows_by_tile

CHUNK = 1 << 25     # elements of one float64 chunk (256 MB)


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


def forward_launches(T, B, S, nskip, W0=64):
    """Every implicit-GEMM forward convolution of one bf16 vgg step (encode, then decode), in engine order."""
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


def backward_launches(T, B, S, nskip, W0=64, has_cpc=True):
    """The data-gradient (kind 5) and weight-gradient (kind 4) launches of one bf16 vgg step, in the order the step enqueues
    them (engine.py TrainEngine.phases, mode A): backward_decoder's decoder_backward(0, S) with weight and skip gradients over
    the S B reconstruction images (engine.py:1236), the CPC decode's decoder_backward(S, S + 1) with data gradients only over
    B images (backward_prior, :1355), then encoder_backward over all T B frames, where the first layer (3 input channels) has
    an explicit weight gradient and no data gradient."""
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


# ------------------------------------------------------------------ exact reductions

def binary01(shape, p=0.25):
    """bf16 0 / 1 operand, 1 with probability p.  Products are 0 / 1 and a K-long sum of them is an integer <= K: below 2^24 every
    fp32 partial sum is exact in any order, so a kernel's result must equal the float64 reference bit for bit."""
    return (torch.rand(*shape, device="cuda") < p).to(torch.bfloat16)


def assert_exact(got, ref, K, name):
    """The fp32 result of a reduction of 0 / 1 products over K < 2^24 terms equals float64 exactly."""
    assert K < 1 << 24, f"{name}: K = {K} is too long for exact fp32 integer sums"
    bad = got.double() != ref
    if bad.any():
        i = tuple(int(v) for v in torch.unravel_index(torch.nonzero(bad.flatten())[0, 0], got.shape))
        raise AssertionError(f"{name}: {int(bad.sum())}/{bad.numel()} elements differ from the exact integer sum, first at {i}: "
                             f"got {got[i].item():.9g}, exact {ref[i].item():.9g}")
    print(f"[exact] {name}: K={K}, largest sum {ref.max().item():.0f}, exact")


# ------------------------------------------------------------------ fused statistics

A_STAT = 2.0 ** -18   # a statistics row: a fixed-order fp32 tree over 128 stored values (see test_tc_schedule_gpu.py)


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


def bound_check(got, ref, bound, name):
    """|got - ref| <= bound element-wise (float64 ref and bound); returns the worst ratio."""
    diff = (got.double() - ref).abs()
    ratio = torch.where(bound > 0, diff / bound.clamp_min(1e-300), torch.where(diff > 0, torch.inf, 0.0))
    ratio = torch.nan_to_num(ratio, nan=torch.inf)
    worst = ratio.max().item()
    if worst > 1.0:
        i = int(ratio.argmax())
        raise AssertionError(f"{name}: worst ratio {worst:.3g} at {i}: got {got.flatten()[i].item():.8g}, "
                             f"ref {ref.flatten()[i].item():.8g}, bound {bound.flatten()[i].item():.3g}")
    return worst


def finalize_ref(s1, s2, m1, R, gamma, beta, eps, a_rel):
    """Float64 mean / invstd / var_unbiased / scale / shift of groups whose sums are (s1, s2) with magnitudes (m1 = sum|x|,
    s2 = sum x^2), each sum known within a_rel of its magnitude; returns [(ref, bound)] in the kernel's output order."""
    E1, E2 = m1 / R, s2 / R
    m = s1 / R
    var = (s2 / R - m * m).clamp_min(0.0)
    g, bt = gamma.double(), beta.double()
    invstd = 1.0 / torch.sqrt(var + eps)
    u = 2.0 ** -23
    d_m = a_rel * E1 + u * m.abs()
    d_var = 3.0 * a_rel * E2 + u * var
    d_is = invstd * (0.5 * d_var / (var + eps) * 1.01 + u)
    sc = g * invstd
    d_sc = g.abs() * d_is + u * sc.abs()
    sh = bt - m * sc
    d_sh = m.abs() * d_sc + sc.abs() * d_m + u * (bt.abs() + (m * sc).abs()) * 2
    varu = var * R / (R - 1)
    return [(m, d_m), (invstd, d_is), (varu, d_var * R / (R - 1) + u * varu), (sc, d_sc), (sh, d_sh)]


def check_finalize_vs_output(K, part, parts_per_group, out, G, rows_per_group, Cn, name=""):
    """bn_fwd_finalize_tiles with the engine's parts_per_group against float64 statistics of the stored output."""
    gamma = torch.rand(Cn, device=out.device) + 0.5
    beta = torch.randn(Cn, device=out.device)
    outs = [torch.empty(G * Cn, device=out.device) for _ in range(5)]
    K.bn_fwd_finalize_tiles(part, parts_per_group, Cn, 1, G, rows_per_group, Cn, gamma, beta, *outs)
    flat = out.reshape(G, rows_per_group, Cn)
    s1 = torch.empty(G, Cn, dtype=torch.float64, device=out.device)
    s2, m1 = torch.empty_like(s1), torch.empty_like(s1)
    per = max(1, CHUNK // Cn)
    for g in range(G):
        a = b = c = 0.0
        for r0 in range(0, rows_per_group, per):
            x = flat[g, r0:r0 + per].double()
            a, b, c = a + x.sum(0), b + (x * x).sum(0), c + x.abs().sum(0)
        s1[g], s2[g], m1[g] = a, b, c
    worst = 0.0
    for got, (ref, bound), nm in zip(outs, finalize_ref(s1, s2, m1, rows_per_group, gamma, beta, 1e-5, A_STAT),
                                     ("mean", "invstd", "var_unbiased", "scale", "shift")):
        worst = max(worst, bound_check(got.view(G, Cn), ref, bound, f"{name} finalize {nm}"))
    print(f"[bound] {name} finalize ({G} groups x {parts_per_group} parts): worst error/bound {worst:.3g}")
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


# ------------------------------------------------------------------ GEMM (p2pvg_gemm)

def gemm_ref64(A, B, M, N, Kd, a_mn, b_mn, lda, ldb, bias=None, addend=None, ldd=None, c0=None, rows=None):
    """C = opA(A) opB(B) + bias + addend + c0 in float64 (and over |.|) on strided views of the operands, chunked over M and K.
    rows = (m0, m1): only those rows of C (addend and c0 are then those rows too)."""
    Av = A.as_strided((Kd, M), (lda, 1)) if a_mn else A.as_strided((M, Kd), (lda, 1))
    if rows is not None:
        Av = Av[:, rows[0]:rows[1]] if a_mn else Av[rows[0]:rows[1]]
        M = rows[1] - rows[0]
    Bv = B.as_strided((Kd, N), (ldb, 1)) if b_mn else B.as_strided((N, Kd), (ldb, 1))
    ref = torch.zeros(M, N, dtype=torch.float64, device=A.device)
    absref = torch.zeros_like(ref)
    mc = max(1, min(M, CHUNK // max(1, min(Kd, 4096))))
    kc = max(1, min(Kd, CHUNK // max(mc, N)))
    for m0 in range(0, M, mc):
        for k0 in range(0, Kd, kc):
            a = (Av[k0:k0 + kc, m0:m0 + mc].t() if a_mn else Av[m0:m0 + mc, k0:k0 + kc]).double()
            b = (Bv[k0:k0 + kc] if b_mn else Bv[:, k0:k0 + kc].t()).double()
            ref[m0:m0 + mc] += a @ b
            absref[m0:m0 + mc] += a.abs() @ b.abs()
    for extra in (bias, addend, c0):
        if extra is not None:
            e = extra.double()
            ref += e
            absref += e.abs()
    return ref, absref


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
