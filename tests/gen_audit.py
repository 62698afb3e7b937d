"""Float64 statements of the generation-only launches and an audited eager run of a captured generate call's body
(tests/test_generate_audit_gpu.py; the corruption tests in tests/test_gen_audit_cpu.py).

GenerateEngine._body (p2pvg_b200/gen_engine.py, and the vgg / pose hooks) is what every graphed generate, chain, lengths,
evaluate and vis_seq call replays.  ``audited_call`` runs one real call of a captured signature with its replay replaced by
the body run eagerly on ``GenAudit``, a view of CudaKernels that checks every launch against float64 on its own operands as
it runs (launch_audit.AuditKernels); the call's frames, LSTM state and output buffer must then equal a plain replay of the
same call bit for bit.

The float64 restatements below are plain torch functions (device-agnostic), so the CPU test can feed them emulations of the
kernels with deliberate corruptions.  Rounding: u = 2^-24; gamma(n) = n u / (1 - n u) bounds n fp32 roundings (Higham).
"""
import contextlib

import torch

from tests.dcgan_ref import check_conv4_sums, conv4_ref64_elem
from tests.launch_audit import kernel_for, simt_alpha
from tests.loss_ref import ACT_LRELU, ACT_TANH, TINY, act_fwd_ref
from tests.lstm_schedule import U, gamma
from tests.ref64 import bound_check
from tests.tc_schedule import BETA, alpha_for, assert_within, cdiv, gemm_tc_tiles
from tests.vgg_ref import VggAudit, check_conv3_sums, conv3_ref64_elem

LIBM = 4 * U          # expf, tanhf, rsqrtf: at most 2 ulp (CUDA C Programming Guide, single-precision maximum ulp errors)
LN_EPS = 1e-5         # pose_mlp.cu:24
POSE = 51


def dot_gamma(K, extra=0):
    """warp_dot (cluster_rows.cuh:8-22): each lane chains ceil(K / 32) fmaf, then 5 shuffle adds combine the lanes; `extra`
    roundings follow (bias adds)."""
    return gamma(cdiv(K, 32) + 5 + extra)


def linear64(x, w, b):
    """(x W^T + b, |x| |W|^T + |b|) in float64."""
    x, w = x.double(), w.double()
    ref, mag = x @ w.t(), x.abs() @ w.abs().t()
    if b is not None:
        ref, mag = ref + b.double(), mag + b.double().abs()
    return ref, mag


def _lin_err(x, xe, w, b, extra):
    """A warp_dot Linear on computed inputs x (float64 values of the fp32 operands) off by at most xe from the exact ones:
    (ref on x, bound of the fp32 result against the exact inputs' float64 value)."""
    ref, mag = linear64(x, w, b)
    e = dot_gamma(w.shape[1], extra) * mag
    if xe is not None:
        prop = xe.double() @ w.double().abs().t()
        e = e + prop * (1 + dot_gamma(w.shape[1], extra))
    return ref, e


# ------------------------------------------------------------------ p2pvg_lstm_step (lstm_step.cu)

def lstm_input64(seg_a, ia, ga, seg_b, ib, gb, tuc, dt, counter_rows, rows):
    """The module input rows of one launch (lstm_step.cu:23-30): [seg_a[ia] | seg_b[ib] | tuc | dt], row b reading the
    counters of group b // counter_rows (counter_rows 0: group 0).  Exact: a gather of fp32 values."""
    parts = [seg_a.reshape(-1)[ia * rows * ga:(ia + 1) * rows * ga].view(rows, ga).double()]
    if gb:
        parts.append(seg_b.reshape(-1)[ib * rows * gb:(ib + 1) * rows * gb].view(rows, gb).double())
    grp = torch.arange(rows, device=seg_a.device) // counter_rows if counter_rows > 0 else torch.zeros(rows, dtype=torch.long,
                                                                                                        device=seg_a.device)
    parts += [tuc.reshape(-1).double()[grp][:, None], dt.reshape(-1).double()[grp][:, None]]
    return torch.cat(parts, 1)


def embed64(X, w, b):
    """The embed Linear (lstm_step.cu:66-70): (float64 value, bound of the fp32 result).  One bias add after warp_dot."""
    return _lin_err(X, None, w, b, 1)


def lstm_cell64(x, xe, h0, c0, w_ih, b_ih, w_hh, b_hh):
    """One nn.LSTMCell (gate order i, f, g, o) in float64 on the input x (off by at most xe; None: exact) and the pre-launch
    state h0, c0, with the bound of lstm_step.cu's fp32 result.  Returns (h, c, e_h, e_c).

    Gate pre-activations (:83-86): two warp_dots, then (acc_ih + b_ih) + (acc_hh + b_hh): three roundings after the dots, and
    |W_ih| xe carried in from the input.  sigmoidf_ = 1 / (1 + expf(-x)) (common.cuh:103): expf 2 ulp, the add and the IEEE
    division one rounding each, so within 8u of its value, and Lipschitz 1/4 in its argument; tanhf 2 ulp and Lipschitz 1.
    c = f c0 + i g (:92) two roundings; h = o tanhf(c) (:93) tanhf's error, c's error, one rounding."""
    R = h0.shape[1]
    gi, mi = linear64(x, w_ih, b_ih)
    gh, mh = linear64(h0, w_hh, b_hh)
    pre = gi + gh
    n = max(cdiv(w_ih.shape[1], 32), cdiv(R, 32)) + 5 + 3
    e_pre = gamma(n) * (mi + mh)
    if xe is not None:
        e_pre = e_pre + (xe.double() @ w_ih.double().abs().t()) * (1 + gamma(n))
    q = [slice(k * R, (k + 1) * R) for k in range(4)]
    si, sf, so = (torch.sigmoid(pre[:, s]) for s in (q[0], q[1], q[3]))
    tg = torch.tanh(pre[:, q[2]])
    ei, ef, eo = (e_pre[:, s] / 4 + 8 * U * v for s, v in ((q[0], si), (q[1], sf), (q[3], so)))
    eg = e_pre[:, q[2]] + LIBM * tg.abs() + TINY
    c0 = c0.double()
    c = sf * c0 + si * tg
    e_c = ef * c0.abs() + ei * tg.abs() + (si + ei) * eg + 2.02 * U * (sf * c0.abs() + si * tg.abs())
    tc = torch.tanh(c)
    h = so * tc
    e_h = eo * tc.abs() + (so + eo) * (e_c + LIBM * tc.abs() + TINY) + 1.01 * U * h.abs()
    return h, c, e_h, e_c


def head_tanh64(h, w, b):
    """The lstm head tanh(h W^T + b) (lstm_step.cu:103-108): (value, bound)."""
    pre, e = _lin_err(h, None, w, b, 1)
    y = torch.tanh(pre)
    return y, e + LIBM * y.abs() + TINY


def head_gauss64(h, w_mu, b_mu, w_lv, b_lv, eps):
    """The gaussian head eps * exp(lv / 2) + mu (lstm_step.cu:109-121): (value, bound).  expf 2 ulp; its argument's error
    e_lv / 2 scales the exponential by at most exp(e_lv / 2); the product and the sum (or one fmaf) two roundings."""
    mu, e_mu = _lin_err(h, None, w_mu, b_mu, 1)
    lv, e_lv = _lin_err(h, None, w_lv, b_lv, 1)
    E = torch.exp(0.5 * lv)
    e_E = E * (torch.expm1(0.5 * e_lv) * (1 + LIBM) + LIBM)
    eps = eps.double()
    y = eps * E + mu
    return y, eps.abs() * e_E + e_mu + 2.02 * U * (eps.abs() * (E + e_E) + mu.abs()) + TINY


# ------------------------------------------------------------------ p2pvg_pose_mlp (pose_mlp.cu)

def residual_params(rl):
    """The parameters of a models.h36m_mlp.residual_linear as a dict of tensors."""
    return dict(w_sc=rl.shortcut[0].weight, b_sc=rl.shortcut[0].bias, w1=rl.long_path[0].weight, b1=rl.long_path[0].bias,
                w2=rl.long_path[2].weight, b2=rl.long_path[2].bias, w3=rl.long_path[4].weight, b3=rl.long_path[4].bias,
                gamma=rl.norm.weight, beta=rl.norm.bias)


def residual64(p, x, xe):
    """residual_linear (models/h36m_mlp.py:7-15) in float64 on x (off by at most xe; None: exact) with the bound of
    pose_mlp.cu's residual(): each Linear a warp_dot plus a bias add, ReLU Lipschitz 1, the residual add (:86) one rounding.
    LayerNorm (:90-103): the mean from lane sums (ceil(n / 32) adds per lane, 5 shuffles, the division), d = y - m one
    rounding, the variance the same over fmaf(d, d), var + eps and rsqrtf (2 ulp) with |d r'| <= r^3 / 2, then
    (d r) gamma + beta three roundings.  Returns (value, bound)."""
    a1, e1 = _lin_err(x, xe, p["w1"], p["b1"], 1)
    a1, e1 = a1.clamp_min(0), e1
    a2, e2 = _lin_err(a1, e1, p["w2"], p["b2"], 1)
    a2 = a2.clamp_min(0)
    a3, e3 = _lin_err(a2, e2, p["w3"], p["b3"], 1)
    sc, esc = _lin_err(x, xe, p["w_sc"], p["b_sc"], 1)
    y = sc.clamp_min(0) + a3.clamp_min(0)
    ey = (esc + e3) * (1 + U) + 1.01 * U * y.abs()
    n = y.shape[1]
    gs = gamma(cdiv(n, 32) + 5)
    m = y.mean(1, keepdim=True)
    em = (ey.sum(1, keepdim=True) + gs * y.abs().sum(1, keepdim=True)) / n * (1 + U) + 1.01 * U * m.abs()
    d = y - m
    ed = (ey + em) * (1 + U) + 1.01 * U * d.abs()
    var = (d * d).mean(1, keepdim=True)
    ev = ((2 * d.abs() * ed + ed * ed).sum(1, keepdim=True) + gs * (d * d + 2 * d.abs() * ed + ed * ed).sum(1, keepdim=True)) / n
    ev = ev * (1 + U) + 1.01 * U * var
    r = 1.0 / torch.sqrt(var + LN_EPS)
    # rsqrt of var + eps (one rounding of the sum): |d r / d var| = r^3 / 2, taken at the smallest var the error allows
    vlo = (var - ev - U * (var + LN_EPS)).clamp_min(0)
    rmax = 1.0 / torch.sqrt(vlo + LN_EPS)
    er = 0.5 * rmax ** 3 * (ev + 1.01 * U * (var + LN_EPS)) + LIBM * rmax
    g, bt = p["gamma"].double(), p["beta"].double()
    out = d * r * g + bt
    eo = g.abs() * (ed * (r + er) + d.abs() * er) + 3.03 * U * ((d * r * g).abs() + (d.abs() + ed) * er * g.abs() + bt.abs())
    return out, eo


def pose_encoder64(pe, x):
    """The encoder (models/h36m_mlp.py:17-28) on exact inputs x [rows, 51]: (h1, e1), and the fc2 / fc3 stages as functions
    of a stored input, so that each stage is checked on what the kernel stored before it."""
    h1, e1 = residual64(residual_params(pe.fc1), x, None)
    return h1, e1


def pose_encoder_top64(pe, h2):
    """tanh(fc3(h2)) on the stored h2 (pose_mlp.cu:154-159): (value, bound)."""
    return head_tanh64(h2, pe.fc3.weight, pe.fc3.bias)


def pose_decoder64(pd, vec, skip1, skip2, nsrc, skip_row=None):
    """The decoder (models/h36m_mlp.py:31-42; pose_mlp.cu:139-169) on exact inputs vec [rows, g], output row r reading skip
    row r % nsrc of skip1 (h1) and skip2 (h2): d1 = fc1(vec), d2 = fc2([d1 | h2]), out = fc3([d2 | h1]).  Nothing between the
    stages is stored, so each stage's bound is carried into the next.  skip_row(r, nsrc) replaces r % nsrc (the CPU test's
    corruption).  Returns (out, bound)."""
    rows = vec.shape[0]
    r = torch.arange(rows, device=vec.device)
    sr = r % nsrc if skip_row is None else skip_row(r, nsrc)
    s1, s2 = skip1.double()[sr], skip2.double()[sr]
    d1, e1 = residual64(residual_params(pd.fc1), vec.double(), None)
    z = torch.zeros_like(s2)
    d2, e2 = residual64(residual_params(pd.fc2), torch.cat([d1, s2], 1), torch.cat([e1, z], 1))
    return _lin_err(torch.cat([d2, s1], 1), torch.cat([e2, z], 1), pd.fc3.weight, pd.fc3.bias, 1)


# ------------------------------------------------------------------ eval-mode BatchNorm (bn.cu:643-650)

def bn_coeffs64(gamma_, beta, mean, var, eps, with_shift_term=True):
    """scale = gamma / sqrt(var + eps), shift = beta - mean scale in float64, with the bound of bn_eval_coeffs' fp32 result:
    var + eps (eps passed as a float: two roundings, <= u relative after the square root), sqrtf and the division correctly
    rounded (no fast-math): |d scale| <= 3.1 u |scale|; shift: mean * |d scale| plus the product and the difference (or one
    fmaf), <= 2.02 u (|mean scale| + |shift|).  with_shift_term=False drops mean * scale (the CPU test's corruption)."""
    sc = gamma_.double() / torch.sqrt(var.double() + eps)
    ms = mean.double() * sc if with_shift_term else torch.zeros_like(sc)
    sh = beta.double() - ms
    e_sc = 3.1 * U * sc.abs()
    e_sh = mean.double().abs() * e_sc + 2.02 * U * (ms.abs() + sh.abs()) + TINY
    return sc, sh, e_sc, e_sh


def bn_module64(x, gamma_, beta, mean, var, eps):
    """The module's eval form (x - running_mean) / sqrt(running_var + eps) * gamma + beta in float64, per channel (last dim)."""
    return (x.double() - mean.double()) / torch.sqrt(var.double() + eps) * gamma_.double() + beta.double()


def fold_bound(x, gamma_, beta, mean, var, eps):
    """|fmaf(x, scale, shift) - module(x)| with scale / shift from bn_eval_coeffs, x exact:
        |x| |d scale| + |d shift| + u |result|
      <= 3.1 u |x scale| + (3.1 + 2.02) u |mean scale| + 2.02 u |shift| + 1.01 u |result|.
    The first two terms do not shrink with the result: where |running_mean| >> sqrt(running_var) and x sits near the mean,
    |x scale| ~ |mean scale| ~ |mean| / sqrt(var) |gamma| while the result is ~ |gamma|, so the folded form loses about
    log2(|mean| / sqrt(var)) bits against the module's formula (at 100x: ~2^-15.5 relative to |gamma|, below one bf16
    rounding, about 160 fp32 roundings)."""
    sc = gamma_.double() / torch.sqrt(var.double() + eps)
    ms = (mean.double() * sc).abs()
    y = bn_module64(x, gamma_, beta, mean, var, eps)
    sh = (beta.double() - mean.double() * sc).abs()
    return 3.1 * U * (x.double() * sc).abs() + 5.12 * U * ms + 2.02 * U * sh + 1.01 * U * y.abs() + TINY


def act64(v, act):
    """The epilogue activation in float64 and its own rounding: LeakyReLU's 0.2f v one rounding, tanhf 2 ulp."""
    if act == ACT_LRELU:
        y = torch.where(v > 0, v, 0.2 * v)
        return y, 1.01 * U * y.abs()
    if act == ACT_TANH:
        y = torch.tanh(v)
        return y, LIBM * y.abs() + TINY
    return v, torch.zeros_like(v)


# ------------------------------------------------------------------ the explicit 4x4 / stride-2 lowering (conv_lower.cu)

def im2col4_ref(x):
    """col [N (H/2) (W/2), 16 C], K order (kh, kw, c) (conv_lower.cu:9): x[n, 2 oy + kh - 1, 2 ox + kw - 1, c], 0 outside."""
    N, H, W, C = x.shape
    xp = torch.nn.functional.pad(x.permute(0, 3, 1, 2), (1, 1, 1, 1)).permute(0, 2, 3, 1)
    taps = [xp[:, kh:kh + H:2, kw:kw + W:2] for kh in range(4) for kw in range(4)]
    return torch.stack(taps, 3).reshape(N * (H // 2) * (W // 2), 16 * C)


def col2im4_ref(col, N, Hi, Wi, C, bias=None):
    """y [N, 2 Hi, 2 Wi, C] = bias + sum of the taps (kh, kw) of input pixel (iy, ix) landing on (2 iy + kh - 1, 2 ix + kw - 1)
    (conv_lower.cu:105-147), float64 (value, sum of magnitudes)."""
    c = col.double().view(N, Hi, Wi, 4, 4, C)
    y = torch.zeros(N, 2 * Hi + 2, 2 * Wi + 2, C, dtype=torch.float64, device=col.device)
    m = torch.zeros_like(y)
    for kh in range(4):
        for kw in range(4):
            y[:, kh:kh + 2 * Hi:2, kw:kw + 2 * Wi:2] += c[:, :, :, kh, kw]
            m[:, kh:kh + 2 * Hi:2, kw:kw + 2 * Wi:2] += c[:, :, :, kh, kw].abs()
    y, m = y[:, 1:-1, 1:-1], m[:, 1:-1, 1:-1]
    if bias is not None:
        y, m = y + bias.double(), m + bias.double().abs()
    return y, m


# ------------------------------------------------------------------ the audited view

def _ptr_map(model):
    return {mod.embed.weight.data_ptr(): name for name in ("posterior", "prior", "frame_predictor")
            for mod in (getattr(model, name),)}


def _sample_images(N, nsrc):
    """The images an element-wise check covers: the ends, the middle and both sides of the first group boundary of a
    grp_zero addend (image nsrc reads source image 0 again)."""
    s = {0, N // 2, N - 1}
    if 0 < nsrc < N:
        s |= {nsrc - 1, nsrc}
    return sorted(i for i in s if 0 <= i < N)


class GenAudit(VggAudit):
    """AuditKernels for GenerateEngine._body: every launch of the dcgan, vgg and pose bodies checked against float64 on its
    own operands as it runs.  `model` is the P2PModel whose body runs (the LSTM and pose launches find their modules
    through it), `bufs` the graph's buffers (the LSTM state)."""
    PRINT_RECORDS = False

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.model, self.bufs = None, None
        self.bn_of = {}      # scale data_ptr -> (gamma, beta, running_mean, running_var, eps) of the module it came from
        self.fold_worst = 0.0

    def gemm_bound(self, A, B, M, N, K, a_mn, b_mn, lda, ldb, extra):
        if A.dtype == torch.bfloat16:
            s = gemm_tc_tiles(M, N, K, self._sms)
            return alpha_for(s.kb_per_split * 64 + 16 * s.splits), "tc"
        kern = kernel_for(M, N, K, a_mn, b_mn, lda, ldb, 0, 0, False)
        return simt_alpha(K, kern, extra), "simt"

    def gemm_variant(self, A, kern, a_mn, b_mn, accumulate, bias, strided):
        return ("gemm", str(A.dtype)[6:], kern)

    # ---- eval-mode BatchNorm
    def bn_eval_coeffs(self, gamma_, beta, rmean, rvar, C, scale, shift, eps=1e-5):
        self._sync("bn_eval_coeffs", gamma_, beta, rmean, rvar, C, scale, shift, eps)
        sc, sh, e_sc, e_sh = bn_coeffs64(gamma_[:C], beta[:C], rmean[:C], rvar[:C], eps)
        w = max(bound_check(scale[:C], sc, e_sc, "audit bn_eval_coeffs scale"), bound_check(shift[:C], sh, e_sh, "audit bn_eval_coeffs shift"))
        self.bn_of[scale.data_ptr()] = tuple(t[:C].detach().clone() for t in (gamma_, beta, rmean, rvar)) + (eps,)
        big = bool(((rmean[:C].double().abs() >= 100 * rvar[:C].double().sqrt())).any())
        self._rec(f"bn_eval_coeffs C={C}", ("bn_eval_coeffs", big), w)

    def _bn_ref(self, pre, pre_err, scale, act):
        """act(module BatchNorm(pre)) for the coefficients `scale` was computed from, and the bound of the kernel's
        act(fmaf(pre, scale, shift)) for a pre-activation off by at most pre_err."""
        g, b, m, v, eps = self.bn_of[scale.data_ptr()]
        y = bn_module64(pre, g, b, m, v, eps)
        fb = fold_bound(pre, g, b, m, v, eps)
        self.fold_worst = max(self.fold_worst, ((fb - 1.01 * U * y.abs()) / (g.double().abs() + TINY)).max().item())
        sc = g.double() / torch.sqrt(v.double() + eps)
        out, ea = act64(y, act)
        return out, pre_err * sc.abs() * (1 + 4 * U) + fb + ea

    def bn_act(self, x, y, scale, shift, G, R, C, act):
        assert G == 1
        torch.cuda.synchronize()
        xin = x.reshape(-1)[:R * C].clone().view(R, C)
        self._sync("bn_act", x, y, scale, shift, G, R, C, act)
        w = 0.0
        step = max(1, (1 << 24) // C)
        for r0 in range(0, R, step):
            ref, e = self._bn_ref(xin[r0:r0 + step], 0.0, scale, act)
            got = y.reshape(-1)[r0 * C:min(R, r0 + step) * C].view(-1, C)
            w = max(w, bound_check(got, ref, e + BETA[y.dtype] * ref.abs(), f"audit bn_act R={R} C={C} act={act}"))
        self._rec(f"bn_act R={R} C={C} act={act}", ("bn_act", act, str(y.dtype)[6:]), w)

    # ---- convolutions
    def conv_gemm(self, kind, a, b, c, N, H, W, Ck, Cn, Cm=0, ldb=None, ldc=None, bias=None, addend=None, grp_src=None,
                  imgs_per_group=0, accumulate=False, stat_partial=None, eval_scale=None, eval_shift=None, act=0):
        assert kind in (0, 2, 3) and H == W and not accumulate and stat_partial is None, f"unexpected conv_gemm kind {kind}"
        self._sync("conv_gemm", kind, a, b, c, N, H, W, Ck, Cn, Cm, ldb, ldc, bias, addend, grp_src, imgs_per_group, accumulate,
                   stat_partial, eval_scale, eval_shift, act)
        Ha, Ho = {0: (2 * H, H), 2: (H, 2 * H), 3: (H, H)}[kind]
        taps = 9 if kind == 3 else 16
        x = a.view(-1)[:N * Ha * Ha * Ck].view(N, Ha, Ha, Ck)
        wt = b.view(-1)[:taps * Ck * Cn].view(*((Cn, taps * Ck) if kind != 2 else (Ck, 16 * Cn)))
        out = c.view(-1)[:N * Ho * Ho * Cn].view(N, Ho, Ho, Cn)
        add, idx = self._addend(addend, grp_src, imgs_per_group, N, Ho, Cn) if addend is not None else (None, None)
        nm = f"conv_gemm kind {kind} N={N} {H}x{H} {Ck}->{Cn}" + (" eval" if eval_scale is not None else "")
        w = 0.0
        if eval_scale is None:
            chk = check_conv3_sums if kind == 3 else check_conv4_sums
            w = chk(out, kind, x, wt, N, H, Ck, Cn, bias, add, idx, name="audit " + nm)
        for i0 in _sample_images(N, imgs_per_group if addend is not None else 0):
            rows = add[idx[i0:i0 + 1]] if add is not None else None
            if kind == 3:
                pre, mag = conv3_ref64_elem(3, x[i0:i0 + 1], wt, H, Ck, Cn, bias, rows)
            else:
                pre, mag = conv4_ref64_elem(kind, x[i0:i0 + 1], wt, H, Ck, Cn, bias, rows)
            if eval_scale is None:
                w = max(w, assert_within(out[i0:i0 + 1], pre, mag, taps * Ck, out.dtype, quiet=True, name=f"audit {nm} image {i0}"))
            else:
                # act(scale (conv + bias + addend) + shift) against act(module BatchNorm(conv + bias + addend)): the
                # accumulation bound (alpha_for, as test_tc_schedule_gpu.py's eval epilogue) scaled by |scale|, plus the fold
                ref, e = self._bn_ref(pre, alpha_for(taps * Ck) * mag, eval_scale, act)
                w = max(w, bound_check(out[i0:i0 + 1], ref, e + BETA[out.dtype] * ref.abs(), f"audit {nm} image {i0}"))
        tiled = addend is not None and imgs_per_group < N
        self._rec(nm, ("conv_gemm", kind, eval_scale is not None, tiled), w)

    # ---- the explicit 4x4 lowering
    def im2col(self, x, col, N, H, W, C):
        self._sync("im2col", x, col, N, H, W, C)
        ref = im2col4_ref(x.reshape(-1)[:N * H * W * C].view(N, H, W, C))
        assert torch.equal(col.reshape(-1)[:ref.numel()].view(ref.shape), ref), f"audit im2col N={N} {H}x{W}x{C}"
        self._rec(f"im2col N={N} {H}x{W}x{C}", ("im2col", C), 0.0)

    def col2im(self, col, y, N, Hi, Wi, C, bias=None, col2=None, grp_src=None, imgs_per_group=0, accumulate=False):
        assert not accumulate
        self._sync("col2im", col, y, N, Hi, Wi, C, bias, col2, grp_src, imgs_per_group, accumulate)
        n = Hi * Wi * 16 * C
        ref, mag = col2im4_ref(col.reshape(-1)[:N * n], N, Hi, Wi, C, bias)
        if col2 is not None:
            # an image of col2 is Hi Wi 16 C elements, which _addend takes as a (4 Hi) x (4 Hi) x C map
            srcs, idx = self._addend(col2, grp_src, imgs_per_group, N, 4 * Hi, C)
            c2 = srcs.reshape(srcs.shape[0], n)[idx]
            r2, m2 = col2im4_ref(c2, N, Hi, Wi, C)
            ref, mag = ref + r2, mag + m2
        got = y.reshape(-1)[:ref.numel()].view(ref.shape)
        # up to 4 col taps, 4 col2 taps and the bias: 8 fp32 adds, then the stored dtype
        w = bound_check(got, ref, gamma(8) * mag + BETA[y.dtype] * ref.abs(), f"audit col2im N={N} {Hi}x{Wi}x{C}")
        self._rec(f"col2im N={N} {Hi}x{Wi}x{C}", ("col2im", C, col2 is not None), w)

    # ---- layouts, casts and the closing sigmoid
    def permute4(self, src, dst, dims, strides, accumulate=False):
        assert not accumulate
        self._sync("permute4", src, dst, dims, strides, accumulate)
        n = dims[0] * dims[1] * dims[2] * dims[3]
        ref = src.as_strided(tuple(dims), tuple(strides)).reshape(-1).to(dst.dtype)   # widening exact, narrowing to nearest even
        got = dst.reshape(-1)[:n]
        assert torch.equal(got.view(torch.int16 if got.dtype == torch.bfloat16 else torch.int32),
                           ref.view(torch.int16 if ref.dtype == torch.bfloat16 else torch.int32)), \
            f"audit permute4 {tuple(dims)} {src.dtype}->{dst.dtype}: not bit-exact"
        self._rec(f"permute4 {tuple(dims)}", ("permute4", str(src.dtype)[6:], str(dst.dtype)[6:]), 0.0)

    def gather_add(self, dst, src, grp_src, G, n):
        """VggAudit's check group by group: at 128x128 one group of the fp32 mode's skip sum is 1 GiB in float64."""
        torch.cuda.synchronize()
        d0 = dst.view(-1)[:G * n].clone()
        self._sync("gather_add", dst, src, grp_src, G, n)
        srcl = grp_src.tolist()
        self.skip_reads.append(srcl[:G])
        rel = 2.0 ** -7 if dst.dtype == torch.bfloat16 else 2.0 ** -23
        w = 0.0
        for g in range(G):
            ref = d0[g * n:(g + 1) * n].double() + src.view(-1)[srcl[g] * n:(srcl[g] + 1) * n].double()
            w = max(w, bound_check(dst.view(-1)[g * n:(g + 1) * n], ref, rel * ref.abs(), f"audit gather_add group {g}"))
        self._rec(f"gather_add G={G}", ("gather_add",), w)

    def transpose_batched(self, src, dst, A, P, Q):
        self._sync("transpose_batched", src, dst, A, P, Q)
        ref = src.reshape(-1)[:A * P * Q].view(A, P, Q).transpose(1, 2).to(dst.dtype)
        assert torch.equal(dst.reshape(-1)[:A * P * Q].view(A, Q, P), ref), f"audit transpose_batched {A}x{P}x{Q}: not bit-exact"
        self._rec(f"transpose_batched {A}x{P}x{Q}", ("transpose_batched", str(src.dtype)[6:], str(dst.dtype)[6:]), 0.0)

    def act_fwd(self, x, n, act):
        torch.cuda.synchronize()
        x0 = x.reshape(-1)[:n].clone()
        self._sync("act_fwd", x, n, act)
        ref, err = act_fwd_ref(x0, act)
        self._rec(f"act_fwd {act} n={n}", ("act_fwd", act), bound_check(x.reshape(-1)[:n], ref, err + TINY, f"audit act_fwd {act}"))

    # ---- vgg thin ends (bounds of test_vgg_generate_gpu.py)
    def vgg_first_eval(self, x, nc, w, bias, scale, shift, y, N, H, W):
        self._sync("vgg_first_eval", x, nc, w, bias, scale, shift, y, N, H, W)
        F = torch.nn.functional
        wd = 0
        for i in _sample_images(N, 0):
            xi = x.reshape(-1)[i * nc * H * W:(i + 1) * nc * H * W].view(1, nc, H, W).double()
            pre = F.conv2d(xi, w.double(), bias.double(), padding=1)
            mag = F.conv2d(xi.abs(), w.double().abs(), bias.double().abs(), padding=1)
            ref, _ = act64(pre * scale.double()[:, None, None] + shift.double()[:, None, None], ACT_LRELU)
            mag = mag * scale.double().abs()[:, None, None] + shift.double().abs()[:, None, None]
            got = y.reshape(-1)[i * H * W * 64:(i + 1) * H * W * 64].view(1, H, W, 64).permute(0, 3, 1, 2)
            # 28 fp32 FFMA and the epilogue, then the stored dtype
            wd = max(wd, bound_check(got, ref, 30 * U * mag + BETA[y.dtype] * ref.abs() * (y.dtype == torch.bfloat16), "audit vgg_first_eval"))
        self._rec(f"vgg_first_eval N={N} nc={nc}", ("vgg_first_eval", nc), wd)

    def vgg_last_eval(self, d, w, bias, out, nc, N, H, W):
        self._sync("vgg_last_eval", d, w, bias, out, nc, N, H, W)
        F = torch.nn.functional
        wd = 0
        for i in _sample_images(N, 0):
            di = d.reshape(-1)[i * H * W * 64:(i + 1) * H * W * 64].view(1, H, W, 64).permute(0, 3, 1, 2).double()
            pre = F.conv_transpose2d(di, w.double(), bias.double(), padding=1)
            mag = F.conv_transpose2d(di.abs(), w.double().abs(), bias.double().abs(), padding=1)
            got = out.reshape(-1)[i * nc * H * W:(i + 1) * nc * H * W].view(1, nc, H, W)
            # sigmoid' <= 1/4: an fp32 accumulation of 577 terms, then expf
            wd = max(wd, bound_check(got, torch.sigmoid(pre), 0.25 * 600 * U * mag + 1e-6, "audit vgg_last_eval"))
        self._rec(f"vgg_last_eval N={N} nc={nc}", ("vgg_last_eval", nc), wd)

    # ---- the recurrent step
    def lstm_step(self, modules, rows, R):
        torch.cuda.synchronize()
        names = _ptr_map(self.model)
        pre = []
        for md in modules:
            m = names[md["w_embed"].data_ptr()]
            hs, cs = self.bufs[f"{m}_h"], self.bufs[f"{m}_c"]
            out = md["out"]
            base = out._base if out._base is not None else out
            pre.append((m, hs.clone(), cs.clone(), base, base.clone()))
        self._sync("lstm_step", modules, rows, R)
        w = 0.0
        written = {}
        for md, (m, h0, c0, base, base0) in zip(modules, pre):
            mod = getattr(self.model, m)
            L = md["layers"]
            hs, cs = self.bufs[f"{m}_h"], self.bufs[f"{m}_c"]
            # the device pointer table names this module's weights and the graph's state rows
            want = [t.data_ptr() for cell in mod.lstm for t in (cell.weight_ih, cell.bias_ih, cell.weight_hh, cell.bias_hh)]
            want += [t.data_ptr() for l in range(L) for t in (hs[l], cs[l], hs[l], cs[l])]
            assert md["layer_w"].tolist() + md["state"].tolist() == want, f"audit lstm_step {m}: pointer table"
            X = lstm_input64(md["seg_a"], int(md["idx_a"][0]), md["ga"], md["seg_b"], int(md["idx_b"][0]), md["gb"], md["tuc"],
                             md["dt"], md["counter_rows"], rows)
            xin, xe = embed64(X, mod.embed.weight, mod.embed.bias)
            for l in range(L):
                cell = mod.lstm[l]
                h, c, eh, ec = lstm_cell64(xin, xe, h0[l, :rows], c0[l, :rows], cell.weight_ih, cell.bias_ih, cell.weight_hh, cell.bias_hh)
                w = max(w, bound_check(cs[l, :rows], c, ec, f"audit lstm_step {m} layer {l} c"),
                        bound_check(hs[l, :rows], h, eh, f"audit lstm_step {m} layer {l} h"))
                # the next layer reads this layer's stored h: exact from here on
                xin, xe = hs[l, :rows].double(), None
            assert torch.equal(hs[:, rows:], h0[:, rows:]) and torch.equal(cs[:, rows:], c0[:, rows:]), \
                f"audit lstm_step {m}: state rows past the active {rows} written"
            out = md["out"]
            got = out.reshape(-1)[:rows * md["out_dim"]].view(rows, md["out_dim"])
            if md["head"] == 1:
                ref, e = head_gauss64(xin, mod.mu_net.weight, mod.mu_net.bias, mod.logvar_net.weight, mod.logvar_net.bias,
                                      md["eps"].reshape(-1)[:rows * md["out_dim"]].view(rows, md["out_dim"]))
            else:
                ref, e = head_tanh64(xin, mod.output[0].weight, mod.output[0].bias)
            w = max(w, bound_check(got, ref, e, f"audit lstm_step {m} head"))
            o0 = out.storage_offset() - base.storage_offset()
            written.setdefault(base.data_ptr(), (base, base0, []))[2].append((o0, o0 + rows * md["out_dim"]))
        for base, base0, spans in written.values():
            keep = torch.ones(base.numel(), dtype=torch.bool, device=base.device)
            for s0, s1 in spans:
                keep[s0:s1] = False
            assert torch.equal(base.reshape(-1)[keep], base0.reshape(-1)[keep]), "audit lstm_step: output rows past the active rows written"
        cr = modules[0]["counter_rows"]
        self._rec(f"lstm_step rows={rows} R={R} x{len(modules)}", ("lstm_step", len(modules)), w)
        for v in (("lstm_step", "counter_rows", cr > 0), ("lstm_step", "layers", max(md["layers"] for md in modules))):
            self.seen.add(v)
        if rows % 8:
            self.seen.add(("lstm_step", "partial_slab"))

    def pose_mlp(self, mod, decoder, src, out, rows, src_idx=None, skips=None, nsrc=0, h1=None, h2=None):
        torch.cuda.synchronize()
        o0 = out.clone()
        s0 = [t.clone() if t is not None else None for t in (h1, h2)]
        self._sync("pose_mlp", mod, decoder, src, out, rows, src_idx, skips, nsrc, h1, h2)
        g = mod.fc1.norm.normalized_shape[0]
        ind = int(src_idx[0]) if src_idx is not None else 0
        w = 0.0
        nout = POSE if decoder else g
        if decoder:
            vec = src.reshape(-1)[ind * rows * g:(ind + 1) * rows * g].view(rows, g)
            ref, e = pose_decoder64(mod, vec, skips[0].reshape(-1, g), skips[1].reshape(-1, g), nsrc)
            w = bound_check(out.reshape(-1)[:rows * POSE].view(rows, POSE), ref, e, "audit pose_mlp decoder")
        else:
            x = src.reshape(-1)[ind * rows * POSE:(ind + 1) * rows * POSE].view(rows, POSE).double()
            ref, e = pose_encoder64(mod, x)
            w = bound_check(h1.reshape(-1)[:rows * g].view(rows, g), ref, e, "audit pose_mlp encoder h1")
            ref, e = residual64(residual_params(mod.fc2), h1.reshape(-1)[:rows * g].view(rows, g).double(), None)
            w = max(w, bound_check(h2.reshape(-1)[:rows * g].view(rows, g), ref, e, "audit pose_mlp encoder h2"))
            ref, e = pose_encoder_top64(mod, h2.reshape(-1)[:rows * g].view(rows, g))
            w = max(w, bound_check(out.reshape(-1)[:rows * g].view(rows, g), ref, e, "audit pose_mlp encoder out"))
            for t, t0 in zip((h1, h2), s0):
                assert torch.equal(t.reshape(-1)[rows * g:], t0.reshape(-1)[rows * g:]), "audit pose_mlp: skip rows past `rows` written"
        assert torch.equal(out.reshape(-1)[rows * nout:], o0.reshape(-1)[rows * nout:]), "audit pose_mlp: rows past `rows` written"
        self._rec(f"pose_mlp {'decoder' if decoder else 'encoder'} rows={rows}", ("pose_mlp", "decoder" if decoder else "encoder"), w)
        if decoder and nsrc < rows:
            self.seen.add(("pose_mlp", "decoder", "tiled"))
        if rows % 8:
            self.seen.add(("pose_mlp", "partial_slab"))


# ------------------------------------------------------------------ one audited call

class _EagerBody:
    """Stands in for a captured graph for one call: replay() runs the engine's body eagerly on the audit view."""

    def __init__(self, eng, G, audit):
        self.eng, self.G, self.audit = eng, G, audit

    def replay(self):
        from p2pvg_b200 import infer
        torch.cuda.synchronize()
        prev, kept = infer.kernels_for, (getattr(self.eng, "K", None), getattr(self.eng, "G", None))
        infer.kernels_for = lambda dev: self.audit   # only while the body runs: _run compares ws_gen outside it
        try:
            self.eng._body(self.G)
        finally:
            infer.kernels_for = prev
            self.eng.K, self.eng.G = kept   # the engine must not keep the audit view (or what it holds) past the call
        torch.cuda.synchronize()


def _state(model):
    return {m: [(h.clone(), c.clone()) for h, c in getattr(model, m).hidden] for m in ("posterior", "prior", "frame_predictor")}


def _flat(res):
    if torch.is_tensor(res):
        return [res]
    out = []
    for r in res:
        out += _flat(r)
    return out


@contextlib.contextmanager
def _seeded(np_seed, torch_seed):
    import numpy as np
    np.random.seed(np_seed)
    torch.manual_seed(torch_seed)
    yield


def audited_call(model, call, audit, seed=0):
    """call(model) three times with the same NumPy and torch seeds: a plain first call (captures the graph of its
    signature), the same call with its replay replaced by the body run eagerly on `audit`, and a plain replay.  The audited
    call's returned frames, .hidden and the graph's output buffer must equal the plain replay's bit for bit.  Returns the
    audited call's result."""
    eng = model._graphed_engine()
    with _seeded(seed, seed):
        call(model)
    torch.cuda.synchronize()
    assert len(eng._graphs) >= 1
    G = next(reversed(eng._graphs.values()))
    n_graphs = len(eng._graphs)
    graph = G.graph
    audit.model, audit.bufs = model, G.bufs
    G.graph = _EagerBody(eng, G, audit)
    try:
        with _seeded(seed, seed):
            got = [t.clone() for t in _flat(call(model))]
        got_state, got_out = _state(model), G.bufs["out"].clone()
    finally:
        G.graph = graph
        audit.bufs = None   # the audit outlives the call: it must not keep the graph's buffers alive
    assert len(eng._graphs) == n_graphs and next(reversed(eng._graphs.values())) is G, "the audited call did not reuse the graph"
    assert audit.log, "the audited body launched nothing"
    with _seeded(seed, seed):
        ref = [t.clone() for t in _flat(call(model))]
    assert len(got) == len(ref)
    for i, (a, b) in enumerate(zip(got, ref)):
        assert torch.equal(a, b), f"returned tensor {i}: the audited eager body differs from the graph replay"
    assert torch.equal(got_out, G.bufs["out"]), "the output buffer of the audited body differs from the graph replay"
    for m, hc in _state(model).items():
        for l, ((h1, c1), (h2, c2)) in enumerate(zip(got_state[m], hc)):
            assert torch.equal(h1, h2) and torch.equal(c1, c2), f"{m}.hidden layer {l}: the audited body differs from the replay"
    return got
