"""The CUDA-core kernels between the big GEMMs and the LSTM scans -- losses, latent assembly, bias sums, weight packing and
Adam -- mirrored on the host: the arguments each receives in one benchmark step, the launch decisions it makes, float64
references of what it computes, and a per-element bound |got - ref| <= bound with its sources (tests/test_loss_optim_gpu.py,
tests/test_loss_ref_cpu.py).

Every reference is computed on the kernel's own (bf16 or fp32) inputs.  Where a kernel consumes an earlier output of its own
(Adam's new moments, LayerNorm's row statistics) the reference is teacher-forced from that output, so each bound covers one
kernel step.  Bound terms:
  U = 2^-24        one fp32 rounding (IEEE / and sqrtf are correctly rounded: the build has no fast-math), and a double
                   partial stored as fp32
  ULP = 2^-23      CUDA Math API maximum errors are quoted in ulp: expf 2, tanhf 2, rsqrtf 2, logf 1
  gamma(n)         Higham's bound for a chain of n fp32 roundings, relative to the sum of the magnitudes involved
  BF16_HALF = 2^-8 half a bf16 ulp, relative, for every bf16 store (8 significant bits)
"""
import math

import numpy as np
import torch

from tests.lstm_schedule import ULP, U, gamma, sigmoid_err, tanh_err

TINY = 2.0 ** -126
BF16_HALF = 2.0 ** -8
MSE_CHUNKS, MSE_BLOCK = 32, 256        # loss_adam.cu:6 MSE_CHUNKS; :171 / :181 grid (MSE_CHUNKS, G) x 256 threads
GRID_CAP = 132 * 16                    # lstm.cu:250-254 grid_for, loss_adam.cu:220 (Adam)
LOWER_GRID_CAP = 132 * 64              # conv_lower.cu:325-329 grid_for (blockdiag)
RKL_CTAS, RKL_THREADS = 8, 1024        # lstm.cu:46 / :271: one cluster of 8 CTAs of 1024 threads
ALIGN_CW, ALIGN_RL = 128, 8            # lstm.cu:159: 128-column passes x 8 row lanes
COLSUM_FOLD = 256                      # lstm.cu:315
LN_ROW_CHUNK, LN_MAX_CHUNKS = 256, 256  # mlp.cu:143-144
LRELU_SLOPE = float(np.float32(0.2))   # lstm.cu:234 0.2f


def cdiv(a, b):
    return (a + b - 1) // b


# ------------------------------------------------------------------ launch shapes of one benchmark step

def arena_numel(cfg):
    """Per-module Adam n (ParamArena.numel: every view padded to 4 floats, engine.py:98-103) and the pooled arena
    (engine.py:164).  Shapes only: the containers are built on the meta device."""
    from oracle import p2p_oracle as O
    from p2pvg_b200.engine import ARENA_ORDER, ParamArena, is_param_key
    g, z, r = cfg["g_dim"], cfg["z_dim"], cfg["rnn_size"]
    with torch.device("meta"):                       # oracle/p2p_oracle.py:264-279 without the initialisation
        mods = dict(frame_predictor=O._lstm_container(g + z + 2, g, r, cfg["predictor_rnn_layers"], gaussian=False),
                    posterior=O._lstm_container(2 * g + 2, z, r, cfg["posterior_rnn_layers"], gaussian=True),
                    prior=O._lstm_container(2 * g + 2, z, r, cfg["prior_rnn_layers"], gaussian=True))
        if cfg.get("backbone") == "mlp":
            mods.update(encoder=O._mlp_encoder_container(51, g, g), decoder=O._mlp_decoder_container(g, 51, g))
        elif cfg.get("backbone") == "vgg":
            mods.update(encoder=O._vgg_encoder_container(g, cfg["channels"], 64), decoder=O._vgg_decoder_container(g, cfg["channels"], 64))
        else:
            mods.update(encoder=O._dcgan_encoder_container(g, cfg["channels"], cfg["image_width"]),
                        decoder=O._dcgan_decoder_container(g, cfg["channels"], cfg["image_width"]))
    params = {m: {k: v for k, v in mods[m].state_dict().items() if is_param_key(k)} for m in ARENA_ORDER}
    per = {m: sum((v.numel() + 3) // 4 * 4 for v in params[m].values()) for m in ARENA_ORDER}
    return per, sum(ParamArena.padded(params[m]) for m in ARENA_ORDER)


def bench_shapes(name, bf16=True, with_arena=False):
    """What the entry points receive in one step of bench.py --config <name> (skip_prob 0, one GPU, weak scaling), derived
    from bench.CONFIGS and the engine's own plan; bf16=False is the engine's fp32 mode."""
    import bench
    from p2pvg_b200.engine import StepPlan
    c = bench.CONFIGS[name]
    T, B, R, g, z = c["T"], c["per_gpu"], c["rnn"], bench.G_DIM, bench.Z_DIM
    plan = StepPlan(T, np.zeros(T - 1), dict(skip_prob=0.0, n_past=1, last_frame_skip=False))
    S = plan.S
    G = S + 1                                            # S recon decodes + the CPC decode (engine.py:818, :892)
    bb = {"dcgan_64": "dcgan", "dcgan_128": "dcgan", "vgg_64": "vgg", "h36m_mlp": "mlp"}[c["backbone"]]
    nc, W = (c["channels"], c["width"]) if bb != "mlp" else (None, None)
    frame = 51 if bb == "mlp" else nc * W * W            # engine.py:159-161
    sh = dict(name=name, backbone=bb, T=T, B=B, S=S, G=G, R=R, g=g, z=z, nc=nc, W=W, E=B * frame, has_cpc=plan.has_cpc,
              in_idx=plan.int_host[slice(*_span(plan, "in_idx"))].tolist(), bf16=bf16)
    # the reconstruction loss (engine.py:893-903, engine_vgg.py, engine_mlp.py:180-183)
    if bb == "mlp":
        sh["loss"] = "mse_plain"
    elif bb == "dcgan" and bf16:                          # fused last layer: engine.py:199, :869, :900
        sh["loss"] = "convt_c1_loss"
        sh["Hi"], sh["C"] = W // 2, nc
    else:
        sh["loss"] = "sigmoid_mse"
    sh["finalize"] = dict(n_recon=S, has_cpc=plan.has_cpc, E=B * frame, batch_size=B, n_align=max(S - 1, 0), seq_len=T)  # engine.py:1116
    sh["align"] = dict(P=S - 1, B=B, g=g, coef=0.5)      # engine.py:1111, weight_align (oracle default_opt)
    sh["reparam_n"] = S * B * z                           # engine.py:794-802, :1140-1143
    sh["concat"] = [(S, 2 * g + 2), (S + 1, g + z + 2)]   # engine.py:772-773 (S, width) / :807
    sh["gather"] = [(S, 2 * g + 2, 0), (S, 2 * g + 2, g), (S, g + z + 2, 0)]   # engine.py:1153-1157 (S, W, col0) into dH[T, B, g]
    # every colsum of the step: (where, rows, cols, bf16 input)
    cs = []
    if bb in ("dcgan", "vgg"):                            # last decoder layer bias, recon calls only: engine.py:935, engine_vgg.py:268
        cs.append(("decoder last bias", S * B * W * W, nc, bf16))
    rows = S * B
    cs += [("lstm bias", rows, 4 * R, False), ("embed bias", rows, R, False), ("mu/logvar bias", rows, z, False),
           ("output bias", rows, g, False)]               # engine.py:1071-1072, :1081, :1099-1100, :1132
    if bb == "mlp":                                       # engine_mlp.py:52, :223, :257
        cs += [("mlp fc3 bias", rows, 51, False), ("mlp decoder bias", rows, g, False), ("mlp encoder bias", T * B, g, False)]
    sh["colsum"] = cs
    if bb == "mlp":                                       # engine_mlp.py:83 (forward rows), :94 / :232 (backward rows), width h_dim = g
        sh["layernorm"] = dict(C=g, rows_fwd=[T * B, G * B], rows_bwd=[T * B, S * B, B])
    sh["transpose"] = transpose_calls(bb, nc, W, g, z, R, bf16)
    sh["blockdiag"] = blockdiag_calls(bb, nc, W) if bf16 else []
    if with_arena:
        cfg, _ = bench.oracle_cfg(c)
        sh["adam_numel"], sh["arena_numel"] = arena_numel(cfg)
    return sh


def _span(plan, key):
    off, n = plan.int_layout[key]
    return off, off + n


def dcgan_chans(W):
    return [64, 128, 256, 512] if W == 64 else [64, 128, 256, 512, 512]   # engine.py:155


def transpose_calls(bb, nc, W, g, z, R, bf16):
    """(A, P, Q, src bf16, dst bf16) of every transpose_batched call of a step and of the weight packing."""
    calls = []
    if bb == "dcgan":
        ch = dcgan_chans(W)
        n = len(ch)
        for l in range(n + 1):                           # encoder packing [co][ci][tap] -> [co][tap][ci]: engine.py:315
            co, ci = (ch[l], nc if l == 0 else ch[l - 1]) if l < n else (g, ch[-1])
            calls.append((co, ci, 16, False, bf16))
            calls.append((co, 16, ci, False, False))     # its weight gradient back: engine.py:1179, :1199, :1207
        for k in range(-1, n):                           # decoder packing [ci][co][tap] -> [ci][tap][co]: engine.py:330
            ci, co = (g, ch[-1]) if k < 0 else (2 * ch[n - 1 - k], ch[n - 2 - k] if k < n - 1 else nc)
            calls.append((ci, co, 16, False, bf16))
            calls.append((ci, 16, co, False, False))     # engine.py:958, :999, :1014
    if bb == "vgg":
        calls.append((g, 16, 512, False, False))         # engine_vgg.py:353
    if bf16:                                             # K-major LSTM weights, tensor-core mode: engine.py:361-365
        for in_dim, heads in ((g + z + 2, [(g, R)]), (2 * g + 2, [])):
            for o, i in [(R, in_dim), (4 * R, R)] + heads:
                calls.append((1, o, i, False, False))
    return sorted(set(calls))


def blockdiag_calls(bb, nc, W):
    """(R, C, g) of the block-diagonal copies of the 1/3-channel ends (engine.py:317-319, :332-336), bf16 -> bf16."""
    if bb != "dcgan" or (16 * nc) % 64 == 0:
        return []
    ch0 = dcgan_chans(W)[0]
    return [(ch0, 16 * nc, 4)]


# ------------------------------------------------------------------ host-side launch decisions

def colsum_plan(rows, cols, ld, ws_floats):
    """lstm.cu:310-337: the levels p2pvg_colsum launches, each dict(rows, cols, nchunk, rpc, fold).  The fold path (cols <= 4,
    contiguous, rows >= 64*256 and a multiple of 256) sums 256-row blocks as rows of 256*cols columns, then the 256 folded
    columns per original column."""
    F = COLSUM_FOLD
    if cols <= 4 and ld == cols and rows >= 64 * F and rows % F == 0 and ws_floats >= 1025 * F * cols:
        inner = 1024 * F * cols
        return [dict(l, fold=True) for l in colsum_plan(rows // F, F * cols, F * cols, inner) + colsum_plan(F, cols, cols, inner)]
    want = (132 * 8) // cdiv(cols, 32) + 1
    nchunk = max(1, min(want, (rows + 63) // 64, 1024))
    assert ws_floats >= nchunk * cols, "colsum: workspace too small"
    rpc = max(1, cdiv(rows, nchunk))
    nchunk = cdiv(rows, rpc) if rows > 0 else 1
    return [dict(rows=rows, cols=cols, nchunk=nchunk, rpc=rpc, fold=False)]


def colsum_chain(plan, accumulate):
    """Longest fp32 chain of one output: per level, a row lane's ceil(rpc/8) adds, the 8 lanes, the nchunk partials; the
    accumulate add."""
    return sum(cdiv(l["rpc"], 8) + 8 + l["nchunk"] for l in plan) + int(bool(accumulate))


def ln_bwd_chunks(rows):
    """mlp.cu:143-147: (nchunk, rows per chunk) of the dgamma / dbeta partials."""
    nchunk = max(1, min(cdiv(rows, LN_ROW_CHUNK), LN_MAX_CHUNKS))
    rpc = cdiv(rows, nchunk)
    return cdiv(rows, rpc), rpc


def grid_for(total, cap=GRID_CAP):
    return max(1, min(cdiv(total, 256), cap))


# ------------------------------------------------------------------ the check

def assert_bound(name, got, ref, bound, where=None, worst=None):
    """|got - ref| <= bound elementwise (flattened).  NaN or Inf in got fails.  On failure: the worst element, described by
    where(flat index) (group, chunk, index ...).  Returns the worst error/bound (folded into worst[name])."""
    got, ref, bound = got.reshape(-1), ref.reshape(-1).double(), bound.reshape(-1).double()
    assert got.numel() == ref.numel(), f"{name}: {got.numel()} values, reference has {ref.numel()}"
    diff = (got.double() - ref).abs()
    ratio = torch.where(bound > 0, diff / bound.clamp_min(1e-300), torch.where(diff > 0, torch.inf, 0.0))
    ratio = torch.nan_to_num(ratio, nan=torch.inf)
    w = ratio.max().item() if ratio.numel() else 0.0
    if w > 1.0:
        i = int(ratio.argmax())
        bad = int((ratio > 1.0).sum())
        at = where(i) if where else f"index {i}"
        raise AssertionError(f"{name}: {bad}/{ratio.numel()} elements out of bound, worst ratio {w:.3g} at {at}: got "
                             f"{got[i].item():.9g}, ref {ref[i].item():.9g}, bound {bound[i].item():.3g}")
    if worst is not None:
        worst[name] = max(worst.get(name, 0.0), w)
    return w


def report(worst, title=""):
    for k, v in sorted(worst.items()):
        print(f"[bound]{' ' + title if title else ''} {k}: worst error/bound {v:.3g}")


def store_bound(ref, bound, bf16):
    """Add the bf16 store's rounding (half an ulp of the fp32 value) when the output is bf16."""
    return bound + BF16_HALF * (ref.abs() + bound) + TINY if bf16 else bound


def _where_mse(g, per=1):
    return lambda i: f"group {g}, chunk {(i // per // MSE_BLOCK) % MSE_CHUNKS}, index {i}"


def chunk_sums(v, per=1):
    """Sum v[0..E) by the chunk that owns each element: the grid-stride loop of a (MSE_CHUNKS x 256)-thread row hands element
    (pixel, for per = C channels) e to chunk (e // 256) % 32."""
    idx = (torch.arange(v.numel(), device=v.device) // per // MSE_BLOCK) % MSE_CHUNKS
    return torch.zeros(MSE_CHUNKS, dtype=torch.float64, device=v.device).index_add_(0, idx, v.double())


def check_partials(name, partial, ref_sq, bound_sq, G, per=1, per_chunk=True, worst=None):
    """partial [G, 32] fp32 against the chunked float64 sums of d^2.  Each chunk is the kernel's double sum of its (fp32 d)^2,
    stored as fp32 (2^-24); per_chunk=False compares only the group totals, the quantity finalize_losses uses."""
    p = partial.reshape(-1)[:G * MSE_CHUNKS].reshape(G, MSE_CHUNKS)
    for g in range(G):
        r, b = chunk_sums(ref_sq[g], per), chunk_sums(bound_sq[g], per)
        b = b + U * r + 2.0 ** -30 * r + 2.0 ** -149     # the store, and the double sum of <= 2^23 terms
        if per_chunk:
            assert_bound(name, p[g], r, b, lambda k, g=g: f"group {g}, chunk {k}", worst)
        assert_bound(name + " (group sum)", p[g].double().sum(), r.sum(), b.sum() + U * r.sum(), lambda k, g=g: f"group {g}", worst)


# ------------------------------------------------------------------ losses

def sigmoid_loss_terms(z, dz, xt, cf):
    """Reference terms of sigmoid + squared error at exact argument z whose kernel value is within dz (float64 tensors).
    s = 1/(1+expf(-v)) (common.cuh:115): its own error sigmoid_err plus the argument error moved by sigma'(z) e^dz dz.
    d = s - x (one rounding); d_raw = cf*2*d*s*(1-s): four roundings (gamma 4) and the propagation of es through
    d s (1-s), whose derivative in s is s(1-s) + d(1-2s)."""
    s = torch.sigmoid(z)
    es = s * (1 - s) * torch.exp(dz) * dz + sigmoid_err(z, dz, False)
    d = s - xt
    ed = es + U * (d.abs() + es)
    q = d * s * (1 - s)
    eq = ed * (s * (1 - s) + es * (1 + es)) + d.abs() * es * ((1 - 2 * s).abs() + es)
    two_cf = 2 * abs(cf)
    dref = 2 * cf * q
    dbound = two_cf * (eq + gamma(4) * (q.abs() + eq)) + TINY
    sq = d * d
    sq_bound = 2 * d.abs() * ed + ed * ed
    return s, es, dref, dbound, sq, sq_bound


def check_sigmoid_mse(raw, x, tgt, coef, G, E, pred, d_raw, partial, per_chunk=True, worst=None, tag="sigmoid_mse"):
    """p2pvg_sigmoid_mse (loss_adam.cu:10-36): pred = sigmoid(raw), d_raw = coef 2 (s - x) s (1 - s), partial = chunked sum of
    (s - x)^2, for every group g against frame tgt[g] of x [*, E] (fp32)."""
    bf16 = raw.dtype == torch.bfloat16
    xs = x.reshape(-1, E)
    sq_all, sqb_all = [], []
    for g in range(G):
        zz = raw.reshape(-1)[g * E:(g + 1) * E].double()
        cf = float(coef[g])
        s, es, dref, dbound, sq, sqb = sigmoid_loss_terms(zz, torch.zeros_like(zz), xs[int(tgt[g])].double(), cf)
        if pred is not None:
            assert_bound(tag + " pred", pred.reshape(-1)[g * E:(g + 1) * E], s, store_bound(s, es, bf16), _where_mse(g), worst)
        if d_raw is not None:
            assert_bound(tag + " d_raw", d_raw.reshape(-1)[g * E:(g + 1) * E], dref, store_bound(dref, dbound, bf16), _where_mse(g), worst)
        sq_all.append(sq)
        sqb_all.append(sqb)
    check_partials(tag + " partial", partial, sq_all, sqb_all, G, 1, per_chunk, worst)


def convt_taps(col, B, Hi, Wi, C):
    """Sum of the transposed-convolution taps (k4 s2 p1) landing on each output pixel, written as a gather: output row
    2m + py takes kernel rows kh with input row iy = (2m + py + 1 - kh) / 2, i.e. py = 0: (kh 1, iy m), (kh 3, iy m - 1);
    py = 1: (kh 0, iy m + 1), (kh 2, iy m); columns alike.  col [B, Hi, Wi, 4, 4, C] float64 -> [B, 2Hi, 2Wi, C]."""
    taps = {0: ((1, 0), (3, -1)), 1: ((0, 1), (2, 0))}
    pad = torch.nn.functional.pad(col, (0, 0, 0, 0, 0, 0, 1, 1, 1, 1))          # zero input rows / columns -1 and Hi, Wi
    out = torch.zeros(B, Hi, 2, Wi, 2, C, dtype=col.dtype, device=col.device)
    for py in (0, 1):
        for px in (0, 1):
            for kh, dy in taps[py]:
                for kw, dx in taps[px]:
                    out[:, :, py, :, px] += pad[:, 1 + dy:1 + dy + Hi, 1 + dx:1 + dx + Wi, kh, kw]
    return out.reshape(B, 2 * Hi, 2 * Wi, C)


def check_convt_c1_loss(col, col2, grp_src, bias, x, tgt, coef, G, B, Hi, Wi, C, d_raw, partial, per_chunk=True, worst=None):
    """p2pvg_convt_c1_loss (loss_adam.cu:43-96): raw = bias + the taps of col (group g) and col2 (skip source grp_src[g]),
    then sigmoid + squared error against frame tgt[g].  The kernel adds each tap as v += (a + b): two roundings per tap, at
    most four taps: gamma(8) of |bias| + sum |a| + |b|."""
    bf16 = col.dtype == torch.bfloat16
    n_in = B * Hi * Wi * 16 * C
    E = B * 4 * Hi * Wi * C
    xs = x.reshape(-1, E)
    b = (bias.double() if bias is not None else torch.zeros(C, dtype=torch.float64, device=col.device)).reshape(C)
    sq_all, sqb_all = [], []
    for g in range(G):
        a = col.reshape(-1)[g * n_in:(g + 1) * n_in].double().reshape(B, Hi, Wi, 4, 4, C)
        sg = int(grp_src[g])
        s2 = col2.reshape(-1)[sg * n_in:(sg + 1) * n_in].double().reshape(B, Hi, Wi, 4, 4, C)
        z = (convt_taps(a + s2, B, Hi, Wi, C) + b).reshape(-1)
        mag = (convt_taps(a.abs() + s2.abs(), B, Hi, Wi, C) + b.abs()).reshape(-1)
        del a, s2
        _, _, dref, dbound, sq, sqb = sigmoid_loss_terms(z, gamma(8) * mag, xs[int(tgt[g])].double(), float(coef[g]))
        assert_bound("convt_c1_loss d_raw", d_raw.reshape(-1)[g * E:(g + 1) * E], dref, store_bound(dref, dbound, bf16),
                     _where_mse(g, C), worst)
        sq_all.append(sq)
        sqb_all.append(sqb)
    check_partials("convt_c1_loss partial", partial, sq_all, sqb_all, G, C, per_chunk, worst)


def check_mse_plain(pred, x, tgt, coef, G, E, d_pred, partial, per_chunk=True, worst=None):
    """p2pvg_mse_plain (mlp.cu:104-126): d = pred - x (one rounding), d_pred = coef 2 d (one more), chunked sum of d^2."""
    xs = x.reshape(-1, E)
    sq_all, sqb_all = [], []
    for g in range(G):
        d = pred.reshape(-1)[g * E:(g + 1) * E].double() - xs[int(tgt[g])].double()
        cf = float(coef[g])
        ed = U * d.abs()
        if d_pred is not None:
            assert_bound("mse_plain d_pred", d_pred.reshape(-1)[g * E:(g + 1) * E], 2 * cf * d, 2 * abs(cf) * gamma(2) * d.abs() + TINY,
                         _where_mse(g), worst)
        sq_all.append(d * d)
        sqb_all.append(2 * d.abs() * ed + ed * ed)
    check_partials("mse_plain partial", partial, sq_all, sqb_all, G, 1, per_chunk, worst)


def finalize_ref(mse_partial, n_recon, has_cpc, E, kl_sum, batch_size, align_partial, n_align, seq_len):
    """p2pvg_finalize_losses (loss_adam.cu:98-123): [mse, kld, cpc, align] from the partials, in float64; each is a double
    quotient stored as fp32 (2^-24 relative, plus the double sums' own 2^-45)."""
    p = mse_partial.reshape(-1).double()
    k = MSE_CHUNKS
    mse = p[:n_recon * k].sum().item()
    cpc = p[n_recon * k:(n_recon + 1) * k].sum().item() if has_cpc else 0.0
    al = align_partial.reshape(-1)[:n_align].double().sum().item() if n_align > 0 else 0.0
    bs, sl = float(np.float32(batch_size)), float(np.float32(seq_len))
    ref = torch.tensor([mse / E / sl, float(kl_sum.reshape(-1)[0]) / bs / sl, cpc / E / sl, al / sl], dtype=torch.float64)
    return ref, (U + 2.0 ** -45) * ref.abs() + 2.0 ** -149


def check_finalize(out, *args, worst=None):
    ref, bound = finalize_ref(*args)
    names = ["mse", "kld", "cpc", "align"]
    assert_bound("finalize_losses", out.reshape(-1)[:4].cpu(), ref, bound, lambda i: f"out[{i}] ({names[i]})", worst)


# ------------------------------------------------------------------ recurrent-phase glue

def _rkl_where(i):
    return f"index {i} (CTA {(i // RKL_THREADS) % RKL_CTAS}, thread {i % RKL_THREADS})"


def check_reparam_kl_fwd(mu, lv, mu_p, lv_p, eps, eps_p, z, z_p, n, kl_sum, worst=None):
    """lstm.cu:47-88.  z = eps expf(lv/2) + mu: expf 2 ulp, then a product and an add (gamma 2).  KL term
    k = logf(s2/s1) + (expf(l1) + d^2) / (2 expf(l2)) - 1/2 with s = expf(l/2): the ratio carries 4 ulp of the two expf and
    one division, logf adds 1 ulp of its result; Q = (e1 + d^2)/(2 e2) carries 2 + 2 ulp of its expf and gamma(4) of d, d*d,
    the add and the division; the two outer adds gamma(2) of their magnitudes.  kl_sum: double sum of the fp32 terms over the
    8 CTAs, stored as fp32."""
    m1, l1, m2, l2, e, ep = (t.reshape(-1)[:n].double() for t in (mu, lv, mu_p, lv_p, eps, eps_p))
    for out, ee, m, l, nm in ((z, e, m1, l1, "z"), (z_p, ep, m2, l2, "z_p")):
        s = torch.exp(0.5 * l)
        ref = ee * s + m
        assert_bound(f"reparam_kl_fwd {nm}", out.reshape(-1)[:n], ref, (ee * s).abs() * 2 * ULP * (1 + gamma(2)) + gamma(2) * ((ee * s).abs() + m.abs()) + TINY,
                     _rkl_where, worst)
    d = m1 - m2
    L = 0.5 * (l2 - l1)
    Q = (torch.exp(l1) + d * d) / (2 * torch.exp(l2))
    k = L + Q - 0.5
    kb = (4 * ULP + 2 * U) * (1 + ULP) + ULP * L.abs() + Q.abs() * (4 * ULP + gamma(4)) * 1.01 + gamma(2) * (L.abs() + Q.abs() + 0.5) + TINY
    ref = k.sum()
    bound = kb.sum() + U * ref.abs() + 2.0 ** -30 * k.abs().sum() + 2.0 ** -149
    assert_bound("reparam_kl_fwd kl_sum", kl_sum.reshape(-1)[:1], ref.reshape(1), bound.reshape(1), lambda i: f"kl_sum over n = {n}", worst)


def check_reparam_kl_bwd(mu, lv, mu_p, lv_p, eps, eps_p, dz, dz_p, kl_coef, dmu, dlv, dmu_p, dlv_p, n, worst=None):
    """lstm.cu:90-114: gradients of kl_coef * KL plus the reparameterisation path of dz / dz_p.  Each fp32 quotient of
    expf values carries 2 + 2 ulp; the remaining products, quotients and adds are counted by gamma(k) of their magnitudes."""
    kc = float(np.float32(kl_coef))
    m1, l1, m2, l2, e, ep = (t.reshape(-1)[:n].double() for t in (mu, lv, mu_p, lv_p, eps, eps_p))
    e1, e2, d = torch.exp(l1), torch.exp(l2), m1 - m2
    X = 4.02 * ULP                                      # two expf values in one ratio
    gm1 = kc * d / e2
    bgm1 = gm1.abs() * (2.01 * ULP + gamma(3))
    q = e1 / (2 * e2)
    gl1 = kc * (-0.5 + q)
    bgl1 = abs(kc) * (q.abs() * (X + U) + gamma(2) * (0.5 + q.abs() * (1 + X)))
    Q = (e1 + d * d) / (2 * e2)
    gl2 = kc * (0.5 - Q)
    bgl2 = abs(kc) * (Q.abs() * (X + gamma(4)) * 1.01 + gamma(2) * (0.5 + Q.abs() * 1.01))
    gm2, bgm2 = -gm1, bgm1
    outs = []
    for gm, bgm, gl, bgl, dzz, ee, l in ((gm1, bgm1, gl1, bgl1, dz, e, l1), (gm2, bgm2, gl2, bgl2, dz_p, ep, l2)):
        if dzz is not None:
            v = dzz.reshape(-1)[:n].double()
            bgm = bgm + U * (gm.abs() + bgm + v.abs())
            gm = gm + v
            t = v * ee * 0.5 * torch.exp(0.5 * l)
            bgl = bgl + t.abs() * (2.01 * ULP + gamma(3)) + U * (gl.abs() + bgl + t.abs() * 1.01)
            gl = gl + t
        outs.append((gm, bgm + TINY, gl, bgl + TINY))
    for (gm, bgm, gl, bgl), (om, ol), tag in zip(outs, ((dmu, dlv), (dmu_p, dlv_p)), ("", "_p")):
        assert_bound(f"reparam_kl_bwd dmu{tag}", om.reshape(-1)[:n], gm, bgm, None, worst)
        assert_bound(f"reparam_kl_bwd dlv{tag}", ol.reshape(-1)[:n], gl, bgl, None, worst)


def build_concat_ref(A, ia, ga, Bm, ib, gb, tuc, dt, S, B, ld):
    """lstm.cu:116-134: dst[s, b, :] = [A[ia[s], b] | Bm[ib[s], b] | tuc[s] | dt[s] | zeros to the pitch] -- a copy, exact."""
    a = A.reshape(-1)[:A.numel() // (B * ga) * B * ga].reshape(-1, B, ga)[ia[:S].long()]
    bm = Bm.reshape(-1)[:Bm.numel() // (B * gb) * B * gb].reshape(-1, B, gb)[ib[:S].long()]
    t1 = tuc[:S].reshape(S, 1, 1).expand(S, B, 1)
    t2 = dt[:S].reshape(S, 1, 1).expand(S, B, 1)
    pad = torch.zeros(S, B, ld - ga - gb - 2, dtype=A.dtype, device=A.device)
    return torch.cat([a, bm, t1, t2, pad], 2).reshape(-1)


def check_gather_add_cols(dst_out, dst_in, src, idx, S, T, B, g, W, col0, init, worst=None):
    """lstm.cu:136-149: dst[t, b, j] (+)= sum over s with idx[s] == t of src[s, b, col0 + j], in s order: a chain of at most
    S + 1 fp32 adds."""
    s = src.reshape(-1)[:S * B * W].reshape(S, B, W)[:, :, col0:col0 + g].double()
    ii = idx[:S].long().to(s.device)
    ref = torch.zeros(T, B, g, dtype=torch.float64, device=s.device).index_add_(0, ii, s)
    mag = torch.zeros_like(ref).index_add_(0, ii, s.abs())
    if not init:
        d0 = dst_in.reshape(-1)[:T * B * g].reshape(T, B, g).double()
        ref, mag = ref + d0, mag + d0.abs()
    where = lambda i: f"t {i // (B * g)}, row {(i // g) % B}, column {i % g}"
    assert_bound("gather_add_cols", dst_out.reshape(-1)[:T * B * g], ref, gamma(S + 1) * mag + TINY, where, worst)


def check_align(H, in_idx, h_pred, P, B, g, coef, loss_partial, d_hpred_in, d_hpred, dH_in, dH, worst=None):
    """lstm.cu:151-198 (models/p2p_model.py:224-225): pair s compares h_pred[s] with row 0 of H[in_idx[s]] broadcast over
    the batch.  invn = 1/(B g) rounds once.
      loss_partial[s] = sum (h0 - hp)^2 * invn: each diff rounds once, double sum, one double product, stored as fp32.
      d_hpred += -coef 2 diff invn: three roundings of the term and the add.
      dH[in_idx[s], 0] += coef 2 t invn, t = the 8 row lanes' sums (ceil(B/8) adds each) added in order: gamma(ceil(B/8) + 8)
      of sum |diff|, plus the diffs' own rounding, then three roundings and the add.
    in_idx must hold distinct frames (as the step's does): each pair then owns its row of dH."""
    Hv = H.reshape(-1)[:H.numel() // (B * g) * B * g].reshape(-1, B, g).double()
    ii = in_idx[:P].long().to(Hv.device)
    h0 = Hv[ii, 0].unsqueeze(1)                              # [P, 1, g]: the row-0 quirk
    hp = h_pred.reshape(-1)[:P * B * g].reshape(P, B, g).double()
    diff = h0 - hp
    invn = float(np.float32(1.0) / (np.float32(B) * np.float32(g)))
    ex = 1.0 / (B * g)
    sq = (diff * diff).sum((1, 2))
    lref = sq * ex
    lb = (2 * U * diff * diff + U * U * diff * diff).sum((1, 2)) * ex * (1 + U) + (U + U) * lref + 2.0 ** -45 * lref + 2.0 ** -149
    assert_bound("align loss_partial", loss_partial.reshape(-1)[:P], lref, lb, lambda i: f"pair {i}", worst)
    cf = float(np.float32(coef))
    if d_hpred is not None:
        d0 = d_hpred_in.reshape(-1)[:P * B * g].double()
        term = (-cf * 2 * diff * ex).reshape(-1)
        ref = d0 + term
        b = gamma(4) * term.abs() + U * (d0.abs() + term.abs()) + TINY
        where = lambda i: f"pair {i // (B * g)}, row {(i // g) % B} (lane {(i // g) % B % ALIGN_RL}), column {i % g}"
        assert_bound("align d_hpred", d_hpred.reshape(-1)[:P * B * g], ref, b, where, worst)
    if dH is not None:
        t = diff.sum(1)                                      # [P, g]
        tb = gamma(cdiv(B, ALIGN_RL) + ALIGN_RL + 1) * diff.abs().sum(1)
        term = cf * 2 * t * ex
        tref = dH_in.reshape(-1)[:dH.numel()].double().clone()
        bound = torch.zeros_like(tref)
        rows = (ii * B * g).unsqueeze(1) + torch.arange(g, device=ii.device)   # [P, g] flat offsets of H[in_idx[s], 0, :]
        d0 = tref[rows]
        tref[rows] = d0 + term
        bound[rows] = 2 * abs(cf) * ex * tb * (1 + gamma(3)) + gamma(3) * term.abs() + U * (d0.abs() + term.abs()) + TINY
        where = lambda i: f"frame {i // (B * g)}, row {(i // g) % B}, column {i % g} (pass {i % g // ALIGN_CW})"
        assert_bound("align dH", dH.reshape(-1), tref, bound, where, worst)


def check_colsum(x, rows, cols, ld, out_in, out, accumulate, ws_floats, worst=None, tag="colsum"):
    """out[c] (+)= sum_r x[r, c] (lstm.cu:200-228, :302-329): float64 sum of the kernel's own input, bound gamma(n) of the
    sum of magnitudes with n the longest chain of the plan the kernel launches (colsum_chain)."""
    plan = colsum_plan(rows, cols, ld, ws_floats)
    n = colsum_chain(plan, accumulate)
    xm = torch.as_strided(x, (rows, cols), (ld, 1), x.storage_offset()).double()
    ref, mag = xm.sum(0), xm.abs().sum(0)
    if accumulate:
        o0 = out_in.reshape(-1)[:cols].double()
        ref, mag = ref + o0, mag + o0.abs()
    desc = " + ".join(f"{l['rows']}x{l['cols']} in {l['nchunk']} chunks of {l['rpc']}" for l in plan)
    assert_bound(f"{tag}", out.reshape(-1)[:cols], ref, gamma(n) * mag + TINY, lambda c: f"column {c} ({desc}; chain {n})", worst)
    return plan


# ------------------------------------------------------------------ activations

ACT_NONE, ACT_LRELU, ACT_TANH, ACT_SIGMOID, ACT_RELU = 0, 1, 2, 3, 4


def act_fwd_ref(x, act):
    """lstm.cu:230-239: tanhf 2 ulp; 0.2f v one rounding; sigmoid as common.cuh:115; ReLU and identity exact."""
    v = x.double()
    if act == ACT_TANH:
        y = torch.tanh(v)
        return y, tanh_err(v, 0.0, False)
    if act == ACT_LRELU:
        y = torch.where(v > 0, v, LRELU_SLOPE * v)
        return y, U * y.abs()
    if act == ACT_SIGMOID:
        return torch.sigmoid(v), sigmoid_err(v, 0.0, False)
    if act == ACT_RELU:
        return v.clamp_min(0), torch.zeros_like(v)
    return v, torch.zeros_like(v)


def act_bwd_ref(dy, y, act):
    """lstm.cu:240-248, dx = dy * act'(from y): tanh 1 - y^2 and sigmoid y (1 - y) round twice and the product once
    (gamma 3); the leaky slope once; ReLU and identity exact."""
    d, yv = dy.double(), y.double()
    if act == ACT_TANH:
        r = d * (1 - yv * yv)
        return r, gamma(3) * d.abs() * (1 + yv * yv)
    if act == ACT_SIGMOID:
        r = d * yv * (1 - yv)
        return r, gamma(3) * r.abs()
    if act == ACT_LRELU:
        r = torch.where(yv > 0, d, LRELU_SLOPE * d)
        return r, U * r.abs()
    if act == ACT_RELU:
        return torch.where(yv > 0, d, torch.zeros_like(d)), torch.zeros_like(d)
    return d, torch.zeros_like(d)


# ------------------------------------------------------------------ LayerNorm

def check_layernorm_fwd(x, gamma_, beta, y, mean, rstd, rows, C, eps=1e-5, worst=None):
    """mlp.cu:7-32, one warp per row.  mean: lane sums of ceil(C/32) then 5 shuffle adds and the division.  rstd is checked
    against the variance about the kernel's own mean (the fmaf chain: its diffs round once, then gamma(ceil(C/32) + 5)),
    /C and + eps round once each, rsqrtf 2 ulp.  y is teacher-forced from the kernel's mean and rstd: (x - m) r gamma + beta,
    four roundings."""
    eps = float(np.float32(eps))
    xv = x.reshape(-1)[:rows * C].reshape(rows, C).double()
    n = cdiv(C, 32) + 5
    m = xv.mean(1)
    assert_bound("layernorm_fwd mean", mean.reshape(-1)[:rows], m, gamma(n + 1) * xv.abs().mean(1) + TINY, lambda r: f"row {r}", worst)
    mk = mean.reshape(-1)[:rows].double()
    dv = xv - mk[:, None]
    var = (dv * dv).sum(1)
    ev = (gamma(n) + 2 * U + U * U) * var * (1 + gamma(n))
    vv = var / C + eps
    rel = (ev / C) / vv + gamma(2)
    r = 1.0 / torch.sqrt(vv)
    assert_bound("layernorm_fwd rstd", rstd.reshape(-1)[:rows], r, r * (0.5 * rel / (1 - rel) + 2 * ULP) + TINY, lambda i: f"row {i}", worst)
    rk = rstd.reshape(-1)[:rows].double()
    gm, bt = gamma_.reshape(-1)[:C].double(), beta.reshape(-1)[:C].double()
    t = dv * rk[:, None] * gm
    ref = t + bt
    assert_bound("layernorm_fwd y", y.reshape(-1)[:rows * C], ref, gamma(4) * (t.abs() + bt.abs()) + TINY,
                 lambda i: f"row {i // C}, column {i % C}", worst)


def check_layernorm_bwd(dy, x, mean, rstd, gamma_, dx, dgamma, dbeta, rows, C, worst=None):
    """mlp.cu:34-101 from the kernel's inputs (mean and rstd are inputs here).  g = dy gamma and xh = (x - m) r round once and
    twice; s0 = mean(g), s1 = mean(g xh): warp chains of ceil(C/32) + 5 and the division; dx = r (g - s0 - xh s1): the
    inputs' errors plus four roundings.  dgamma = sum dy xh, dbeta = sum dy over rows in chunks (ln_bwd_chunks): chains of
    ceil(rpc/8) + 8 + nchunk."""
    d = dy.reshape(-1)[:rows * C].reshape(rows, C).double()
    xv = x.reshape(-1)[:rows * C].reshape(rows, C).double()
    m, r = mean.reshape(-1)[:rows].double()[:, None], rstd.reshape(-1)[:rows].double()[:, None]
    gm = gamma_.reshape(-1)[:C].double()
    g = d * gm
    xh = (xv - m) * r
    s0 = g.mean(1, keepdim=True)
    s1 = (g * xh).mean(1, keepdim=True)
    n = cdiv(C, 32) + 5 + 1
    e0 = gamma(n + 1) * g.abs().mean(1, keepdim=True)
    e1 = gamma(n + 4) * (g * xh).abs().mean(1, keepdim=True)
    ref = r * (g - s0 - xh * s1)
    b = r.abs() * (U * g.abs() + e0 + xh.abs() * e1 + s1.abs() * gamma(2) * xh.abs()
                   + gamma(3) * (g.abs() + s0.abs() + e0 + (xh * s1).abs() * 1.01 + xh.abs() * e1)) + U * ref.abs() + TINY
    assert_bound("layernorm_bwd dx", dx.reshape(-1)[:rows * C], ref, b, lambda i: f"row {i // C}, column {i % C}", worst)
    if dgamma is not None:
        nchunk, rpc = ln_bwd_chunks(rows)
        nc = cdiv(rpc, 8) + 8 + nchunk
        where = lambda c: f"column {c} ({nchunk} chunks of {rpc} rows)"
        assert_bound("layernorm_bwd dgamma", dgamma.reshape(-1)[:C], (d * xh).sum(0), gamma(nc + 3) * (d * xh).abs().sum(0) + TINY, where, worst)
        assert_bound("layernorm_bwd dbeta", dbeta.reshape(-1)[:C], d.sum(0), gamma(nc) * d.abs().sum(0) + TINY, where, worst)


# ------------------------------------------------------------------ Adam

def adam_step_size(lr, beta1, beta2, t):
    """loss_adam.cu:139-144: lr sqrt(1 - beta2^t) / (1 - beta1^t) in double, rounded to fp32."""
    bc1, bc2 = 1.0 - beta1 ** t, 1.0 - beta2 ** t
    return float(np.float32(lr * math.sqrt(bc2) / bc1))


def check_adam(p0, g, m0, v0, p, m, v, n, lr, beta1, beta2, eps, t, worst=None):
    """loss_adam.cu:134-158 (PyTorch 1.0 arithmetic, scalars rounded to fp32 as torch rounds them).
      m = m0 beta1 + (1 - beta1) g: three roundings (two once contracted);  v = v0 beta2 + (1 - beta2) g g: four.
      p = p0 - ss m/(sqrtf(v) + eps), teacher-forced from the kernel's m and v: sqrtf, + eps, /, * ss and the subtraction
      round once each (gamma 5 of |p0| + |ss q|)."""
    b1, b2, ep = (float(np.float32(c)) for c in (beta1, beta2, eps))
    o1, o2 = float(np.float32(1.0 - beta1)), float(np.float32(1.0 - beta2))
    gg, mm0, vv0, pp0 = (a.reshape(-1)[:n].double() for a in (g, m0, v0, p0))
    blocks = grid_for(n)
    where = lambda i: f"index {i} (block {i // 256 % blocks}, grid-stride round {i // (256 * blocks)})"
    mref = mm0 * b1 + o1 * gg
    assert_bound("adam m", m.reshape(-1)[:n], mref, gamma(3) * ((mm0 * b1).abs() + (o1 * gg).abs()) + TINY, where, worst)
    vref = vv0 * b2 + o2 * gg * gg
    assert_bound("adam v", v.reshape(-1)[:n], vref, gamma(4) * ((vv0 * b2).abs() + o2 * gg * gg) + TINY, where, worst)
    ss = adam_step_size(lr, beta1, beta2, t)
    mk, vk = m.reshape(-1)[:n].double(), v.reshape(-1)[:n].double()
    q = ss * mk / (torch.sqrt(vk) + ep)
    assert_bound("adam p", p.reshape(-1)[:n], pp0 - q, gamma(5) * (pp0.abs() + q.abs()) + TINY, where, worst)


# ------------------------------------------------------------------ weight packing

def transpose_ref(src, A, P, Q, dtype):
    """dst[a][q][p] = src[a][p][q] (conv_lower.cu:301-323), cast to the destination dtype by round to nearest even."""
    return src.reshape(-1)[:A * P * Q].reshape(A, P, Q).float().transpose(1, 2).reshape(-1).to(dtype)


def blockdiag_ref(src, R, C, g, dtype):
    """dst[(gi, r), (gj, c)] = src[r, c] if gi == gj else 0 (conv_lower.cu:285-299)."""
    m = src.reshape(-1)[:R * C].reshape(R, C).float()
    out = torch.zeros(g, R, g, C, dtype=torch.float32, device=src.device)
    for i in range(g):
        out[i, :, i] = m
    return out.reshape(-1).to(dtype)


def assert_bitexact(name, got, ref):
    got, ref = got.reshape(-1), ref.reshape(-1)
    same = (got.view(torch.int16 if got.dtype == torch.bfloat16 else torch.int32) ==
            ref.view(torch.int16 if ref.dtype == torch.bfloat16 else torch.int32))
    if not bool(same.all()):
        i = int((~same).nonzero()[0])
        raise AssertionError(f"{name}: {int((~same).sum())}/{got.numel()} elements differ, first at index {i}: got "
                             f"{got[i].item()!r}, ref {ref[i].item()!r}")
