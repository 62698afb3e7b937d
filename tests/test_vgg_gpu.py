"""vgg_64 backbone on the GPU: kernels vs emulation, 3x3 implicit GEMMs vs torch, train step vs oracle / reference
fixture, drop-in API (reference models/vgg_64.py)."""
import os
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import p2p_oracle as O
from p2pvg_b200.engine import StepPlan
from tests.test_oracle_golden import load_fixture

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "step_vgg64_rgb.pt")


def make_cfg(channels, rnn=256):
    return dict(g_dim=128, z_dim=10, rnn_size=rnn, channels=channels, image_width=64, backbone="vgg", predictor_rnn_layers=2,
                posterior_rnn_layers=1, prior_rnn_layers=1)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_vgg_data_movement_kernels(dtype):
    from p2pvg_b200._lib import CudaKernels
    from tests.emu_vgg import EmuKernelsVGG
    Kc, Ke = CudaKernels("cuda"), EmuKernelsVGG("cuda")
    torch.manual_seed(0)
    N, H, W, C = 3, 8, 16, 24
    x = torch.randn(N, H, W, C, device="cuda").to(dtype)
    x[0, 0, 0, :] = x[0, 0, 1, :]  # ties inside a pooling window: first maximum wins
    dyp = torch.randn(N, H // 2, W // 2, C, device="cuda").to(dtype)
    small = torch.randn(N, H, W, 3, device="cuda").to(dtype)
    bias = torch.randn(3, device="cuda")
    addend = torch.randn(2, 5 * 7, device="cuda")
    src = torch.tensor([1, 0, 1], dtype=torch.int32, device="cuda")
    res = []
    for K in (Kc, Ke):
        out = []
        for sgn in (1, -1):
            col = torch.full((N * H * W * 32,), 7.0, device="cuda").to(dtype)
            K.im2col3(small, col, N, H, W, 3, 32, sgn)
            out.append(col)
        colin = torch.randn(N * H * W, 32, device="cuda").to(dtype)
        torch.manual_seed(3)
        y = torch.empty(N * H * W * 3, device="cuda", dtype=dtype)
        K.col2im3(out[0], y, N, H, W, 3, 32, bias=bias)
        out.append(y)
        p = torch.empty(N * (H // 2) * (W // 2) * C, device="cuda", dtype=dtype)
        K.maxpool2_fwd(x, p, N, H, W, C)
        dx = torch.empty(N * H * W * C, device="cuda", dtype=dtype)
        K.maxpool2_bwd(x, dyp, dx, N, H, W, C)
        u = torch.empty(N * 4 * H * W * C, device="cuda", dtype=dtype)
        K.upsample2_fwd(x, u, N, H, W, C)
        du = torch.empty(N * (H // 2) * (W // 2) * C, device="cuda", dtype=dtype)
        K.upsample2_bwd(x, du, N, H // 2, W // 2, C)
        dst = torch.ones(3, 5 * 7, device="cuda").to(dtype)
        K.gather_add(dst, addend, src, 3, 5 * 7)
        out += [p, dx, u, du, dst]
        res.append(out)
    tol = 1e-6 if dtype == torch.float32 else 2e-2
    for i, (a, b) in enumerate(zip(*res)):
        assert torch.allclose(a.float(), b.float(), rtol=tol, atol=tol), i


def _ref_conv3(x_nhwc, w):
    return F.conv2d(x_nhwc.permute(0, 3, 1, 2).float(), w.float(), padding=1).permute(0, 2, 3, 1)


@pytest.mark.parametrize("N,H,Ck,Cn", [(2, 64, 64, 64), (3, 32, 64, 128), (5, 16, 128, 256), (6, 8, 512, 512), (7, 8, 256, 64), (2, 128, 64, 64)])
def test_conv3_implicit_gemm(N, H, Ck, Cn):
    from p2pvg_b200._lib import CudaKernels
    K = CudaKernels("cuda")
    torch.manual_seed(N)
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        x = torch.randn(N, H, H, Ck, device="cuda").bfloat16()
        w = (torch.randn(Cn, Ck, 3, 3, device="cuda") / (3 * Ck ** 0.5)).bfloat16()
        bias = torch.randn(Cn, device="cuda")
        wp = w.permute(0, 2, 3, 1).contiguous()           # [Cn, (kh,kw,Ck)]
        # kind 3: forward (+ bias + addend gathered per group of 1 image)
        ngrp = 2
        addend = torch.randn(ngrp, H, H, Cn, device="cuda")
        src = torch.tensor([i % ngrp for i in range(N)], dtype=torch.int32, device="cuda")
        y = torch.empty(N, H, H, Cn, device="cuda", dtype=torch.bfloat16)
        K.conv_gemm(3, x, wp, y, N, H, H, Ck, Cn, bias=bias, addend=addend, grp_src=src, imgs_per_group=1)
        ref = _ref_conv3(x, w) + bias + addend[src.long()]
        assert torch.allclose(y.float(), ref, rtol=2e-2, atol=2e-2)
        y32 = torch.empty(N, H, H, Cn, device="cuda")
        K.conv_gemm(3, x, wp, y32, N, H, H, Ck, Cn)
        assert torch.allclose(y32, _ref_conv3(x, w), rtol=1e-3, atol=1e-3)
        # kind 5: data gradient  dx = conv_transpose(dy, w)
        dy = torch.randn(N, H, H, Cn, device="cuda").bfloat16()
        wt = w.permute(1, 2, 3, 0).contiguous()           # [Ck, (kh,kw,Cn)]
        dx = torch.empty(N, H, H, Ck, device="cuda")
        K.conv_gemm(5, dy, wt, dx, N, H, H, Cn, Ck)
        refdx = F.conv_transpose2d(dy.permute(0, 3, 1, 2).float(), w.float(), padding=1).permute(0, 2, 3, 1)
        assert torch.allclose(dx, refdx, rtol=1e-3, atol=1e-3)
        # kind 4: weight gradient  gw[Cn, (kh,kw,Ck)]
        gw = torch.empty(Cn, 9 * Ck, device="cuda")
        K.conv_gemm(4, dy, x, gw, N, H, H, 0, Ck, Cm=Cn)
        xr = x.permute(0, 3, 1, 2).float().requires_grad_(False)
        refgw = torch.nn.grad.conv2d_weight(xr, (Cn, Ck, 3, 3), dy.permute(0, 3, 1, 2).float(), padding=1)
        refgw = refgw.permute(0, 2, 3, 1).reshape(Cn, 9 * Ck)
        scale = refgw.abs().max().item()
        assert (gw - refgw).abs().max().item() <= 2e-3 * scale
    finally:
        torch.backends.cudnn.allow_tf32 = prev


def run_step(optkw, T, B, channels, precision, np_seed=0, kernels=None):
    from p2pvg_b200._lib import CudaKernels
    from p2pvg_b200.engine_vgg import TrainEngineVGG
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    cfg = make_cfg(channels)
    state = O.build_state(cfg, seed=1)
    opt = O.default_opt(**optkw)
    opt["batch_size"] = opt["batch_size"] or B
    adt = torch.float32 if precision == "fp32" else torch.bfloat16
    eng = TrainEngineVGG(O.clone_state(state), cfg, opt, kernels or CudaKernels("cuda"), act_dtype=adt)
    x = torch.rand(T, B, channels, 64, 64, generator=torch.Generator().manual_seed(5))
    np.random.seed(np_seed)
    probs = np.random.uniform(0, 1, T - 1)
    eps = O.draw_eps(StepPlan(T, probs, opt).S, B, 10, seed=11)
    got = eng.step(x.cuda(), probs=probs, eps=eps.cuda())
    return (state, opt, x, eps, probs), got, eng


def oracle_step(args):
    state, opt, x, eps, probs = args
    adam = {m: O.new_adam_state(state[m]) for m in O.MODULES}
    return O.train_step(state, adam, x, opt, "vgg", eps, probs, mode="A")


@pytest.mark.parametrize("optkw,T,B,ch,seed", [({}, 4, 2, 3, 0), (dict(skip_prob=0.5, n_past=2, last_frame_skip=True), 6, 2, 1, 3)])
def test_vgg_step_fp32_vs_oracle(optkw, T, B, ch, seed):
    args, got, eng = run_step(optkw, T, B, ch, "fp32", seed)
    ref = oracle_step(args)
    np.testing.assert_allclose(got, np.array(ref["losses"], dtype=np.float32), rtol=1e-4, atol=1e-6)
    for m in O.MODULES:
        for k, gref in ref["grads"][m].items():
            if k.endswith("main.0.bias") or k in ("c5.0.bias", "upc1.0.bias"):
                continue  # bias in front of a training-mode BatchNorm: exactly zero, rounding noise in the oracle
            g = eng.arena[m].g[k].cpu()
            cos = torch.nn.functional.cosine_similarity(g.flatten().double(), gref.flatten().double(), dim=0).item()
            assert cos >= 1 - 1e-4, f"grad {m}.{k}: cosine {cos:.7f}"


def test_vgg_step_bf16_vs_emulation_and_oracle():
    """bf16 activations: the CUDA path (implicit 3x3 GEMMs) against the torch emulation of the same schedule at the same
    precision, and against the fp32 oracle with bf16-level tolerances."""
    from tests.emu_vgg import EmuKernelsVGG
    args, got, eng = run_step({}, 3, 8, 3, "bf16", 1)
    os.environ["P2PVG_IMPLICIT"] = "0"   # the emulation takes the explicit im2col3 route: two independent lowerings
    try:
        _, got_e, eng_e = run_step({}, 3, 8, 3, "bf16", 1, kernels=EmuKernelsVGG("cuda"))
    finally:
        del os.environ["P2PVG_IMPLICIT"]
    assert eng.implicit and not eng_e.implicit
    ref = oracle_step(args)
    np.testing.assert_allclose(got, got_e, rtol=2e-2, atol=1e-5)
    np.testing.assert_allclose(got, np.array(ref["losses"], dtype=np.float32), rtol=3e-2, atol=1e-5)
    rows = []
    for m in O.MODULES:
        for k, gref in ref["grads"][m].items():
            if k.endswith("main.0.bias") or k in ("c5.0.bias", "upc1.0.bias"):
                continue
            g = eng.arena[m].g[k].float().flatten().double().cpu()
            ge = eng_e.arena[m].g[k].float().flatten().double().cpu()
            cs = torch.nn.functional.cosine_similarity
            rows.append((cs(g, ge, dim=0).item(), cs(g, gref.flatten().double(), dim=0).item(),
                         cs(ge, gref.flatten().double(), dim=0).item(), f"{m}.{k}"))
    # 23 bf16 layers deep at batch 8: the two bf16 lowerings must agree closely, and against fp32 the CUDA path must be
    # no further away than the bf16 emulation of the same schedule is
    worst = sorted(rows)[:6]
    assert min(r[0] for r in rows) >= 0.93, worst
    assert float(np.median([r[1] for r in rows])) >= 0.93, worst
    assert min(r[1] - r[2] for r in rows) >= -0.05, sorted(rows, key=lambda r: r[1] - r[2])[:6]


def test_vgg_step_vs_reference_golden():
    from p2pvg_b200._lib import CudaKernels
    from p2pvg_b200.engine_vgg import TrainEngineVGG
    fix = load_fixture(GOLD)
    state = O.build_state(fix["cfg"], seed=fix["init_seed"])
    cfg = dict(fix["cfg"], image_width=64)
    eng = TrainEngineVGG(state, cfg, dict(fix["opt"]), CudaKernels("cuda"), act_dtype=torch.float32)
    rec = fix["steps"][0]
    got = eng.step(rec["x"].cuda(), probs=rec["probs"].numpy(), eps=rec["eps"].cuda())
    np.testing.assert_allclose(got, np.array(rec["losses"], dtype=np.float32), rtol=1e-4, atol=1e-7)
    bad = []
    for m, digs in rec["grad_digest"].items():
        for k, d in digs.items():
            if k.endswith("main.0.bias") or k in ("c5.0.bias", "upc1.0.bias"):
                continue
            f = eng.arena[m].g[k].double().reshape(-1).cpu()
            err = (f[d["idx"]] - d["samples"]).abs()
            # a LeakyReLU slope that flips on a pre-activation within rounding of zero moves one output channel: allow
            # isolated sample outliers, require the bulk to agree
            if (err > 3e-2 * max(d["absmax"], 1e-30)).float().mean().item() > 0.02:
                bad.append((m, k, err.max().item(), d["absmax"]))
    assert not bad, bad


def test_vgg128_step_vs_reference_golden():
    """models/vgg_128.py (5 stages, 128x128): fp32 CUDA path against the unmodified reference's numbers."""
    from p2pvg_b200._lib import CudaKernels
    from p2pvg_b200.engine_vgg import TrainEngineVGG
    fix = load_fixture(os.path.join(os.path.dirname(__file__), "golden", "step_vgg128_gray.pt"))
    state = O.build_state(fix["cfg"], seed=fix["init_seed"])
    cfg = dict(fix["cfg"], image_width=128)
    eng = TrainEngineVGG(state, cfg, dict(fix["opt"]), CudaKernels("cuda"), act_dtype=torch.float32)
    rec = fix["steps"][0]
    got = eng.step(rec["x"].cuda(), probs=rec["probs"].numpy(), eps=rec["eps"].cuda())
    np.testing.assert_allclose(got, np.array(rec["losses"], dtype=np.float32), rtol=1e-4, atol=1e-7)
    bad = []
    for m, digs in rec["grad_digest"].items():
        for k, d in digs.items():
            if k.endswith("main.0.bias") or k in ("c6.0.bias", "upc1.0.bias"):
                continue
            f = eng.arena[m].g[k].double().reshape(-1).cpu()
            err = (f[d["idx"]] - d["samples"]).abs() / max(d["absmax"], 1e-30)
            # 29 BatchNorm layers at batch 2: fp32 noise floor ~2x that of vgg_64 (see tests/test_engine_vgg_emu.py); the bulk
            # of the sampled elements must agree to 1 % of the largest, isolated LeakyReLU-flip outliers are tolerated
            if err.median().item() > 1e-2 or (err > 0.1).float().mean().item() > 0.05:
                bad.append((m, k, err.median().item(), err.max().item()))
    assert not bad, bad


def test_p2pmodel_vgg128_dropin_bf16():
    from p2pvg_b200.models import vgg_128
    from p2pvg_b200.models.p2p_model import P2PModel
    os.environ["P2PVG_PRECISION"], os.environ["P2PVG_GRAPH"] = "bf16", "1"
    T, B = 4, 4
    opt = types.SimpleNamespace(dataset="bair", backbone_net=vgg_128, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0,
                                weight_align=0.5, skip_prob=0.0, n_past=1, last_frame_skip=False, batch_size=B)
    torch.manual_seed(1)
    model = P2PModel(B, 3, 128, 10, 256, 1, 1, 2, opt=opt).cuda()
    assert "c6.0.weight" in model.encoder.state_dict() and "upc6.1.weight" in model.decoder.state_dict()
    x = torch.rand(T, B, 3, 128, 128, generator=torch.Generator().manual_seed(2)).cuda()
    outs = [model(x, 0, T - 1) for _ in range(3)]      # eager, capture, replay
    for o in outs:
        assert len(o) == 4 and all(np.isfinite(float(v)) for v in o)
    assert float(outs[-1][0]) < float(outs[0][0])
    model.eval()
    seq = model.p2p_generate([t for t in x], len_output=4, eval_cp_ix=3)
    assert len(seq) == 4 and seq[1].shape == (B, 3, 128, 128) and torch.isfinite(seq[1]).all()


def test_p2pmodel_vgg_dropin():
    from p2pvg_b200.models import vgg_64
    from p2pvg_b200.models.p2p_model import P2PModel
    os.environ["P2PVG_PRECISION"], os.environ["P2PVG_GRAPH"] = "bf16", "1"
    T, B = 6, 8
    opt = types.SimpleNamespace(dataset="weizmann", backbone_net=vgg_64, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0,
                                weight_align=0.5, skip_prob=0.0, n_past=1, last_frame_skip=False, batch_size=B)
    torch.manual_seed(1)
    model = P2PModel(B, 3, 128, 10, 256, 1, 1, 2, opt=opt).cuda()
    keys = set(model.encoder.state_dict()) | set(model.decoder.state_dict())
    assert "c1.0.main.0.weight" in keys and "upc5.1.weight" in keys and "c5.1.running_mean" in keys
    x = torch.rand(T, B, 3, 64, 64, generator=torch.Generator().manual_seed(2)).cuda()
    outs = [model(x, 0, T - 1) for _ in range(4)]      # eager, capture, replay, replay
    for o in outs:
        assert len(o) == 4 and all(np.isfinite(float(v)) for v in o)
    assert float(outs[-1][0]) < float(outs[0][0])
    model.eval()
    seq = model.p2p_generate([t for t in x], len_output=6, eval_cp_ix=5)
    assert len(seq) == 6 and seq[2].shape == (B, 3, 64, 64) and torch.isfinite(seq[2]).all()
    # stand-alone module calls (train-mode BatchNorm) against the oracle's functional forward
    model.train()
    os.environ["P2PVG_PRECISION"] = "fp32"
    try:
        h, skips = model.encoder(x[0])
        p = {k: v.detach().float().cpu() for k, v in model.encoder.state_dict().items()}
        h_ref, skips_ref = O.vgg_encoder_fwd(p, x[0].cpu())
        assert torch.allclose(h.cpu(), h_ref, atol=2e-4) and torch.allclose(skips[2].cpu(), skips_ref[2], atol=2e-4)
        out = model.decoder([h, skips])
        pd = {k: v.detach().float().cpu() for k, v in model.decoder.state_dict().items()}
        out_ref = O.vgg_decoder_fwd(pd, h_ref, skips_ref)
        assert torch.allclose(out.cpu(), out_ref, atol=5e-4)
    finally:
        os.environ["P2PVG_PRECISION"] = "bf16"
