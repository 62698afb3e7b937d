"""Implicit-GEMM convolution family (p2pvg_conv_gemm: 4-D TMA pixel-box loads + wgmma) against torch's
conv2d / conv_transpose2d on the same bf16 operands (fp32 reference arithmetic)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def K():
    from p2pvg_b200._lib import CudaKernels
    return CudaKernels("cuda")


def nhwc(t):  # NCHW -> flat NHWC
    return t.permute(0, 2, 3, 1).contiguous()


SHAPES = [  # N, H(small), Ck, Cn
    (5, 8, 64, 128), (3, 4, 128, 64), (2, 16, 64, 64), (9, 4, 512, 256), (2, 32, 64, 64), (17, 8, 256, 128), (1, 16, 128, 256),
]


@pytest.mark.parametrize("N,H,Ck,Cn", SHAPES)
def test_kind0_conv_s2(K, N, H, Ck, Cn):
    torch.manual_seed(0)
    x = (torch.randn(N, Ck, 2 * H, 2 * H, device="cuda") * 0.5).bfloat16()
    w = (torch.randn(Cn, Ck, 4, 4, device="cuda") * 0.05).bfloat16()
    bias = torch.randn(Cn, device="cuda")
    ref = F.conv2d(x.float(), w.float(), bias, stride=2, padding=1)
    wp = w.permute(0, 2, 3, 1).contiguous()  # [Cn, kh, kw, Ck]
    out = torch.empty(N, H, H, Cn, device="cuda", dtype=torch.bfloat16)
    K.conv_gemm(0, nhwc(x), wp, out, N, H, H, Ck, Cn, bias=bias)
    err = (out.float() - nhwc(ref)).abs().max().item()
    assert err <= 2e-2 * ref.abs().max().item() + 1e-2, err
    out32 = torch.empty(N, H, H, Cn, device="cuda")
    K.conv_gemm(0, nhwc(x), wp, out32, N, H, H, Ck, Cn, bias=bias)
    assert (out32 - nhwc(ref)).abs().max().item() <= 2e-3 * ref.abs().max().item() + 1e-3


@pytest.mark.parametrize("N,H,Ck,Cn", SHAPES)
def test_kind2_conv_transpose_s2(K, N, H, Ck, Cn):
    torch.manual_seed(1)
    B = 1 if N % 2 else 2  # images per group
    G = N // B
    x = (torch.randn(N, Ck, H, H, device="cuda") * 0.5).bfloat16()
    w = (torch.randn(Ck, Cn, 4, 4, device="cuda") * 0.05).bfloat16()
    bias = torch.randn(Cn, device="cuda")
    ref = F.conv_transpose2d(x.float(), w.float(), bias, stride=2, padding=1)
    wp = w.permute(0, 2, 3, 1).contiguous()  # [Ck, kh, kw, Cn]
    out = torch.empty(N, 2 * H, 2 * H, Cn, device="cuda")
    K.conv_gemm(2, nhwc(x), wp, out, N, H, H, Ck, Cn, bias=bias)
    assert (out - nhwc(ref)).abs().max().item() <= 2e-3 * ref.abs().max().item() + 1e-3
    # shared addend (skip half) indexed through grp_src, bf16 output
    nsrc = 2
    addend = torch.randn(nsrc * B, 2 * H, 2 * H, Cn, device="cuda")
    src = torch.tensor([g % nsrc for g in range(G)], dtype=torch.int32, device="cuda")
    idx = torch.tensor([(g % nsrc) * B + b for g in range(G) for b in range(B)], device="cuda")
    outb = torch.empty(N, 2 * H, 2 * H, Cn, device="cuda", dtype=torch.bfloat16)
    K.conv_gemm(2, nhwc(x), wp, outb, N, H, H, Ck, Cn, bias=bias, addend=addend, grp_src=src, imgs_per_group=B)
    want = nhwc(ref) + addend[idx]
    assert (outb.float() - want).abs().max().item() <= 2e-2 * want.abs().max().item() + 1e-2
    # the same with the addend stored in bf16 (p2pvg_conv_fusion.addend_dtype)
    add16 = addend.bfloat16()
    outc = torch.empty_like(outb)
    K.conv_gemm(2, nhwc(x), wp, outc, N, H, H, Ck, Cn, bias=bias, addend=add16, grp_src=src, imgs_per_group=B)
    want16 = nhwc(ref) + add16.float()[idx]
    assert (outc.float() - want16).abs().max().item() <= 2e-2 * want16.abs().max().item() + 1e-2


@pytest.mark.parametrize("N,H,Cm,Cn", [(5, 8, 128, 64), (3, 4, 64, 128), (2, 16, 64, 64), (64, 4, 512, 256), (40, 8, 256, 128), (9, 32, 64, 64)])
def test_kind1_weight_gradient(K, N, H, Cm, Cn):
    torch.manual_seed(2)
    a = (torch.randn(N, Cm, H, H, device="cuda") * 0.5).bfloat16()          # small map (e.g. dY of a conv)
    b = (torch.randn(N, Cn, 2 * H, 2 * H, device="cuda") * 0.5).bfloat16()  # big map (e.g. the conv input)
    # reference: d/dW of sum(conv2d(b, W) * a) = conv weight gradient [Cm, Cn, 4, 4]
    w = torch.zeros(Cm, Cn, 4, 4, device="cuda", requires_grad=True)
    (F.conv2d(b.float(), w, stride=2, padding=1) * a.float()).sum().backward()
    ref = w.grad.permute(0, 2, 3, 1).reshape(Cm, 16 * Cn)
    out = torch.empty(Cm, 16 * Cn, device="cuda")
    K.conv_gemm(1, nhwc(a), nhwc(b), out, N, H, H, 0, Cn, Cm=Cm)
    assert (out - ref).abs().max().item() <= 2e-3 * ref.abs().max().item() + 1e-2
    out2 = out.clone()
    K.conv_gemm(1, nhwc(a), nhwc(b), out2, N, H, H, 0, Cn, Cm=Cm, accumulate=True)
    assert (out2 - 2 * ref).abs().max().item() <= 4e-3 * ref.abs().max().item() + 2e-2


@pytest.mark.parametrize("kind,N,H,Ck,Cn,B", [(0, 16, 8, 64, 128, 4), (0, 32, 4, 128, 256, 8), (0, 6, 16, 64, 64, 2), (2, 16, 8, 128, 64, 4),
                                               (2, 24, 4, 256, 128, 8), (2, 4, 16, 64, 256, 2), (0, 5, 8, 64, 128, 0)])
def test_fused_batchnorm_statistics(K, kind, N, H, Ck, Cn, B):
    """BatchNorm forward statistics from the GEMM epilogue (per-tile column sums + p2pvg_bn_fwd_finalize_tiles) against the
    statistics of the stored bf16 output, per group of B images.  B = 0: one ragged group (rows not a multiple of 128):
    only the per-tile sums are checked."""
    torch.manual_seed(3)
    Hin = 2 * H if kind == 0 else H
    Hout = H if kind == 0 else 2 * H
    x = (torch.randn(N, Hin, Hin, Ck, device="cuda") * 0.5).bfloat16()
    taps = 16
    wp = (torch.randn(Cn if kind == 0 else Ck, taps * (Ck if kind == 0 else Cn), device="cuda") * 0.05).bfloat16()
    bias = torch.randn(Cn, device="cuda")
    out = torch.empty(N, Hout, Hout, Cn, device="cuda", dtype=torch.bfloat16)
    phases = 4 if kind == 2 else 1
    rows = N * H * H
    ntiles = (rows + 127) // 128
    part = torch.full((ntiles * phases, Cn, 2), float("nan"), device="cuda")
    K.conv_gemm(kind, x, wp, out, N, H, H, Ck, Cn, bias=bias, stat_partial=part)
    ref_out = torch.empty_like(out)
    K.conv_gemm(kind, x, wp, ref_out, N, H, H, Ck, Cn, bias=bias)
    assert torch.equal(out, ref_out), "the fused statistics must not change the stored output"
    o = out.float()
    tot = part.double().sum(0)
    assert torch.isfinite(part).all()
    s_ref, q_ref = o.double().sum((0, 1, 2)), (o.double() ** 2).sum((0, 1, 2))
    assert torch.allclose(tot[:, 0], s_ref, rtol=1e-5, atol=1e-2) and torch.allclose(tot[:, 1], q_ref, rtol=1e-5, atol=1e-2)
    if B == 0:
        return
    G = N // B
    R = B * Hout * Hout
    gamma, beta = torch.rand(Cn, device="cuda") + 0.5, torch.randn(Cn, device="cuda")
    outs = [torch.empty(G * Cn, device="cuda") for _ in range(5)]
    K.bn_fwd_finalize_tiles(part, (B * H * H // 128) * phases, Cn, 1, G, R, Cn, gamma, beta, *outs)
    refs = [torch.empty(G * Cn, device="cuda") for _ in range(5)]
    K.bn_fwd_stats(out, G, R, Cn, gamma, beta, *refs)
    for a, b, nm in zip(outs, refs, ("mean", "invstd", "var_unbiased", "scale", "shift")):
        assert torch.allclose(a, b, rtol=2e-5, atol=2e-6), nm
