"""256-row tiles of the 64-channel transposed convolutions (kind 2, Cn = 64) and the row-cooperative epilogue with a bf16
skip addend (kinds 0 and 2), at the dcgan_64 C2 launch shapes.

Each launch is held two ways: against float64 (torch.conv_transpose2d on the same bf16 operands, on a sample of images
for the large launches), and for bit-identity against the same launch with fused BatchNorm statistics, which runs on
128-row tiles with the thread-per-row epilogue and stores exactly what the plain launch stores."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def K():
    from p2pvg_b200._lib import CudaKernels
    return CudaKernels("cuda")


def operands(N, H, Ck, Cn, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn(N, H, H, Ck, device="cuda", generator=g) * 0.5).bfloat16()          # NHWC small map
    wp = (torch.randn(Ck, 4, 4, Cn, device="cuda", generator=g) * 0.05).bfloat16()       # [Ck, kh, kw, Cn]
    bias = torch.randn(Cn, device="cuda", generator=g)
    return x, wp, bias


def reference(x, wp, bias, idx):
    """float64 transposed convolution of images idx, NHWC"""
    w = wp.permute(0, 3, 1, 2).double()
    y = F.conv_transpose2d(x[idx].permute(0, 3, 1, 2).double(), w, None if bias is None else bias.double(), stride=2, padding=1)
    return y.permute(0, 2, 3, 1)


def sample(N):
    """all images of a small launch; for a large one the first, last and middle ones and those around image 256"""
    if N <= 16:
        return torch.arange(N, device="cuda")
    picks = {0, 1, N // 2, N - 2, N - 1} | {i for i in (255, 256, 257) if i < N}
    return torch.tensor(sorted(picks), device="cuda")


def check_bf16(out, want):
    """one rounding to bf16 of a float32 accumulation: relative 2^-8, plus the float32 sums' own error"""
    err = (out.double() - want).abs()
    tol = want.abs() * 2.0 ** -8 + 1e-4 * want.abs().max().item() + 1e-6
    assert (err <= tol).all(), (err - tol).max().item()


def stat_partial(N, H, Cn):
    return torch.empty((N * H * H + 127) // 128 * 4, Cn, 2, device="cuda")


# N, H(small), Ck: dec2 / the enc1 data gradient (T * B = 7680 images of 16 x 16), the skip half (B = 256 images), maps
# whose pixel count is not a multiple of 256 (5 x 8 x 8 = 320, 7 x 4 x 4 = 112, 3 x 2 x 2 = 12), 256-pixel boxes spanning
# one image row block (H = 32) and 16 images (H = 4)
SHAPES = [(7680, 16, 128), (256, 16, 128), (5, 8, 128), (7, 4, 64), (3, 2, 128), (6, 32, 64), (40, 4, 128)]


@pytest.mark.parametrize("N,H,Ck", SHAPES)
def test_kind2_cn64_plain(K, N, H, Ck):
    """bias, bf16 and fp32 outputs (row-cooperative and thread-per-row stores of 256-row tiles)"""
    Cn = 64
    x, wp, bias = operands(N, H, Ck, Cn, seed=10 + N)
    out = torch.empty(N, 2 * H, 2 * H, Cn, device="cuda", dtype=torch.bfloat16)
    K.conv_gemm(2, x, wp, out, N, H, H, Ck, Cn, bias=bias)
    idx = sample(N)
    want = reference(x, wp, bias, idx)
    check_bf16(out[idx], want)
    out32 = torch.empty(N, 2 * H, 2 * H, Cn, device="cuda")
    K.conv_gemm(2, x, wp, out32, N, H, H, Ck, Cn, bias=bias)
    assert ((out32[idx].double() - want).abs() <= 1e-4 * want.abs().max().item() + 1e-6).all()
    ref = torch.empty_like(out)
    K.conv_gemm(2, x, wp, ref, N, H, H, Ck, Cn, bias=bias, stat_partial=stat_partial(N, H, Cn))
    assert torch.equal(out, ref), "256-row tiles must store what 128-row tiles store"


@pytest.mark.parametrize("N,H,Ck,Cn,B", [(7680, 16, 128, 64, 256), (7680, 8, 256, 128, 256), (5, 8, 128, 64, 1),
                                        (12, 4, 64, 64, 3), (20, 8, 128, 128, 4), (6, 32, 64, 64, 2)])
def test_kind2_skip_addend(K, N, H, Ck, Cn, B):
    """dec2 (Cn = 64, 256-row tiles) and dec1 (Cn = 128) with the skip half as a bf16 addend indexed through grp_src, no
    bias (it is folded into the addend), plus a bias at a small shape"""
    x, wp, bias = operands(N, H, Ck, Cn, seed=20 + N + Cn)
    G, nsrc = N // B, 2
    g = torch.Generator(device="cuda").manual_seed(7)
    addend = torch.randn(nsrc * B, 2 * H, 2 * H, Cn, device="cuda", generator=g).bfloat16()
    src = torch.tensor([(3 * gi + 1) % nsrc for gi in range(G)], dtype=torch.int32, device="cuda")
    img_src = (src.long().repeat_interleave(B) * B + torch.arange(N, device="cuda") % B)
    idx = sample(N)
    for b in (None, bias) if N < 1000 else (None,):
        out = torch.empty(N, 2 * H, 2 * H, Cn, device="cuda", dtype=torch.bfloat16)
        K.conv_gemm(2, x, wp, out, N, H, H, Ck, Cn, bias=b, addend=addend, grp_src=src, imgs_per_group=B)
        want = reference(x, wp, b, idx) + addend[img_src[idx]].double()
        check_bf16(out[idx], want)
        ref = torch.empty_like(out)
        K.conv_gemm(2, x, wp, ref, N, H, H, Ck, Cn, bias=b, addend=addend, grp_src=src, imgs_per_group=B,
                    stat_partial=stat_partial(N, H, Cn))
        assert torch.equal(out, ref), "the row-cooperative addend epilogue must store what the thread-per-row one stores"


@pytest.mark.parametrize("N,H,Ck,Cn,B", [(16, 8, 64, 128, 4), (6, 16, 128, 64, 2), (5, 8, 64, 64, 5)])
def test_kind0_skip_addend(K, N, H, Ck, Cn, B):
    """kind 0 (stride-2 convolution) with a bf16 addend on the row-cooperative epilogue"""
    g = torch.Generator(device="cuda").manual_seed(30 + N)
    x = (torch.randn(N, 2 * H, 2 * H, Ck, device="cuda", generator=g) * 0.5).bfloat16()
    wp = (torch.randn(Cn, 4, 4, Ck, device="cuda", generator=g) * 0.05).bfloat16()   # [Cn, kh, kw, Ck]
    bias = torch.randn(Cn, device="cuda", generator=g)
    G, nsrc = N // B, 2
    addend = torch.randn(nsrc * B, H, H, Cn, device="cuda", generator=g).bfloat16()
    src = torch.tensor([(gi + 1) % nsrc for gi in range(G)], dtype=torch.int32, device="cuda")
    img_src = src.long().repeat_interleave(B) * B + torch.arange(N, device="cuda") % B
    out = torch.empty(N, H, H, Cn, device="cuda", dtype=torch.bfloat16)
    K.conv_gemm(0, x, wp, out, N, H, H, Ck, Cn, bias=bias, addend=addend, grp_src=src, imgs_per_group=B)
    y = F.conv2d(x.permute(0, 3, 1, 2).double(), wp.permute(0, 3, 1, 2).double(), bias.double(), stride=2, padding=1)
    want = y.permute(0, 2, 3, 1) + addend[img_src].double()
    check_bf16(out, want)
    ref = torch.empty_like(out)
    part = torch.empty((N * H * H + 127) // 128, Cn, 2, device="cuda")
    K.conv_gemm(0, x, wp, ref, N, H, H, Ck, Cn, bias=bias, addend=addend, grp_src=src, imgs_per_group=B, stat_partial=part)
    assert torch.equal(out, ref)
