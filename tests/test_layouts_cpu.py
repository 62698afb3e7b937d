"""Every format of p2pvg_b200/layouts.py, run through the torch emulation of the kernel ABI and compared element for element
with a plain-torch statement of the format, at the layer shapes of dcgan_64, dcgan_128, vgg_64 and vgg_128 (nc = 1 and 3)."""
import pytest
import torch

from p2pvg_b200 import layouts as L
from p2pvg_b200.engine_vgg import VGG_DEC, VGG_DEC_128, VGG_ENC, VGG_ENC_128
from p2pvg_b200.models.backbone import STAGE_CHANNELS
from tests.emu_backend import EmuKernels

G = 128   # g_dim of every benchmark configuration
K = EmuKernels("cpu")


def _dcgan_convs(width, nc):
    """(Cout, Cin) of every 4x4 conv of the encoder, the final 4x4-valid conv included."""
    chans = STAGE_CHANNELS[width]
    return sorted(set(zip(chans, [nc] + chans[:-1])) | {(G, chans[-1])})


def _dcgan_convts(width, nc):
    """(Cin, Cout) of every 4x4 ConvTranspose of the decoder: upc1, then [d, skip] -> the next stage."""
    chans = STAGE_CHANNELS[width][::-1]
    return sorted({(G, chans[0])} | {(2 * cd, co) for cd, co in zip(chans, chans[1:] + [nc])})


def _vgg_convs(width, nc):
    """(Cout, Cin_total, c0, cin) of every 3x3 pack: both halves of a torch.cat input, and the last ConvTranspose2d(64, nc, 3)
    whose weight [64, nc, 3, 3] is packed as a conv."""
    enc, dec = (VGG_ENC_128, VGG_DEC_128) if width == 128 else (VGG_ENC, VGG_DEC)
    out = {(co, nc if ci is None else ci, 0, nc if ci is None else ci) for stage in enc for ci, co in stage}
    for stage in dec:
        (ci, co), rest = stage[0], stage[1:]
        out |= {(co, ci, 0, ci // 2), (co, ci, ci // 2, ci // 2)} | {(c, i, 0, i) for i, c in rest}
    return sorted(out | {(64, nc, 0, nc)})


def _all(shapes_of):
    return sorted({s for width in (64, 128) for nc in (1, 3) for s in shapes_of(width, nc)})


def _w(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("cout,cin", _all(_dcgan_convs))
def test_conv4_pack_and_unpack(cout, cin):
    w = _w(cout, cin, 4, 4)
    wp = torch.empty(cout * 16 * cin, dtype=torch.bfloat16)
    L.pack_conv4(K, w, wp)
    assert torch.equal(wp, w.permute(0, 2, 3, 1).reshape(-1).to(torch.bfloat16))
    w32 = torch.empty(cout * 16 * cin)
    L.pack_conv4(K, w, w32)
    back = torch.empty_like(w)
    L.unpack_conv4(K, w32, back)
    assert torch.equal(back, w)


@pytest.mark.parametrize("cin,cout", _all(_dcgan_convts))
def test_convt4_pack_and_unpack(cin, cout):
    w = _w(cin, cout, 4, 4)
    wp = torch.empty(cin * 16 * cout, dtype=torch.bfloat16)
    L.pack_convt4(K, w, wp)
    assert torch.equal(wp, w.permute(0, 2, 3, 1).reshape(-1).to(torch.bfloat16))
    w32 = torch.empty(cin * 16 * cout)
    L.pack_convt4(K, w, w32)
    back = torch.empty_like(w)
    L.unpack_convt4(K, w32, back)
    assert torch.equal(back, w)


@pytest.mark.parametrize("reps,C", [(16, 512), (4, 64)])
def test_tile_bias(reps, C):
    b = _w(C)
    out = torch.empty(reps * C)
    L.tile_bias(K, b, out, reps)
    assert torch.equal(out, b.repeat(reps))


@pytest.mark.parametrize("cout,cin_total,c0,cin", _all(_vgg_convs))
def test_conv3_packs(cout, cin_total, c0, cin):
    w = _w(cout, cin_total, 3, 3)
    ld = L.up8(9 * cin)
    ref = w[:, c0:c0 + cin].permute(0, 2, 3, 1).reshape(cout, 9 * cin)
    scratch = torch.zeros(cout * 9 * cin + 8)
    out = torch.empty(cout * ld) if ld != 9 * cin else scratch
    L.pack_conv3(K, w, out, c0, cin, scratch=scratch)
    rows = out[:cout * ld].view(cout, ld)
    assert torch.equal(rows[:, :9 * cin], ref)
    # pad columns: the next row's first weights, the zero slack after the last row
    flat = torch.cat([ref.reshape(-1), torch.zeros(8)])
    pad = torch.arange(1, cout + 1)[:, None] * 9 * cin + torch.arange(ld - 9 * cin)
    assert torch.equal(rows[:, 9 * cin:], flat[pad])
    wt = torch.empty(cin * 9 * cout, dtype=torch.bfloat16)
    L.pack_conv3_t(K, w, wt, c0, cin)
    assert torch.equal(wt, w[:, c0:c0 + cin].permute(1, 2, 3, 0).reshape(-1).to(torch.bfloat16))


@pytest.mark.parametrize("cout,cin_total,c0,cin", [s for s in _all(_vgg_convs) if s[2] == 0])
def test_conv3_unpack(cout, cin_total, c0, cin):
    """unpack_conv3 inverts pack_conv3: of the whole weight, or (halves = 2) of the two halves of a torch.cat input."""
    w = _w(cout, cin_total, 3, 3)
    ld = L.up8(9 * cin)
    halves = cin_total // cin
    gw = torch.empty(halves * cout * ld)
    scratch = torch.zeros(cout * 9 * cin + 8)
    for h in range(halves):
        L.pack_conv3(K, w, gw[h * cout * ld:], h * cin, cin, scratch=scratch)
    back = torch.empty_like(w)
    L.unpack_conv3(K, gw, back, halves=halves)
    assert torch.equal(back, w)


@pytest.mark.parametrize("N,C,H", [(6, 1, 64), (4, 3, 64), (2, 3, 128), (3, 512, 4)])
def test_nchw_nhwc(N, C, H):
    x = _w(N, C, H, H)
    a = torch.empty(N * H * H * C, dtype=torch.bfloat16)
    L.nchw_to_nhwc(K, x, a, N, H * H, C)
    assert torch.equal(a, x.permute(0, 2, 3, 1).reshape(-1).to(torch.bfloat16))
    back = torch.empty(N, C, H, H)
    L.nhwc_to_nchw(K, a, back, N, H * H, C)
    assert torch.equal(back, x.to(torch.bfloat16).float())


def test_cast():
    x = _w(1000)
    b = torch.full((1024,), 7.0, dtype=torch.bfloat16)
    L.cast(K, x, b, 1000)
    assert torch.equal(b[:1000], x.to(torch.bfloat16)) and bool((b[1000:] == 7).all())
    f = torch.empty(1000)
    L.cast(K, b, f, 1000)
    assert torch.equal(f, x.to(torch.bfloat16).float())


def test_up8_and_implicit_shape():
    assert [L.up8(n) for n in (1, 8, 9, 27, 576)] == [8, 8, 16, 32, 576]
    assert L.implicit_shape(64, 512) and L.implicit_shape(1024, 512)
    assert not L.implicit_shape(3, 64) and not L.implicit_shape(64, 1) and not L.implicit_shape(96, 64)
