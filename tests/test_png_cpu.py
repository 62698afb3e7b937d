"""The NumPy PNG reader against PIL, and the PNG encoder's host-side plan and Adler-32 combination against zlib (no GPU)."""
import io
import sys
import types
import zlib

import numpy as np
import pytest
from PIL import Image

from p2pvg_b200 import png
from tests.png_ref import read_png


@pytest.mark.parametrize("mode,shape", [("RGB", (1, 1)), ("RGB", (7, 13)), ("RGB", (64, 333)), ("L", (31, 17)),
                                        ("RGBA", (9, 5))])
@pytest.mark.parametrize("optimize", [False, True])
def test_reader_matches_pil(mode, shape, optimize):
    g = np.random.RandomState(shape[0] * 1000 + shape[1])
    ch = {"RGB": 3, "L": 1, "RGBA": 4}[mode]
    # smooth content with noise and flat areas, so that PIL picks every filter type somewhere
    y, x = np.mgrid[:shape[0], :shape[1]]
    a = (y[..., None] * 3 + x[..., None] * 5 + g.randint(0, 4, shape + (ch,))) % 256
    a[: shape[0] // 3] = 0
    a = a.astype(np.uint8)
    img = Image.fromarray(a[..., 0] if ch == 1 else a, mode)
    buf = io.BytesIO()
    img.save(buf, format="PNG", optimize=optimize)
    px, info = read_png(buf.getvalue())
    want = np.asarray(Image.open(io.BytesIO(buf.getvalue())))
    assert np.array_equal(px.reshape(want.shape), want)
    assert (info["H"], info["W"]) == shape


def test_reader_rejects_a_bad_crc():
    buf = io.BytesIO()
    Image.fromarray(np.zeros((4, 4, 3), np.uint8)).save(buf, format="PNG")
    data = bytearray(buf.getvalue())
    data[20] ^= 1   # inside IHDR
    with pytest.raises(AssertionError, match="CRC"):
        read_png(bytes(data))


@pytest.mark.parametrize("H,W", [(1, 1), (1, 21845), (1, 21846), (50, 1000), (3840, 1920), (640, 3840)])
def test_segment_plan_covers_the_stream(H, W):
    plan = png.segment_plan(H, W)
    n = png.stream_bytes(H, W)
    assert plan[0][0] == 0 and sum(length for _, length in plan) == n
    assert all(s + length == t for (s, length), (t, _) in zip(plan, plan[1:]))
    assert all(length == png.SEGMENT for _, length in plan[:-1]) and 0 < plan[-1][1] <= png.SEGMENT


@pytest.mark.parametrize("n,seg", [(1, 7), (100, 7), (1000, 64), (300000, 65536), (200003, 65536)])
def test_adler32_combine_matches_zlib(n, seg):
    data = np.random.RandomState(n).randint(0, 256, n).astype(np.uint8).tobytes()
    if n > 1000:
        data = data[:n // 2] + b"\xff" * (n - n // 2)   # long runs of the largest byte stress the sums
    pieces = [data[s:s + seg] for s in range(0, n, seg)]
    got = png.adler32_combine([png.adler32_parts(p) for p in pieces], [len(p) for p in pieces])
    assert got == zlib.adler32(data)


def test_save_image_falls_back_to_torchvision_for_cpu_input(monkeypatch, tmp_path):
    import torch
    calls = []
    fake = types.SimpleNamespace(save_image=lambda t, fp, format=None, **kw: calls.append((fp, format, kw)),
                                 make_grid=None)
    tv = types.ModuleType("torchvision")
    tv.utils = fake
    monkeypatch.setitem(sys.modules, "torchvision", tv)
    monkeypatch.setitem(sys.modules, "torchvision.utils", fake)
    png.save_image(torch.zeros(3, 4, 4), str(tmp_path / "a.png"), nrow=2)
    assert calls == [(str(tmp_path / "a.png"), None, {"nrow": 2})]


def test_encode_png_rejects_bad_input():
    import torch
    with pytest.raises(ValueError, match="rule"):
        png.encode_png([], rule="jpeg")
    assert png.encode_png([]) == []
    with pytest.raises(ValueError, match="CUDA"):
        png.encode_png([torch.zeros(3, 2, 2)])


def test_dropin_vis_seq_passes_the_gpu_writer(monkeypatch):
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    monkeypatch.syspath_prepend(os.path.join(root, "dropin"))
    for m in [m for m in sys.modules if m == "misc" or m.startswith("misc.")]:
        monkeypatch.delitem(sys.modules, m)
    import misc.visualize as dv
    seen = {}
    monkeypatch.setattr(dv._fast, "check_vis_seq", lambda *a, **k: None)
    monkeypatch.setattr(dv._fast, "vis_seq", lambda *a, **k: seen.update(k))
    dv.vis_seq(None, None, 0, 10)
    assert seen["save_png"] is png.save_image
