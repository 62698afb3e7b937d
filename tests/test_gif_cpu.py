"""The NumPy GIF reader against PIL, the encoder's segment, bit-offset and sub-block plan against a host restatement, and
the native CRC-32C against TensorBoard's (no GPU)."""
import io
import os
import sys
import types

import numpy as np
import pytest
from PIL import Image

from p2pvg_b200 import gif, tboard
from tests.gif_ref import encode_frame_data, lzw_segment, read_gif

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DROPIN_PACKAGES = ("tensorboardX", "misc")


@pytest.fixture
def dropin(monkeypatch):
    """dropin/ first on sys.path with no tensorboardX or misc module loaded; afterwards every such module the test
    imported is removed and the ones loaded before are restored, so later tests see the interpreter's own modules
    (importlib.util.find_spec answers from sys.modules)."""
    monkeypatch.syspath_prepend(os.path.join(ROOT, "dropin"))
    for m in [m for m in sys.modules if m.split(".")[0] in DROPIN_PACKAGES]:
        monkeypatch.delitem(sys.modules, m)
    yield
    for m in [m for m in sys.modules if m.split(".")[0] in DROPIN_PACKAGES]:
        del sys.modules[m]


def pil_gif(frames, **kw):
    buf = io.BytesIO()
    ims = [Image.fromarray(f) for f in frames]
    ims[0].save(buf, format="GIF", save_all=True, append_images=ims[1:], **kw)
    return buf.getvalue()


def pil_frames(data):
    im = Image.open(io.BytesIO(data))
    out, durations = [], []
    for k in range(getattr(im, "n_frames", 1)):
        im.seek(k)
        out.append(np.asarray(im.convert("RGB")))
        durations.append(im.info.get("duration"))
    return np.stack(out), durations, im.info.get("loop")


@pytest.mark.parametrize("kind", ["grey", "colour", "flat", "tiny"])
def test_reader_matches_pil(kind):
    g = np.random.RandomState(3)
    if kind == "grey":
        frames = [np.repeat(g.randint(0, 256, (40, 57, 1)), 3, 2).astype(np.uint8) for _ in range(3)]
    elif kind == "colour":
        y, x = np.mgrid[:48, :64]
        frames = [np.stack([(x * 4 + t * 9) % 256, (y * 5) % 256, g.randint(0, 256, x.shape)], -1).astype(np.uint8)
                  for t in range(4)]
    elif kind == "flat":
        frames = [np.full((16, 16, 3), v, np.uint8) for v in (0, 90, 255)]
    else:
        frames = [g.randint(0, 256, (1, 1, 3)).astype(np.uint8) for _ in range(2)]
    data = pil_gif(frames, duration=70, loop=0)
    got, info = read_gif(data)
    want, durations, loop = pil_frames(data)
    assert np.array_equal(got, want)
    assert info["loop"] == loop == 0
    assert [10 * d for d in info["delays"]] == durations


def test_reader_sees_no_loop_block_without_loop():
    data = pil_gif([np.zeros((4, 4, 3), np.uint8), np.full((4, 4, 3), 200, np.uint8)], duration=100)
    assert read_gif(data)[1]["loop"] is None


@pytest.mark.parametrize("H,W", [(1, 1), (1, 65536), (1, 65537), (7, 13), (384, 640), (768, 1280), (65535, 3)])
def test_segment_plan_covers_the_frame(H, W):
    plan = gif.segment_plan(H, W)
    assert plan[0][0] == 0 and sum(n for _, n in plan) == H * W
    assert all(s + n == t for (s, n), (t, _) in zip(plan, plan[1:]))
    assert all(n == gif.SEGMENT for _, n in plan[:-1]) and 0 < plan[-1][1] <= gif.SEGMENT


@pytest.mark.parametrize("bits", [[27], [9, 12, 31], [100] * 50, [8 * 4097 + 3, 5, 12 * 8192]])
def test_bit_offsets_are_an_exclusive_scan(bits):
    offs, nbytes = gif.bit_offsets(bits)
    acc = 0
    for b, o in zip(bits, offs.tolist()):
        assert o == acc
        acc += b
    assert nbytes == -(-acc // 8)


@pytest.mark.parametrize("n", [1, 254, 255, 256, 510, 511, 65536, 1_000_003])
def test_subblock_framing_size(n):
    blocks = [min(255, n - s) for s in range(0, n, 255)]
    assert gif.subblock_bytes(n) == n + len(blocks) + 1
    assert all(0 < b <= 255 for b in blocks)


def _stream_gif(idx, H, W, palette):
    """A one-frame GIF around the host restatement's LZW data, framed as csrc/gif.cu frames it."""
    data = encode_frame_data(idx)
    out = bytearray(b"GIF89a" + W.to_bytes(2, "little") + H.to_bytes(2, "little") + bytes([0x70, 0, 0]))
    out += b"\x21\xf9\x04\x00\x0a\x00\x00\x00"
    out += b"\x2c\0\0\0\0" + W.to_bytes(2, "little") + H.to_bytes(2, "little") + b"\x87"
    out += palette.astype(np.uint8).tobytes() + b"\x08"
    for s in range(0, len(data), 255):
        out += bytes([len(data[s:s + 255])]) + data[s:s + 255]
    out += b"\x00\x3b"
    assert len(out) == 13 + 8 + 10 + 768 + 1 + gif.subblock_bytes(len(data)) + 1
    return bytes(out)


@pytest.mark.parametrize("case", ["noise", "runs", "two_values", "full_table", "odd"])
def test_segmented_lzw_decodes_with_pil(case):
    """The segment scheme (post-clear start, closing CLEAR at the segment's own width, EOI last, CLEAR at 12 bits when the
    table fills) decodes with PIL and with gif_ref across segment boundaries."""
    g = np.random.RandomState(11)
    H, W = {"noise": (200, 700), "runs": (256, 513), "two_values": (300, 300), "full_table": (2, 35000),
            "odd": (3, 21846)}[case]
    n = H * W
    if case == "noise":
        idx = g.randint(0, 256, n)
    elif case == "runs":
        idx = np.repeat(g.randint(0, 256, n // 37 + 1), 37)[:n]
    elif case == "two_values":
        idx = g.randint(0, 2, n) * 255
    elif case == "full_table":
        idx = g.randint(0, 256, n)
    else:
        idx = np.arange(n) % 7
    idx = idx.astype(np.uint8)
    if case == "full_table":
        codes = lzw_segment(idx[:gif.SEGMENT], True, False)
        assert sum(1 for c, w in codes[1:-1] if c == 256 and w == 12) >= 1
    palette = np.stack([np.arange(256), 255 - np.arange(256), (np.arange(256) * 7) % 256], 1)
    data = _stream_gif(idx, H, W, palette)
    want = palette[idx].reshape(H, W, 3).astype(np.uint8)
    assert np.array_equal(read_gif(data)[0][0], want)
    assert np.array_equal(np.asarray(Image.open(io.BytesIO(data)).convert("RGB")), want)


@pytest.mark.parametrize("n,offset", [(0, 0), (1, 0), (7, 3), (4096, 1), (3 << 20, 5)])
def test_native_crc32c_matches_tensorboard(n, offset):
    from tensorboard.compat.tensorflow_stub.pywrap_tensorflow import masked_crc32c
    data = np.random.RandomState(n).randint(0, 256, n + offset).astype(np.uint8).tobytes()[offset:]
    assert tboard.masked_crc32c(data) == masked_crc32c(data)


def test_native_crc32c_continues_a_crc():
    from p2pvg_b200._lib import crc32c
    a, b = b"event header", os.urandom(1000)
    assert crc32c(b, crc32c(a)) == crc32c(a + b)


def test_encode_gif_rejects_bad_input():
    import torch
    with pytest.raises(ValueError, match="rule"):
        gif.encode_gif([], rule="jpeg")
    with pytest.raises(ValueError, match="delay_cs"):
        gif.encode_gif([], delay_cs=70000)
    with pytest.raises(ValueError, match="loop"):
        gif.encode_gif([], loop=-1)
    assert gif.encode_gif([]) == []
    with pytest.raises(ValueError, match="CUDA"):
        gif.encode_gif([torch.zeros(2, 4, 4, 3, dtype=torch.uint8)])


def test_save_gif_passes_other_input_to_imageio(monkeypatch, tmp_path):
    calls = []
    monkeypatch.setitem(sys.modules, "imageio", types.SimpleNamespace(
        mimsave=lambda name, frames, **kw: calls.append((name, len(frames), kw))))
    frames = [np.zeros((4, 4), np.uint8)] * 3   # grey frames: imageio's
    gif.save_gif(str(tmp_path / "a.gif"), frames)
    gif.save_gif(str(tmp_path / "b.gif"), [np.zeros((4, 4, 3), np.uint8)] * 2, duration=0.5)
    assert calls == [(str(tmp_path / "a.gif"), 3, {}), (str(tmp_path / "b.gif"), 2, {"duration": 0.5})]


def test_dropin_vis_seq_passes_the_gpu_gif_writer(monkeypatch, dropin):
    import misc.visualize as dv
    seen = {}
    monkeypatch.setattr(dv._fast, "check_vis_seq", lambda *a, **k: None)
    monkeypatch.setattr(dv._fast, "vis_seq", lambda *a, **k: seen.update(k))
    dv.vis_seq(None, None, 0, 10)
    assert seen["save_gif"] is gif.save_gif


def test_dropin_writer_defers_videos_it_does_not_take(monkeypatch, tmp_path, dropin):
    """Without a device (or for a 1-channel video) add_video reaches the base writer with its arguments unchanged."""
    import tensorboardX
    Base = [c for c in tensorboardX.SummaryWriter.__mro__ if c.__module__.startswith(("torch.", "tensorboardX."))][-1]
    seen = []
    monkeypatch.setattr(Base, "add_video", lambda self, *a, **k: seen.append((a, k)))
    w = tensorboardX.SummaryWriter(str(tmp_path))
    vid = np.zeros((1, 2, 1, 4, 4), np.float32)
    w.add_video("v", vid, 3, fps=2)
    w.close()
    (a, k), = seen
    assert a[0] == "v" and a[1] is vid and k == dict(global_step=3, fps=2, walltime=None)
