"""A PNG reader in NumPy, independent of PIL and of the encoder under test, and the synthetic pictures the PNG tests and
tools/bench_png.py encode.

read_png parses every chunk and checks its CRC-32 with zlib.crc32, inflates the joined IDAT data with zlib, checks the
Adler-32 at its end against zlib.adler32 of the inflated stream, and undoes the five row filters.  The filters are undone
along anti-diagonals (pixel (y, x) needs only (y, x - 1), (y - 1, x) and (y - 1, x - 1)), so a 3840 x 1920 picture takes
H + W vectorised steps."""
import os
import struct
import zlib

import numpy as np
import torch

SIG = b"\x89PNG\r\n\x1a\n"
BPP = {0: 1, 2: 3, 4: 2, 6: 4}   # 8-bit grey, RGB, grey + alpha, RGBA


def chunks(data):
    """[(type, payload)] of a PNG file; AssertionError on a bad signature, length or CRC."""
    assert data[:8] == SIG, "not a PNG signature"
    out, i = [], 8
    while i < len(data):
        n, = struct.unpack(">I", data[i:i + 4])
        typ, body = data[i + 4:i + 8], data[i + 8:i + 8 + n]
        assert len(body) == n, "truncated chunk"
        crc, = struct.unpack(">I", data[i + 8 + n:i + 12 + n])
        assert crc == zlib.crc32(typ + body) & 0xffffffff, f"bad CRC on {typ!r}"
        out.append((typ.decode("ascii"), body))
        i += 12 + n
    assert out[0][0] == "IHDR" and out[-1] == ("IEND", b""), "IHDR first and an empty IEND last"
    return out


def unfilter(raw, H, W, bpp):
    """Pixels uint8 [H, W, bpp] of a filtered stream (per row a filter byte 0-4 and W * bpp bytes)."""
    a = np.frombuffer(raw, dtype=np.uint8)
    assert a.size == H * (1 + W * bpp), "stream length"
    a = a.reshape(H, 1 + W * bpp)
    ft = a[:, 0].astype(np.int64)
    assert ft.max(initial=0) <= 4, "unknown filter type"
    res = a[:, 1:].reshape(H, W, bpp).astype(np.int64)
    out = np.zeros((H + 1, W + 1, bpp), np.int64)    # a zero row above and a zero column to the left
    for k in range(H + W - 1):
        ys = np.arange(max(0, k - W + 1), min(H - 1, k) + 1)
        xs = k - ys
        A, B, C = out[ys + 1, xs], out[ys, xs + 1], out[ys, xs]
        p = A + B - C
        pa, pb, pc = np.abs(p - A), np.abs(p - B), np.abs(p - C)
        paeth = np.where((pa <= pb) & (pa <= pc), A, np.where(pb <= pc, B, C))
        f = ft[ys][:, None]
        pred = np.select([f == 0, f == 1, f == 2, f == 3], [np.zeros_like(A), A, B, (A + B) // 2], paeth)
        out[ys + 1, xs + 1] = (res[ys, xs] + pred) & 255
    return out[1:, 1:].astype(np.uint8)


def read_png(data):
    """(pixels uint8 [H, W, channels], info) of an 8-bit, non-interlaced PNG; info holds the IHDR fields, the IDAT count
    and the zlib header."""
    ch = chunks(data)
    W, H, depth, ctype, comp, filt, inter = struct.unpack(">IIBBBBB", ch[0][1])
    assert depth == 8 and comp == 0 and filt == 0 and inter == 0 and ctype in BPP, "8-bit, non-interlaced only"
    idat = [b for t, b in ch if t == "IDAT"]
    z = b"".join(idat)
    d = zlib.decompressobj()
    raw = d.decompress(z) + d.flush()
    assert d.eof and not d.unused_data, "the zlib stream ends with the last IDAT"
    assert struct.unpack(">I", z[-4:])[0] == zlib.adler32(raw) & 0xffffffff, "Adler-32"
    px = unfilter(raw, H, W, BPP[ctype])
    return px, dict(W=W, H=H, ctype=ctype, n_idat=len(idat), zlib_header=z[:2], filters=raw[::1 + W * BPP[ctype]])


# -- pictures -----------------------------------------------------------------------------------------------------------
DIGITS = os.path.join(os.path.dirname(__file__), "golden", "mmnist_digits.pt")


def _border(frame, t, n):
    frame[:, :3], frame[:, -3:], frame[:, :, :3], frame[:, :, -3:] = 0, 0, 0, 0
    if t == 0:
        col = (1.0, 165 / 255, 0.0)
    elif t == n - 1:
        col = (1.0, 0.0, 0.0)
    else:
        return
    for c in range(3):
        frame[c, :3], frame[c, -3:], frame[c, :, :3], frame[c, :, -3:] = col[c], col[c], col[c], col[c]


def mnist_canvas(rows=60, cols=30, size=64, seed=0):
    """A vis_seq-like canvas [3, rows * size, cols * size] of grey digits moving over black frames, orange borders on the
    first frame of each row and red on the last (dcgan_64 Moving MNIST: 10 blocks of 6 rows, 30 frames)."""
    g = np.random.RandomState(seed)
    digits = torch.load(DIGITS, weights_only=False)["digits"].float()
    digits = digits / max(float(digits.max()), 1.0)
    out = torch.zeros(3, rows * size, cols * size)
    for r in range(rows):
        d = digits[g.randint(len(digits))]
        y, x = g.randint(0, size - 32, 2)
        vy, vx = g.randint(-3, 4, 2)
        for t in range(cols):
            f = torch.zeros(3, size, size)
            y, x = min(max(y + vy, 0), size - 32), min(max(x + vx, 0), size - 32)
            f[:, y:y + 32, x:x + 32] = d
            _border(f, t, cols)
            out[:, r * size:(r + 1) * size, t * size:(t + 1) * size] = f
    return out


def rgb_canvas(rows=60, cols=30, size=64, seed=0):
    """A canvas of smooth colour frames with sensor-like noise and the same borders (vgg_64 on natural video)."""
    g = torch.Generator().manual_seed(seed)
    out = torch.zeros(3, rows * size, cols * size)
    for r in range(rows):
        base = torch.rand(1, 3, 6, 6, generator=g)
        for t in range(cols):
            drift = 0.05 * torch.randn(1, 3, 6, 6, generator=g)
            f = torch.nn.functional.interpolate(base + drift, size=(size, size), mode="bilinear", align_corners=False)[0]
            f = (f + 0.02 * torch.randn(3, size, size, generator=g)).clamp(0, 1)
            _border(f, t, cols)
            out[:, r * size:(r + 1) * size, t * size:(t + 1) * size] = f
    return out
