"""A NumPy GIF reader and a host restatement of the encoder's LZW segments, for the tests of p2pvg_b200.gif.

  read_gif(data)      -> (frames [T, H, W, 3] uint8 composited as PIL shows them, info): info holds the per-frame delays
                         (cs), the loop count (None without a NETSCAPE2.0 block), the per-frame index maps, local
                         palettes, LZW minimum code sizes and sub-block lengths, and the logical screen size
  lzw_segment(idx, first, last) -> [(code, width)] of one segment as csrc/gif.cu codes it
  encode_frame_data(idx)        -> the LZW data of a whole frame from its segments, LSB-first, as csrc/gif.cu packs it
"""
import numpy as np

from p2pvg_b200 import gif


def _subblocks(data, p):
    out, sizes = bytearray(), []
    while True:
        n = data[p]
        p += 1
        if n == 0:
            return bytes(out), sizes, p
        sizes.append(n)
        out += data[p:p + n]
        p += n


def lzw_decode(data, min_size, n_pixels):
    clear, eoi = 1 << min_size, (1 << min_size) + 1
    pad = bytes(data) + b"\0\0\0"
    pos, out = 0, bytearray()
    width, nxt, prev = min_size + 1, eoi + 1, None
    table = [bytes([i]) for i in range(clear)] + [b"", b""]
    nbits = 8 * len(data)
    while pos + width <= nbits:
        i = pos >> 3
        code = ((pad[i] | pad[i + 1] << 8 | pad[i + 2] << 16) >> (pos & 7)) & ((1 << width) - 1)
        pos += width
        if code == clear:
            width, nxt, prev = min_size + 1, eoi + 1, None
            del table[eoi + 1:]
            continue
        if code == eoi:
            break
        if prev is None:
            entry = table[code]
        else:
            entry = table[code] if code < nxt else table[prev] + table[prev][:1]
            assert code <= nxt, f"LZW code {code} beyond the table ({nxt})"
            if nxt < 4096:
                table.append(table[prev] + entry[:1])
                nxt += 1
                if nxt == 1 << width and width < 12:
                    width += 1
        out += entry
        prev = code
    assert len(out) >= n_pixels, f"LZW data holds {len(out)} of {n_pixels} pixels"
    return np.frombuffer(bytes(out[:n_pixels]), np.uint8)


def read_gif(data):
    assert data[:6] in (b"GIF89a", b"GIF87a"), data[:6]
    SW, SH, packed = int.from_bytes(data[6:8], "little"), int.from_bytes(data[8:10], "little"), data[10]
    p = 13
    gct = None
    if packed & 0x80:
        n = 2 << (packed & 7)
        gct = np.frombuffer(data[p:p + 3 * n], np.uint8).reshape(n, 3)
        p += 3 * n
    info = dict(width=SW, height=SH, delays=[], loop=None, indices=[], palettes=[], min_sizes=[], block_sizes=[])
    canvas = np.zeros((SH, SW, 3), np.uint8)
    frames, delay, transp = [], 0, None
    while True:
        b = data[p]
        if b == 0x3b:
            break
        if b == 0x21:
            label = data[p + 1]
            body, _, p2 = _subblocks(data, p + 2)
            if label == 0xf9:
                delay = int.from_bytes(body[1:3], "little")
                transp = body[3] if body[0] & 1 else None
            elif label == 0xff and body[:11] == b"NETSCAPE2.0":
                info["loop"] = int.from_bytes(body[12:14], "little")
            p = p2
            continue
        assert b == 0x2c, f"unexpected block 0x{b:02x} at {p}"
        x, y, w, h = (int.from_bytes(data[p + k:p + k + 2], "little") for k in (1, 3, 5, 7))
        flags = data[p + 9]
        assert not flags & 0x40, "interlaced frames are not read"
        p += 10
        pal = gct
        if flags & 0x80:
            n = 2 << (flags & 7)
            pal = np.frombuffer(data[p:p + 3 * n], np.uint8).reshape(n, 3)
            p += 3 * n
        min_size = data[p]
        body, sizes, p = _subblocks(data, p + 1)
        idx = lzw_decode(body, min_size, w * h)
        rgb = pal[idx].reshape(h, w, 3)
        region = canvas[y:y + h, x:x + w]
        keep = np.ones((h, w), bool) if transp is None else idx.reshape(h, w) != transp
        region[keep] = rgb[keep]
        frames.append(canvas.copy())
        info["delays"].append(delay)
        info["indices"].append(idx.reshape(h, w))
        info["palettes"].append(pal)
        info["min_sizes"].append(min_size)
        info["block_sizes"].append(sizes)
        delay, transp = 0, None
    return np.stack(frames), info


def lzw_segment(idx, first, last):
    """[(code, width)] of one segment of 8-bit indices: from the post-clear state (a CLEAR first when ``first``), a CLEAR
    at 12 bits when the table reaches 4096 codes, the closing EOI (``last``) or CLEAR; the width of the j-th code after a
    CLEAR is the bit length of 257 + j, at most 12."""
    out = []
    j = 0

    def emit(c):
        nonlocal j
        out.append((c, min(12, (257 + j).bit_length())))
        j += 1

    if first:
        emit(256)
        j = 0
    table, nxt = {}, 258
    P = int(idx[0])
    for k in idx[1:].tolist():
        c = table.get((P, k))
        if c is not None:
            P = c
            continue
        emit(P)
        table[(P, k)] = nxt
        nxt += 1
        if nxt == 4096:
            emit(256)
            j, table, nxt = 0, {}, 258
        P = k
    emit(P)
    emit(257 if last else 256)
    return out


def encode_frame_data(idx):
    """The LZW data (before sub-block framing) of a frame's index map: its segments' codes packed LSB-first at the bit
    offsets of gif.bit_offsets."""
    idx = np.asarray(idx, np.uint8).reshape(-1)
    plan = gif.segment_plan(1, idx.size)
    segs = [lzw_segment(idx[s:s + n], s == 0, s + n == idx.size) for s, n in plan]
    offs, nbytes = gif.bit_offsets([sum(w for _, w in sg) for sg in segs])
    acc = 0
    for off, sg in zip(offs.tolist(), segs):
        for c, w in sg:
            acc |= c << off
            off += w
    return acc.to_bytes(nbytes, "little")


def frame_stream_bytes(data):
    """The LZW data of each frame of a GIF file (its sub-blocks joined)."""
    out, p = [], 13
    if data[10] & 0x80:
        p += 3 * (2 << (data[10] & 7))
    while data[p] != 0x3b:
        if data[p] == 0x21:
            _, _, p = _subblocks(data, p + 2)
            continue
        flags = data[p + 9]
        p += 10 + (3 * (2 << (flags & 7)) if flags & 0x80 else 0)
        body, _, p = _subblocks(data, p + 1)
        out.append(body)
    return out
