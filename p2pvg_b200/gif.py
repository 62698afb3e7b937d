"""GIF animations encoded on the GPU, for the reference's ``vis_seq`` GIF files and TensorBoard video summaries.

``p2pvg_gif_encode`` (``csrc/gif.cu``) turns a batch of animations into complete GIF89a files in one call: quantisation,
each frame's colour set and 256-entry local palette, the index map, LZW in independent segments of ``SEGMENT`` pixels,
the bit packing and the data sub-blocks, all on the device.  The host reads the file sizes and copies the packed files once.

- ``encode_gif(animations, rule, delay_cs, loop)``: the GIF bytes of many CUDA animations in one call.
- ``save_gif(name, frames)``: ``imageio.mimsave(name, frames)`` for uint8 [T, H, W, 3] frames, encoded on the GPU.

Palette rule: a frame of at most 256 distinct colours keeps exactly those (the frame decodes to its pixels); a frame of more
gets median cut to 256 boxes and 3 Lloyd iterations over its distinct colours, every pixel its nearest entry.  Neither
Pillow's nor moviepy's palette is reproduced bit for bit.
"""
from __future__ import annotations

import numpy as np
import torch

from ._lib import F32, kernels_for
from .png import RULES, U8

SEGMENT = 65536          # P2PVG_GIF_SEGMENT: pixels per LZW segment
DELAY_CS = 10            # imageio 2.x's GIF writer: fps=10
LOOP = 0                 # forever
MAX_SIDE = 65535         # T, H and W, and the delay and loop fields


def segment_plan(H, W):
    """(start, length) of each LZW segment of an H x W frame's pixels, in order."""
    n = H * W
    return [(s, min(SEGMENT, n - s)) for s in range(0, n, SEGMENT)]


def segment_codes_bound(length):
    """The most codes a segment of ``length`` pixels emits: one per pixel, a CLEAR per 3838 codes when the table fills,
    the closing CLEAR or EOI and the stream's opening CLEAR."""
    return length + length // 3838 + 3


def bit_offsets(bits):
    """Each segment's first bit in its frame's code stream (an exclusive scan of the segments' bit lengths) and the
    frame's byte count: segments are packed LSB-first back to back, sharing their boundary bytes."""
    off = np.concatenate([[0], np.cumsum(np.asarray(bits, dtype=np.int64))])
    return off[:-1], int((off[-1] + 7) // 8)


def subblock_bytes(n):
    """Bytes of n bytes of image data framed as GIF data sub-blocks: a length byte per 255 bytes, then the 0 terminator."""
    return n + (n + 254) // 255 + 1


def _frames_of(t, i):
    if not torch.is_tensor(t) or t.device.type != "cuda":
        raise ValueError(f"encode_gif: animation {i} is not a CUDA tensor")
    if t.dtype == torch.uint8:
        ok = t.dim() == 4 and t.shape[3] == 3
        T, H, W = (t.shape[:3] if ok else (0, 0, 0))
    elif t.dtype == torch.float32:
        ok = t.dim() == 4 and t.shape[1] == 3
        T, H, W = ((t.shape[0], t.shape[2], t.shape[3]) if ok else (0, 0, 0))
    else:
        raise ValueError(f"encode_gif: animation {i} has dtype {t.dtype} (uint8 [T, H, W, 3] or float32 [T, 3, H, W])")
    if not ok:
        raise ValueError(f"encode_gif: animation {i} has shape {tuple(t.shape)}: uint8 frames are [T, H, W, 3], float32 "
                         f"frames [T, 3, H, W]")
    if not all(1 <= int(v) <= MAX_SIDE for v in (T, H, W)):
        raise ValueError(f"encode_gif: animation {i} is {int(T)} frames of {int(H)} x {int(W)} (1..{MAX_SIDE} each)")
    if not t.is_contiguous():
        raise ValueError(f"encode_gif: animation {i} is not contiguous")
    return int(T), int(H), int(W)


def encode_gif(animations, rule="tensorboard", delay_cs=DELAY_CS, loop=LOOP):
    """The GIF files (bytes) of a list of contiguous CUDA animations -- uint8 [T, H, W, 3] or float32 [T, 3, H, W], each its
    own size -- from one p2pvg_gif_encode call on the current stream, one device-to-host copy of the sizes and one of the
    files.  float32 frames are quantised with ``rule`` as ``png.encode_png`` quantises ("tensorboard": trunc(clamp(x * 255,
    0, 255)); "save_image" rounds); NaN is outside the contract.  Every frame shows for ``delay_cs`` centiseconds; ``loop``
    is the NETSCAPE2.0 loop count (0: forever).  ValueError before any launch for input the encoder does not take."""
    if rule not in RULES:
        raise ValueError(f"encode_gif: rule {rule!r} (one of {sorted(RULES)})")
    for name, v in (("delay_cs", delay_cs), ("loop", loop)):
        if not isinstance(v, (int, np.integer)) or not 0 <= v <= MAX_SIDE:
            raise ValueError(f"encode_gif: {name} {v!r} is not an integer in 0..{MAX_SIDE}")
    animations = list(animations)
    if not animations:
        return []
    dev, rows = None, []
    for i, t in enumerate(animations):
        T, H, W = _frames_of(t, i)
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise ValueError(f"encode_gif: animations on {dev} and {t.device}; one call covers one device")
        rows.append((t.data_ptr(), F32 if t.dtype == torch.float32 else U8, T, H, W, int(delay_cs), int(loop)))
    table = np.array(rows, dtype=np.int64)
    K = kernels_for(dev)
    ws_bytes, out_bytes = K.gif_bytes(table)
    if ws_bytes == 0:
        raise ValueError("encode_gif: too many pixels or frames for one call")
    with torch.cuda.device(dev):
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        out = torch.empty(out_bytes, dtype=torch.uint8, device=dev)
        files = torch.empty(len(animations), 2, dtype=torch.int64, device=dev)
        K.gif_encode(table, RULES[rule], ws, out, files)
        fl = files.cpu().numpy()
        total = int(fl[-1, 0] + fl[-1, 1])
        host = torch.empty(total, dtype=torch.uint8, pin_memory=True)
        host.copy_(out[:total])
    buf = host.numpy().tobytes()
    return [buf[o:o + s] for o, s in fl.tolist()]


def _gpu_frames(frames):
    """frames as a contiguous uint8 CUDA [T, H, W, 3] tensor when save_gif's GPU path takes them, else None."""
    if torch.is_tensor(frames):
        t = frames.detach()
        if t.device.type != "cuda":
            return None
    elif isinstance(frames, (list, tuple, np.ndarray)) and len(frames) and torch.cuda.is_available():
        if not all(isinstance(f, np.ndarray) and f.dtype == np.uint8 for f in frames):
            return None
        if len({f.shape for f in frames}) != 1:
            return None
        t = torch.from_numpy(np.ascontiguousarray(np.stack(list(frames)))).cuda()
    else:
        return None
    if t.dtype != torch.uint8 or t.dim() != 4 or t.shape[3] != 3 or not all(1 <= int(v) <= MAX_SIDE for v in t.shape[:3]):
        return None
    return t.contiguous()


def save_gif(name, frames, **kwargs):
    """``imageio.mimsave(name, frames)`` with the GIF encoded on the GPU, for uint8 [T, H, W, 3] frames given as a CUDA
    tensor or as a list or array of NumPy frames (uploaded).  The file shows every frame for 10 centiseconds and loops
    forever: the defaults of imageio 2.x's GIF writer (``fps=10``, ``loop=0``) in the reference's era.  Any other input,
    and any call with keyword arguments, goes to ``imageio.mimsave`` unchanged."""
    t = None if kwargs else _gpu_frames(frames)
    if t is None:
        import imageio
        return imageio.mimsave(name, frames, **kwargs)
    data, = encode_gif([t], delay_cs=DELAY_CS, loop=LOOP)
    with open(name, "wb") as f:
        f.write(data)
