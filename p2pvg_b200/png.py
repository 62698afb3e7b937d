"""PNG files encoded on the GPU, pixel-identical to ``torchvision.utils.save_image`` and TensorBoard's image summaries.

``p2pvg_png_encode`` (``csrc/png.cu``) turns a batch of fp32 or uint8 images into complete PNG files (8-bit RGB) in one
call: quantisation with the writer's rounding rule, libpng's per-row filter choice, deflate in segments of ``SEGMENT``
filtered bytes with one CTA each, the zlib framing and every chunk CRC, all on the device.  The host reads the file sizes
and copies the packed files once.

- ``encode_png(images, rule)``: the PNG bytes of many CUDA images in one call.
- ``save_image(tensor, fp, **kw)``: ``torchvision.utils.save_image`` with the encoding on the GPU for finite fp32 CUDA
  input and a PNG destination; any other call is torchvision's, unchanged.

A file decodes to exactly the pixels torchvision's (or TensorBoard's) writer stores; the compressed bytes differ.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from ._lib import F32, kernels_for

U8 = 3                                         # P2PVG_PNG_U8
RULES = {"save_image": 0, "tensorboard": 1}    # P2PVG_PNG_SAVE_IMAGE, P2PVG_PNG_TENSORBOARD
SEGMENT = 65536                                # P2PVG_PNG_SEGMENT: filtered bytes per deflate segment and IDAT chunk
ADLER_MOD = 65521


def stream_bytes(H, W):
    """Bytes of the filtered stream of an H x W RGB image: per row a filter byte and 3 W residuals."""
    return H * (1 + 3 * W)


def segment_plan(H, W):
    """(start, length) of each deflate segment of an H x W image's filtered stream, in order; one IDAT chunk each."""
    n = stream_bytes(H, W)
    return [(s, min(SEGMENT, n - s)) for s in range(0, n, SEGMENT)]


def adler32_parts(data):
    """The parts one segment contributes to the Adler-32 of the stream: (sum of its bytes, sum over its bytes of (bytes
    from there to the segment's end) * byte), both exact."""
    d = np.frombuffer(bytes(data), dtype=np.uint8).astype(np.int64)
    return int(d.sum()), int((d * np.arange(d.size, 0, -1, dtype=np.int64)).sum())


def adler32_combine(parts, lengths):
    """The Adler-32 of the concatenation of segments, from their adler32_parts and lengths, as the encoder's last CTA of
    an image combines them: a = 1 + sum S_k, b = N + sum (W_k + (bytes after segment k) * S_k), mod 65521."""
    N = sum(lengths)
    a, b, after = 1, N % ADLER_MOD, N
    for (s, w), n in zip(parts, lengths):
        after -= n
        a = (a + s) % ADLER_MOD
        b = (b + w + after * s) % ADLER_MOD
    return b << 16 | a


def _image_table(images):
    if not images:
        return None, np.zeros((0, 5), np.int64)
    dev = None
    rows = []
    for i, t in enumerate(images):
        if not torch.is_tensor(t) or t.device.type != "cuda":
            raise ValueError(f"encode_png: image {i} is not a CUDA tensor")
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise ValueError(f"encode_png: images on {dev} and {t.device}; one call covers one device")
        if t.dtype not in (torch.float32, torch.uint8):
            raise ValueError(f"encode_png: image {i} has dtype {t.dtype} (float32 or uint8)")
        if t.dim() != 3 or t.shape[0] not in (1, 3) or t.shape[1] < 1 or t.shape[2] < 1:
            raise ValueError(f"encode_png: image {i} has shape {tuple(t.shape)}, not [C, H, W] with C 1 or 3")
        if not t.is_contiguous():
            raise ValueError(f"encode_png: image {i} is not contiguous")
        rows.append((t.data_ptr(), F32 if t.dtype == torch.float32 else U8, *t.shape))
    return dev, np.array(rows, dtype=np.int64)


def encode_png(images, rule="save_image"):
    """The PNG files (bytes) of a list of contiguous CUDA images [C, H, W] (float32 or uint8, C 1 or 3, each its own size),
    from one p2pvg_png_encode call on the current stream, one device-to-host copy of the sizes and one of the files.  float32
    images are quantised with ``rule``: "save_image" (torchvision.utils.save_image) or "tensorboard"
    (torch.utils.tensorboard's image summary); uint8 images are taken as they are.  NaN values are outside the contract.
    ValueError before any launch for input the encoder does not take."""
    if rule not in RULES:
        raise ValueError(f"encode_png: rule {rule!r} (one of {sorted(RULES)})")
    images = list(images)
    dev, table = _image_table(images)
    if dev is None:
        return []
    K = kernels_for(dev)
    ws_bytes, out_bytes = K.png_bytes(table)
    if ws_bytes == 0:
        raise ValueError("encode_png: an image is too large (2^24 rows or columns or more)")
    with torch.cuda.device(dev):
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        out = torch.empty(out_bytes, dtype=torch.uint8, device=dev)
        files = torch.empty(len(images), 2, dtype=torch.int64, device=dev)
        K.png_encode(table, RULES[rule], ws, out, files)
        fl = files.cpu().numpy()
        total = int(fl[-1, 0] + fl[-1, 1])
        host = torch.empty(total, dtype=torch.uint8, pin_memory=True)
        host.copy_(out[:total])
    buf = host.numpy().tobytes()
    return [buf[o:o + s] for o, s in fl.tolist()]


def _png_destination(fp, format):
    if format is not None:
        return str(format).lower() == "png"
    return isinstance(fp, (str, os.PathLike)) and os.fspath(fp).lower().endswith(".png")


def save_image(tensor, fp, format=None, **kwargs):
    """``torchvision.utils.save_image(tensor, fp, format, **kwargs)``.  The grid is built by torchvision's ``make_grid`` on
    the tensor's device; a finite float32 CUDA grid of 3 channels written as PNG is encoded on the GPU.  Every other input
    (a CPU tensor or list, another dtype, NaN or inf, another format) goes to torchvision's save_image unchanged."""
    import torchvision.utils as vutils
    t = tensor[0] if isinstance(tensor, (list, tuple)) and tensor else tensor
    if torch.is_tensor(t) and t.is_cuda and t.dtype == torch.float32 and _png_destination(fp, format):
        grid = vutils.make_grid(tensor, **kwargs)
        if grid.dim() == 3 and grid.shape[0] == 3 and grid.dtype == torch.float32 and bool(torch.isfinite(grid).all()):
            data, = encode_png([grid.contiguous()], "save_image")
            if isinstance(fp, (str, os.PathLike)):
                with open(fp, "wb") as f:
                    f.write(data)
            else:
                fp.write(data)
            return
    vutils.save_image(tensor, fp, format=format, **kwargs)
