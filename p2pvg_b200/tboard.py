"""TensorBoard histograms computed on the GPU.

The reference's ``train.py`` logs every parameter and its gradient as a TensorBoard histogram every 50 iterations
(``train.py:225-233``): per tensor a device-to-host copy, then ``np.histogram`` over TensorBoard's 1548 default buckets and
``min`` / ``max`` / ``sum`` / ``dot`` on the host.  Here the counts and statistics of all tensors come from one launch of
``p2pvg_histograms`` (``csrc/histogram.cu``) and one device-to-host copy; the host only trims the bucket list and writes the
event records.

- ``histograms(tensors, bins)``: counts and (min, max, num, sum, sum_squares) of many CUDA tensors in one launch.
- ``histogram_fields(counts, stats, edges, max_bins)``: the ``add_histogram_raw`` arguments that ``add_histogram`` would
  have written (TensorBoard's ``make_histogram`` after ``np.histogram``).
- ``add_param_histograms(writer, model, step)``: ``train.py``'s logging block in one launch.
- ``HistogramWriterMixin``: a writer whose ``add_histogram`` takes the GPU path for fp32 / fp64 values and TensorBoard's
  default (or an explicit) edge table; ``dropin/tensorboardX`` puts it under ``train.py``'s ``SummaryWriter``.
- ``add_image_gpu(writer, ...)``: ``add_image`` of a 3-channel float32 / uint8 image with the PNG encoded on the GPU
  (``p2pvg_b200.png``); ``dropin/tensorboardX``'s ``SummaryWriter.add_image`` takes it first.
- ``add_video_gpu(writer, ...)``: ``add_video`` of one 3-channel float32 / uint8 video with the GIF encoded on the GPU
  (``p2pvg_b200.gif``); ``dropin/tensorboardX``'s ``SummaryWriter.add_video`` takes it first.
- ``native_record_crc(file_writer)``: the file writer's event records framed with the library's CRC-32C instead of
  TensorBoard's pure-Python one; the same bytes.

The one visible difference from the host computation: sum and sum_squares are fp64 sums in another order (fixed-size
chunks of each tensor), so they agree with ``values.sum()`` / ``values.dot(values)`` to rounding, not bit for bit.
Buckets, limits, num, min and max are exact.
"""
from __future__ import annotations

import struct

import numpy as np
import torch

from ._lib import F32, crc32c, kernels_for

F64 = 2           # P2PVG_F64
MAX_EDGES = 4096  # the largest edge table p2pvg_histograms takes


def _default_bins():
    # TensorBoard's "tensorflow" buckets, built with the writers' own float64 loop so that every edge is the same double
    v, pos, neg = 1e-12, [], []
    while v < 1e20:
        pos.append(v)
        neg.append(-v)
        v *= 1.1
    return np.array(neg[::-1] + [0] + pos, dtype=np.float64)


DEFAULT_BINS = _default_bins()   # 1549 edges, 774 on each side of 0
DEFAULT_BINS.setflags(write=False)


def check_edges(bins) -> np.ndarray:
    """bins as a contiguous float64 edge table the kernel takes, or ValueError."""
    e = np.ascontiguousarray(np.asarray(bins, dtype=np.float64))
    if e.ndim != 1 or not 2 <= e.size <= MAX_EDGES:
        raise ValueError(f"histogram edges: need a 1-D table of 2..{MAX_EDGES} edges, got shape {e.shape}")
    if not np.all(np.isfinite(e)):
        raise ValueError("histogram edges: every edge must be finite")
    if not np.all(e[1:] > e[:-1]):
        raise ValueError("histogram edges: the edges must be strictly increasing")
    return e


def _check_tensors(tensors):
    tensors = list(tensors)
    if not tensors:
        return tensors, None
    dev = None
    for i, t in enumerate(tensors):
        if not torch.is_tensor(t):
            raise ValueError(f"histograms: input {i} is not a tensor")
        if t.device.type != "cuda":
            raise ValueError(f"histograms: input {i} is on {t.device}, not a CUDA device")
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise ValueError(f"histograms: inputs on {dev} and {t.device}; one launch covers one device")
        if t.dtype not in (torch.float32, torch.float64):
            raise ValueError(f"histograms: input {i} has dtype {t.dtype} (fp32 or fp64 only)")
        if not t.is_contiguous():
            raise ValueError(f"histograms: input {i} is not contiguous")
        if t.numel() == 0:
            raise ValueError(f"histograms: input {i} is empty")
    return tensors, dev


def histograms_device(tensors, bins=DEFAULT_BINS):
    """One launch over the given contiguous fp32 / fp64 CUDA tensors.  Returns (out, n_bins): an int64 device tensor holding
    counts [n, n_bins] followed by the bits of the fp64 stats [n, 5] (min, max, num, sum, sum_squares), stream-ordered on the
    current stream.  ValueError before any launch for input the kernel does not take."""
    edges = check_edges(bins)
    tensors, dev = _check_tensors(tensors)
    n, nb = len(tensors), edges.size - 1
    if n == 0:
        return torch.empty(0, dtype=torch.int64), nb
    segs = np.array([(t.data_ptr(), t.numel(), F64 if t.dtype == torch.float64 else F32) for t in tensors], dtype=np.int64)
    K = kernels_for(dev)
    with torch.cuda.device(dev):
        ws = torch.empty(K.histograms_workspace_bytes(segs, edges.size), dtype=torch.uint8, device=dev)
        out = torch.empty(n * (nb + 5), dtype=torch.int64, device=dev)
        K.histograms(segs, edges, ws, out[:n * nb], out[n * nb:].view(torch.float64))
    return out, nb


def histograms(tensors, bins=DEFAULT_BINS):
    """Per tensor (counts, (min, max, num, sum, sum_squares)): counts is the int64 ``np.histogram(values.astype(np.float64),
    bins=bins)`` count array, the statistics those of the float64 values.  One launch and one device-to-host copy."""
    out, nb = histograms_device(tensors, bins)
    n = len(tensors)
    host = out.cpu().numpy()
    counts = host[:n * nb].reshape(n, nb)
    stats = host[n * nb:].view(np.float64).reshape(n, 5)
    return [(counts[i], (float(s[0]), float(s[1]), int(s[2]), float(s[3]), float(s[4]))) for i, s in enumerate(stats)]


def histogram_fields(counts, stats, edges, max_bins=None):
    """The keyword arguments of ``add_histogram_raw`` (min, max, num, sum, sum_squares, bucket_limits, bucket_counts) that
    ``add_histogram(values, bins=edges, max_bins=max_bins)`` would have recorded, given ``np.histogram``'s counts of the
    values over ``edges`` and their (min, max, num, sum, sum_squares).  TensorBoard's ``make_histogram`` steps: merge runs of
    ``num_bins // max_bins`` buckets when there are more than ``max_bins``, keep the support (from the first to the last
    non-empty bucket) with one empty bucket to its left, and raise ValueError when that leaves nothing."""
    counts = np.asarray(counts, dtype=np.int64).reshape(-1)
    limits = np.asarray(edges, dtype=np.float64).reshape(-1)
    if limits.size != counts.size + 1:
        raise ValueError(f"histogram_fields: {counts.size} counts need {counts.size + 1} edges, got {limits.size}")
    nb = counts.size
    if max_bins is not None and nb > max_bins:
        sub = nb // max_bins
        rem = nb % sub
        if rem:
            counts = np.concatenate([counts, np.zeros(sub - rem, dtype=counts.dtype)])
        counts = counts.reshape(-1, sub).sum(axis=-1)
        limits = np.concatenate([limits[:-1:sub], limits[-1:]])
    # first and last bucket of the support, found as make_histogram finds them (also for the all-empty case)
    cum = np.cumsum(counts > 0)
    start, end = np.searchsorted(cum, [0, cum[-1] - 1], side="right")
    start, end = int(start), int(end) + 1
    counts = counts[start - 1:end] if start > 0 else np.concatenate([np.zeros(1, dtype=counts.dtype), counts[:end]])
    limits = limits[start:end + 1]
    if counts.size == 0 or limits.size == 0:
        raise ValueError("The histogram is empty, please file a bug report.")
    mn, mx, num, sm, sq = stats
    return dict(min=mn, max=mx, num=int(num), sum=sm, sum_squares=sq, bucket_limits=limits.tolist(),
                bucket_counts=counts.tolist())


def param_tensors(model):
    """train.py's tags and tensors, in its order: per parameter with requires_grad its value under name.replace('.', '/'),
    then its gradient under that name + '/grad' when .grad is set."""
    tags, tensors = [], []
    for name, p in model.named_parameters():
        if p.requires_grad:
            name = name.replace('.', '/')
            tags.append(name)
            tensors.append(p.detach())
            if p.grad is not None:
                tags.append(name + '/grad')
                tensors.append(p.grad.detach())
    return tags, tensors


def add_param_histograms(writer, model, global_step, walltime=None):
    """train.py's histogram block (train.py:225-233) with one launch and one device-to-host copy: every parameter with
    requires_grad and every set gradient, with the tags and in the order that block writes them, through
    ``writer.add_histogram_raw`` (tensorboardX and torch.utils.tensorboard share its signature).  The launch is on the
    current stream, behind the training step the model last enqueued."""
    tags, tensors = param_tensors(model)
    for tag, (counts, stats) in zip(tags, histograms(tensors)):
        writer.add_histogram_raw(tag, **histogram_fields(counts, stats, DEFAULT_BINS), global_step=global_step,
                                 walltime=walltime)


def _gpu_input(values):
    """values as a contiguous fp32 / fp64 CUDA tensor when the GPU path takes them, else None."""
    if torch.is_tensor(values):
        t = values.detach()
    elif isinstance(values, np.ndarray):
        if values.dtype not in (np.float32, np.float64):
            return None
        t = torch.from_numpy(np.ascontiguousarray(values))
    else:
        return None
    if t.dtype not in (torch.float32, torch.float64) or t.numel() == 0:
        return None
    if t.device.type != "cuda":
        if t.device.type != "cpu" or not torch.cuda.is_available():
            return None
        t = t.to("cuda")
    return t.contiguous()


def _gpu_edges(bins):
    if isinstance(bins, str):
        return DEFAULT_BINS if bins == "tensorflow" else None
    if np.ndim(bins) != 1:
        return None
    try:
        return check_edges(bins)
    except (ValueError, TypeError):
        return None


class HistogramWriterMixin:
    """Put before a SummaryWriter class: ``add_histogram`` computes the histogram on the GPU when ``values`` is a CUDA tensor
    or an fp32 / fp64 NumPy array or CPU tensor (uploaded), ``bins`` is ``'tensorflow'`` or an edge table the kernel takes,
    and a CUDA device exists, and records it with ``add_histogram_raw``.  Every other call goes to the base class
    unchanged."""

    def add_histogram(self, tag, values, global_step=None, bins='tensorflow', walltime=None, max_bins=None):
        edges = _gpu_edges(bins)
        t = _gpu_input(values) if edges is not None else None
        if t is None:
            return super().add_histogram(tag, values, global_step=global_step, bins=bins, walltime=walltime,
                                         max_bins=max_bins)
        (counts, stats), = histograms([t.view(-1)], edges)
        self.add_histogram_raw(tag, **histogram_fields(counts, stats, edges, max_bins), global_step=global_step,
                               walltime=walltime)


def _gpu_image(img, dataformats):
    """img as a contiguous CUDA [3, H, W] float32 / uint8 tensor when the GPU image path takes it, else None."""
    if dataformats not in ("CHW", "HWC") or not torch.cuda.is_available():
        return None
    if isinstance(img, np.ndarray):
        if img.dtype not in (np.float32, np.uint8):
            return None
        t = torch.from_numpy(np.ascontiguousarray(img))
    elif torch.is_tensor(img):
        t = img.detach()
    else:
        return None
    if t.dtype not in (torch.float32, torch.uint8) or t.dim() != 3 or t.shape[dataformats.index("C")] != 3 or t.numel() == 0:
        return None
    if t.device.type != "cuda":
        if t.device.type != "cpu":
            return None
        t = t.to("cuda")
    if dataformats == "HWC":
        t = t.permute(2, 0, 1)
    t = t.contiguous()
    if t.dtype == torch.float32 and bool(torch.isnan(t).any()):
        return None
    return t


def add_image_gpu(writer, tag, img_tensor, global_step=None, walltime=None, dataformats='CHW'):
    """``writer.add_image`` of a 3-channel float32 or uint8 image (CHW or HWC, a NumPy array or a tensor) with the PNG
    encoded on the GPU, when a CUDA device exists: the base writer's quantisation (float32: x * 255 clipped to [0, 255]
    and truncated; uint8 as it is) and the same ``Summary.Image`` record (tag, step, height, width, colorspace), written
    through ``writer._get_file_writer()``.  The pixels equal the base writer's; the compressed bytes differ.  Returns
    False, having written nothing, for any other call and for float input with NaN."""
    t = _gpu_image(img_tensor, dataformats)
    if t is None:
        return False
    from . import png
    data, = png.encode_png([t], "tensorboard")
    Summary = _summary_class(writer)
    image = Summary.Image(height=int(t.shape[1]), width=int(t.shape[2]), colorspace=3, encoded_image_string=data)
    writer._get_file_writer().add_summary(Summary(value=[Summary.Value(tag=tag, image=image)]), global_step, walltime)
    return True


def _gpu_video(vid):
    """vid as a CUDA [T, 3, H, W] float32 / uint8 tensor when the GPU video path takes it (one video of 3 channels, sides
    in 1..65535, no NaN), else None."""
    from .gif import MAX_SIDE
    if not torch.cuda.is_available():
        return None
    if isinstance(vid, np.ndarray):
        if vid.dtype not in (np.float32, np.uint8):
            return None
        t = torch.from_numpy(np.ascontiguousarray(vid))
    elif torch.is_tensor(vid):
        t = vid.detach()
    else:
        return None
    if t.dtype not in (torch.float32, torch.uint8) or t.dim() != 5 or t.shape[0] != 1 or t.shape[2] != 3:
        return None
    if not all(1 <= int(v) <= MAX_SIDE for v in (t.shape[1], t.shape[3], t.shape[4])):
        return None
    if t.device.type != "cuda":
        if t.device.type != "cpu":
            return None
        t = t.to("cuda")
    t = t[0]
    if t.dtype == torch.float32 and bool(torch.isnan(t).any()):
        return None
    return t


def add_video_gpu(writer, tag, vid_tensor, global_step=None, fps=4, walltime=None):
    """``writer.add_video`` of one video (N = 1) of 3 channels, float32 or uint8, a NumPy array or a tensor [1, T, 3, H, W],
    with the GIF encoded on the GPU, when a CUDA device exists: the base writer's quantisation (float32: x * 255 clipped to
    [0, 255] and truncated; uint8 as it is), every frame shown round(100 / fps) centiseconds, looping forever (moviepy's
    ``write_gif`` defaults), and the base writer's ``Summary.Image`` record (tag, step, height, width, colorspace 3),
    written through ``writer._get_file_writer()``.  A frame of at most 256 colours decodes to the quantised pixels; others
    carry a 256-colour palette (``p2pvg_b200.gif``).  Returns False, having written nothing, for any other call, for float
    input with NaN and for an fps whose delay does not fit the GIF field."""
    from . import gif
    try:
        delay = round(100 / fps)
    except (TypeError, ZeroDivisionError):
        return False
    if not 0 <= delay <= gif.MAX_SIDE:
        return False
    t = _gpu_video(vid_tensor)
    if t is None:
        return False
    frames = t.contiguous() if t.dtype == torch.float32 else t.permute(0, 2, 3, 1).contiguous()
    data, = gif.encode_gif([frames], "tensorboard", delay_cs=int(delay), loop=0)
    Summary = _summary_class(writer)
    image = Summary.Image(height=int(t.shape[2]), width=int(t.shape[3]), colorspace=3, encoded_image_string=data)
    writer._get_file_writer().add_summary(Summary(value=[Summary.Value(tag=tag, image=image)]), global_step, walltime)
    return True


def masked_crc32c(data):
    """TensorBoard's masked CRC-32C of the bytes ``data``, with the library's CRC-32C."""
    x = crc32c(data)
    return (((x >> 15) | (x << 17)) + 0xa282ead8) & 0xffffffff


def _record_writer(file_writer):
    """The RecordWriter under a torch.utils.tensorboard / tensorboard file writer (event_writer._async_writer._writer), or
    None for any other layout."""
    rw = getattr(getattr(getattr(file_writer, "event_writer", None), "_async_writer", None), "_writer", None)
    if rw is None or type(rw).__name__ != "RecordWriter" or not hasattr(rw, "_writer"):
        return None
    return rw


def native_record_crc(file_writer):
    """Frame the file writer's event records with ``masked_crc32c`` above: its RecordWriter instance's ``write`` becomes one
    that writes the same bytes (length, masked CRC of the length, the record, masked CRC of the record).  The module-level
    ``masked_crc32c`` of tensorboard and every other writer stay as they are; a writer of another layout is left alone."""
    rw = _record_writer(file_writer)
    if rw is None or "write" in vars(rw):
        return
    out = rw._writer

    def write(data):
        header = struct.pack("<Q", len(data))
        out.write(header + struct.pack("<I", masked_crc32c(header)) + data + struct.pack("<I", masked_crc32c(data)))

    rw.write = write


def _summary_class(writer):
    """The Summary protobuf class of the writer's base package (the ``summary`` module beside the module of the first base
    class that defines add_image: torch.utils.tensorboard or tensorboardX)."""
    import importlib
    for cls in type(writer).__mro__[1:]:
        if "add_image" in vars(cls):
            return importlib.import_module(cls.__module__.rsplit(".", 1)[0] + ".summary").Summary
    raise TypeError("add_image_gpu needs a SummaryWriter")
