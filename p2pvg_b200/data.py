"""Input pipeline for the train step (SURVEY.md §8f rank 3: "device-side data path").

The reference loop (train.py:212, data/data_utils.py:129-137) does ``x = next(generator); x = x.cuda()`` and then calls the
model, so the H2D copy of a 126 MB batch (T=30, B=256, 64x64) sits on the critical path of every step.
``DevicePrefetcher`` wraps any iterator of host batches: batch i+1 is copied from pinned memory on a side stream while
batch i trains, and is handed out only after the compute stream has been made to wait for its copy.

    for x in DevicePrefetcher(loader, device):      # x: device tensor, time-major like the reference's normalize_data
        losses = model(x, 0, cp_ix)

Moving MNIST needs no host batches at all: ``MovingMNIST`` renders each batch on the device (``p2pvg_moving_mnist``) from
the digits loaded once by ``load_mnist_digits``.

    for x in MovingMNIST(load_mnist_digits(root), batch_size=256, max_seq_len=30, delta_len=5):
        losses = model(x, 0, len(x) - 1)
"""
from __future__ import annotations

import gzip
import os

import numpy as np
import torch

DIGIT_SIZE = 32


def _read_idx_images(path):
    opener = gzip.open if path.endswith(".gz") else open
    with opener(path, "rb") as f:
        raw = f.read()
    if len(raw) < 16 or int.from_bytes(raw[0:4], "big") != 0x803:
        raise ValueError(f"{path}: not an idx3-ubyte image file")
    n, rows, cols = (int.from_bytes(raw[i:i + 4], "big") for i in (4, 8, 12))
    if len(raw) != 16 + n * rows * cols:
        raise ValueError(f"{path}: {len(raw) - 16} bytes of pixels for {n} images of {rows}x{cols}")
    return np.frombuffer(raw, dtype=np.uint8, offset=16).reshape(n, rows, cols)


def load_mnist_digits(root, train=True):
    """MNIST images as uint8 [N, 32, 32]: torchvision's raw files ``<root>/MNIST/raw/{train,t10k}-images-idx3-ubyte[.gz]``,
    each 28x28 digit resized with PIL bilinear, which is what the reference's ``transforms.Scale(32)`` did to the PIL image
    (data/moving_mnist.py:27-35).  Never downloads: missing files raise FileNotFoundError."""
    from PIL import Image
    base = os.path.join(root, "MNIST", "raw", ("train" if train else "t10k") + "-images-idx3-ubyte")
    path = next((p for p in (base, base + ".gz") if os.path.isfile(p)), None)
    if path is None:
        raise FileNotFoundError(f"MNIST images not found: expected {base} or {base}.gz")
    imgs = _read_idx_images(path)
    out = np.empty((len(imgs), DIGIT_SIZE, DIGIT_SIZE), dtype=np.uint8)
    for i, a in enumerate(imgs):
        out[i] = np.asarray(Image.fromarray(a).resize((DIGIT_SIZE, DIGIT_SIZE), Image.BILINEAR))
    return torch.from_numpy(out)


class MovingMNIST:
    """Endless iterator of Moving MNIST training batches rendered on the device: fp32 [T, B, 1, S, S], time-major, what the
    reference's ``get_generator`` yields after ``.permute(1, 0, 2, 3, 4).cuda()[:seq_len]`` (data/data_utils.py:112-122).

    Per batch: ``T = np.random.randint(max_seq_len - 2 * delta_len, max_seq_len + 1)`` from NumPy's global stream, exactly
    where ``get_seq_len()`` is called there (so the stream ``P2PModel.forward`` draws from is unchanged); one ``torch.randint``
    of the trajectory draws on the device from ``generator`` (same distribution as the reference's worker-process NumPy draws,
    other values); one kernel launch into a fresh tensor (a batch handed out is never written again)."""

    def __init__(self, digits, batch_size, max_seq_len, delta_len, image_size=64, num_digits=2, deterministic=False,
                 device="cuda", generator=None):
        from ._lib import kernels_for
        digits = torch.as_tensor(digits)
        if digits.dtype != torch.uint8 or digits.dim() != 3 or tuple(digits.shape[1:]) != (DIGIT_SIZE, DIGIT_SIZE) or len(digits) == 0:
            raise ValueError(f"digits must be a non-empty uint8 tensor [N, 32, 32], got {digits.dtype} {tuple(digits.shape)}")
        if max_seq_len - 2 * delta_len < 1 or delta_len < 0:
            raise ValueError(f"max_seq_len = {max_seq_len}, delta_len = {delta_len}: sequence lengths must be >= 1")
        self.K = kernels_for(device)
        self.device = self.K.device
        self.digits = digits.to(self.device).contiguous()
        self.batch_size, self.max_seq_len, self.delta_len = int(batch_size), int(max_seq_len), int(delta_len)
        self.image_size, self.num_digits, self.deterministic = int(image_size), int(num_digits), bool(deterministic)
        self.generator = generator

    def __iter__(self):
        return self

    def __next__(self):
        T = int(np.random.randint(self.max_seq_len - 2 * self.delta_len, self.max_seq_len + 1))
        B, S, nd = self.batch_size, self.image_size, self.num_digits
        with torch.cuda.device(self.device):
            draws = torch.randint(0, 2 ** 31 - 1, (B, nd, 5 + 4 * T), dtype=torch.int32, device=self.device, generator=self.generator)
            out = torch.empty(T, B, 1, S, S, dtype=torch.float32, device=self.device)
            self.K.moving_mnist(self.digits, draws, out, T, B, S, nd, self.deterministic)
        return out


def _chain_front(first, rest):
    yield first
    yield from rest


class DevicePrefetcher:
    def __init__(self, batches, device, depth: int = 2, early_release: bool = False, copy_streams: int = 1):
        """early_release: the batch handed out is used by exactly ONE train step (``model(x, ...)``) and by nothing after it.
        The CUDA-graph step copies its input into a static buffer first thing and reports that moment, so the slot can be
        refilled while that step still runs (two steps of slack for the H2D copy instead of one).  Leave it off when the
        batch is used again after the step (plots, a second model)."""
        self.early_release = bool(early_release)
        self._handout = 0
        self.it = iter(batches)
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("DevicePrefetcher copies to a CUDA device")
        # copy_streams > 1 splits every batch into that many pieces, each copied on its own stream (some hosts reach the link rate
        # only with several DMA transfers in flight)
        self.copy_streams = [torch.cuda.Stream(self.device) for _ in range(max(1, int(copy_streams)))]
        self.copy_stream = self.copy_streams[0]
        self.depth = max(2, int(depth))
        self.slots = [None] * self.depth      # device buffers, reused round-robin
        self.free_ev = [None] * self.depth    # compute-stream event: the slot's previous consumer has been enqueued
        self.pinned = [None] * self.depth
        self.copied_ev = [None] * self.depth  # copy-stream event: the slot's last H2D copy (reads the pinned staging buffer)
        self.n = 0
        self.queue = []
        self._pending_release = None
        self._fill()

    def _issue(self):
        try:
            host = next(self.it)
        except StopIteration:
            return False
        k = self.n % self.depth
        if k == self._pending_release:
            self.it = _chain_front(host, self.it)   # slot still in use by the un-released batch: retry later
            return False
        self.n += 1
        if not host.is_pinned():  # page-locked staging buffer (reused); pinned inputs are copied from directly
            for ev in self.copied_ev[k] or ():
                ev.synchronize()   # the previous copy out of this staging buffer must have finished
            if self.pinned[k] is None or self.pinned[k].shape != host.shape or self.pinned[k].dtype != host.dtype:
                self.pinned[k] = torch.empty(host.shape, dtype=host.dtype, pin_memory=True)
            self.pinned[k].copy_(host)
            host = self.pinned[k]
        if self.slots[k] is None or self.slots[k].shape != host.shape or self.slots[k].dtype != host.dtype:
            self.slots[k] = torch.empty(host.shape, dtype=host.dtype, device=self.device)
        n = len(self.copy_streams) if host.is_contiguous() and host.numel() >= (1 << 20) else 1
        src, dst = (host.view(-1).chunk(n), self.slots[k].view(-1).chunk(n)) if n > 1 else ((host,), (self.slots[k],))
        ready = []
        for st, h, d in zip(self.copy_streams, src, dst):
            with torch.cuda.stream(st):
                if self.free_ev[k] is not None:
                    st.wait_event(self.free_ev[k])   # do not overwrite a batch the step may still read
                d.copy_(h, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(st)
                ready.append(ev)
        self.copied_ev[k] = ready
        self.queue.append((k, ready))
        return True

    def _fill(self):
        while len(self.queue) < self.depth - 1 and self._issue():
            pass

    def __iter__(self):
        return self

    def __next__(self):
        cur = torch.cuda.current_stream(self.device)
        # everything the caller enqueued since the previous batch was handed out has consumed it: mark its slot
        # re-usable now (an explicit release() after the step does the same earlier)
        self.release()
        if not self.queue:
            self._fill()
            if not self.queue:
                raise StopIteration
        k, ready = self.queue.pop(0)
        for ev in ready:
            cur.wait_event(ev)
        x = self.slots[k]
        # until released, the slot must not be refilled: an un-recorded event would not block the copy stream, so
        # the slot is simply not re-issued before release (depth >= 2 keeps one batch in flight meanwhile)
        self.free_ev[k] = None
        self._pending_release = k
        # a consumer that copies the batch away at once (the CUDA-graph train step: static input buffer) reports the moment
        # through this hook; the slot is then refillable long before the step ends
        self._handout += 1
        if self.early_release:
            x._p2pvg_on_consumed = lambda ev, k=k, tok=self._handout: self._consumed(k, tok, ev)
        elif hasattr(x, "_p2pvg_on_consumed"):
            del x._p2pvg_on_consumed
        self._fill()          # start copying the next batch before the caller blocks on this step's results
        return x

    def _consumed(self, k, tok, ev):
        if self._pending_release == k and self._handout == tok:
            self._pending_release = None
            self.free_ev[k] = ev
            self._fill()

    def release(self):
        """Record that everything enqueued so far on the compute stream has consumed the last batch.  Called
        automatically when the next batch is requested; calling it right after the step lets the refill start earlier."""
        if self._pending_release is None:
            return
        k, self._pending_release = self._pending_release, None
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.device))
        self.free_ev[k] = ev
        self._fill()


def bind_host_to_gpu(index: int):
    """Restrict this process to the CPU cores local to GPU `index` (NVML's ideal CPU affinity), so that pinned staging
    buffers are first-touched on the GPU's NUMA node and the H2D copies run at full PCIe rate.  Returns the previous
    affinity set (to restore with os.sched_setaffinity(0, prev)), or None when nothing was changed."""
    import os
    if not hasattr(os, "sched_setaffinity"):
        return None
    try:
        import pynvml
        pynvml.nvmlInit()
        vis = os.environ.get("CUDA_VISIBLE_DEVICES")
        phys = index
        if vis:
            ent = vis.split(",")[index].strip()
            if ent.isdigit():
                phys = int(ent)
        h = pynvml.nvmlDeviceGetHandleByIndex(phys)
        ncpu = os.cpu_count() or 1
        words = pynvml.nvmlDeviceGetCpuAffinity(h, (ncpu + 63) // 64)
        cpus = {64 * w + b for w, word in enumerate(words) for b in range(64) if (int(word) >> b) & 1}
        prev = os.sched_getaffinity(0)
        cpus &= prev
        if not cpus or cpus == prev:
            return None
        os.sched_setaffinity(0, cpus)
        return prev
    except Exception:
        return None
