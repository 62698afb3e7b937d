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

Weizmann and BAIR are decoded once into a uint8 clip store on the device (``load_weizmann_clips``, ``load_bair_clips``);
``ClipBatches`` then cuts every batch out of it with one ``p2pvg_video_windows`` launch.

    for x in ClipBatches(load_weizmann_clips(root, True, 18, 64), 128, "permutation", seq_len=(10, 18)):
        losses = model(x, 0, len(x) - 1)

Human3.6M poses are uploaded once from the reference dataset's own normalised lists into fp32 stores on the device
(``PoseClips``); ``PoseBatches`` then gathers both outputs of every batch with one ``p2pvg_pose_windows`` launch.

    for x in PoseBatches(PoseClips(d["pose"]["2d"], d["pose"]["3d"], d["camera_view"], 30, 6), 256, (20, 30), (6, 6)):
        losses = model(x, 0, len(x[1]) - 1)
"""
from __future__ import annotations

import gzip
import os
from concurrent.futures import ThreadPoolExecutor

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


class VideoClips:
    """Clips decoded once: ``frames`` uint8 [F, 3, S, S], clip c = ``frames[clip_first[c]:clip_first[c] + clip_len[c]]``.

    With ``paired_flips`` the dataset's entries are 2 * len(names): entry e is clip e >> 1, mirrored left-right when e is odd
    (the order in which ``WeizmannDataset`` appends each clip and its flipped copy); otherwise entry e is clip e.
    ``max_seq_len`` is the window length L every entry is cut to (each clip holds at least L frames)."""

    def __init__(self, frames, clip_first, clip_len, names, paired_flips, max_seq_len):
        self.frames, self.clip_first, self.clip_len = frames, clip_first, clip_len
        self.names, self.paired_flips, self.max_seq_len = list(names), bool(paired_flips), int(max_seq_len)

    def __len__(self):
        return len(self.names) * (2 if self.paired_flips else 1)

    def entry(self, e):
        """(clip name, mirrored) of entry e."""
        return (self.names[e >> 1], bool(e & 1)) if self.paired_flips else (self.names[e], False)

    def to(self, device):
        return VideoClips(self.frames.to(device), self.clip_first.to(device), self.clip_len.to(device), self.names,
                          self.paired_flips, self.max_seq_len)


def _read_frame(path, image_size):
    """One frame as uint8 [3, S, S], what ``ToTensor`` gives the reference before / 255: an RGB frame as is, a mode-L frame
    replicated to the three channels (the reference's broadcasting assignment into its [T, 3, S, S] buffer)."""
    from PIL import Image
    with Image.open(path) as im:
        if im.size != (image_size, image_size):
            raise ValueError(f"{path}: frame is {im.size[0]}x{im.size[1]}, expected {image_size}x{image_size}")
        if im.mode == "RGB":
            return np.asarray(im).transpose(2, 0, 1)
        if im.mode == "L":
            return np.broadcast_to(np.asarray(im), (3, image_size, image_size))
        raise ValueError(f"{path}: image mode {im.mode!r}, expected 'RGB' or 'L'")


def _decode_clips(clips, image_size, device, chunk_frames=4096):
    """clips: [(name, [frame paths])] -> the uint8 store on ``device``, decoded by a thread pool (PIL releases the GIL while it
    decodes) and copied over in chunks, so host memory holds one chunk, not the dataset."""
    if not clips:
        raise ValueError("no clip is long enough for the requested max_seq_len")
    lens = [len(paths) for _, paths in clips]
    paths = [p for _, ps in clips for p in ps]
    S = image_size
    frames = torch.empty((len(paths), 3, S, S), dtype=torch.uint8, device=device)
    buf = np.empty((min(chunk_frames, len(paths)), 3, S, S), dtype=np.uint8)

    def read(i, base):
        buf[i - base] = _read_frame(paths[i], S)

    with ThreadPoolExecutor(max_workers=min(32, os.cpu_count() or 1)) as pool:
        for base in range(0, len(paths), len(buf)):
            n = min(len(buf), len(paths) - base)
            list(pool.map(read, range(base, base + n), [base] * n))
            frames[base:base + n].copy_(torch.from_numpy(buf[:n]))
    first = np.concatenate([[0], np.cumsum(lens)[:-1]])
    return frames, torch.tensor(first, dtype=torch.int64, device=device), torch.tensor(lens, dtype=torch.int32, device=device)


def load_weizmann_clips(data_root, train, max_seq_len, image_size, device="cuda"):
    """``WeizmannDataset`` (data/weizmann.py:34-88) as a ``VideoClips``: identities are the subdirectories of
    ``<data_root>/weizmann``, actions and frames are taken in ``sorted()`` name order, train is frames [0, n * 2 // 3) of each
    action and test the rest, and a split shorter than ``max_seq_len`` is dropped.  Flipped copies are not stored: the kernel
    mirrors odd entries.  Known deviation: the reference takes identities in raw ``os.listdir`` order, which depends on the
    filesystem; here they are sorted, so entry numbers can differ from the reference's while the set of entries is the same.
    Frames must be ``image_size`` square, RGB or L (ValueError naming the file otherwise)."""
    root = os.path.join(data_root, "weizmann")
    clips = []
    for ident in sorted(d for d in os.listdir(root) if os.path.isdir(os.path.join(root, d))):
        for act in sorted(os.listdir(os.path.join(root, ident))):
            names = sorted(os.listdir(os.path.join(root, ident, act)))
            num_train = len(names) * 2 // 3
            lo, hi = (0, num_train) if train else (num_train, len(names))
            if hi - lo < max_seq_len:
                continue
            clips.append((f"{ident}/{act}", [os.path.join(root, ident, act, f) for f in names[lo:hi]]))
    store = _decode_clips(clips, image_size, device)
    return VideoClips(*store, [c[0] for c in clips], paired_flips=True, max_seq_len=max_seq_len)


def load_bair_clips(data_root, train, max_seq_len, image_size, device="cuda"):
    """``BairRobotPush`` (data/bair.py:22-31, 61-69) as a ``VideoClips``: one clip per trajectory directory
    ``<data_root>/bair/processed_data/{train,test}/<d1>/<d2>``, frames ``0.png .. <max_seq_len - 1>.png``.  Known deviation:
    the reference lists d1 and d2 in raw ``os.listdir`` order, which depends on the filesystem; here both are sorted.  Frames
    are not resized: they must already be ``image_size`` square (the reference hard-codes 64 x 64), RGB or L."""
    data_dir = os.path.join(data_root, "bair", "processed_data", "train" if train else "test")
    clips = []
    for d1 in sorted(os.listdir(data_dir)):
        for d2 in sorted(os.listdir(os.path.join(data_dir, d1))):
            traj = os.path.join(data_dir, d1, d2)
            clips.append((f"{d1}/{d2}", [os.path.join(traj, f"{i}.png") for i in range(max_seq_len)]))
    store = _decode_clips(clips, image_size, device)
    return VideoClips(*store, [c[0] for c in clips], paired_flips=False, max_seq_len=max_seq_len)


# BairRobotPush.__len__: a DataLoader epoch over it is 10000 // batch_size batches
BAIR_EPOCH_ITEMS = 10000
SAMPLING = ("permutation", "uniform", "ordered")


class _EpochBatches:
    """What the device batch iterators share with the reference's loop (data/data_utils.py:94-137): per batch,
    ``T = np.random.randint(lo, hi + 1)`` from NumPy's global stream, where the generator calls ``get_seq_len()``; epochs of
    ``epoch_items // batch_size`` batches (drop_last), ``k`` the batch within the current epoch."""

    def __init__(self, batch_size, seq_len, max_seq_len, epoch_items):
        lo, hi = (int(v) for v in seq_len)
        if not 1 <= lo <= hi <= max_seq_len:
            raise ValueError(f"seq_len = ({lo}, {hi}): needs 1 <= lo <= hi <= max_seq_len = {max_seq_len}")
        B = int(batch_size)
        if B < 1:
            raise ValueError(f"batch_size = {B}")
        if epoch_items // B == 0:
            raise ValueError(f"batch_size = {B} exceeds the {epoch_items} items of an epoch: the reference's drop_last loader "
                             "would yield no batch")
        self.batch_size, self.seq_len, self.epoch_batches, self.k = B, (lo, hi), epoch_items // B, 0

    def __iter__(self):
        return self

    def _draw_seq_len(self):
        return int(np.random.randint(self.seq_len[0], self.seq_len[1] + 1))

    def _advance(self):
        self.k = (self.k + 1) % self.epoch_batches


def ordered_schedule(n_entries, batch_size, epoch_items=BAIR_EPOCH_ITEMS):
    """The entries of one epoch of ``ordered`` sampling, batch after batch (int64 [epoch_items // batch_size * batch_size]).
    ``BairRobotPush.get_seq`` walks its trajectories in order and wraps at the end, whatever index it is asked for; each epoch
    of the reference's DataLoader runs in a fresh worker holding a fresh copy of the dataset, so the walk restarts at 0."""
    return torch.arange(epoch_items // batch_size * batch_size) % n_entries


class ClipBatches(_EpochBatches):
    """Endless iterator of fp32 [T, B, 3, S, S] device batches cut from ``clips`` (``p2pvg_video_windows``), time-major like
    the reference's ``get_generator`` after ``.permute(1, 0, 2, 3, 4).cuda()[:seq_len]`` (data/data_utils.py:112-122).

    Per batch, ``T = np.random.randint(lo, hi + 1)`` is drawn from NumPy's global stream, where ``get_generator`` calls
    ``get_seq_len()``.  ``sampling`` picks the entries:
      permutation  ``DataLoader(shuffle=True, drop_last=True)`` over the entries (Weizmann): a device ``randperm`` per epoch,
                   ``len(clips) // B`` batches per epoch, each row's window start drawn on the device (``randint``)
      uniform      entries drawn with replacement, windows start at frame 0 (BAIR train, bair.py:59)
      ordered      entries in order, wrapping at the end, restarting at entry 0 every ``10000 // B`` batches: each epoch's
                   loader worker starts from a fresh copy of the dataset (BAIR test, bair.py:52-57)
    Random draws come from ``generator`` (a CUDA generator) instead of the reference's worker-process NumPy stream: the same
    distributions, other values.  Each batch is a fresh tensor, never written again."""

    def __init__(self, clips, batch_size, sampling, seq_len, device="cuda", generator=None):
        from ._lib import kernels_for
        if sampling not in SAMPLING:
            raise ValueError(f"sampling = {sampling!r}, expected one of {SAMPLING}")
        n = len(clips)
        # a uniform "epoch" is one batch: nothing is drawn per epoch
        items = {"permutation": n, "uniform": int(batch_size), "ordered": BAIR_EPOCH_ITEMS}[sampling]
        super().__init__(batch_size, seq_len, clips.max_seq_len, items)
        self.K = kernels_for(device)
        self.device = self.K.device
        self.clips = clips.to(self.device)
        self.sampling, self.generator = sampling, generator
        self.order = None
        if sampling == "ordered":
            self.order = ordered_schedule(n, self.batch_size).to(self.device, torch.int32)

    def __next__(self):
        T = self._draw_seq_len()
        B, k, c = self.batch_size, self.k, self.clips
        with torch.cuda.device(self.device):
            draws = None
            if self.sampling == "permutation":
                if k == 0:
                    self.order = torch.randperm(len(c), dtype=torch.int32, device=self.device, generator=self.generator)
                draws = torch.randint(0, 2 ** 31 - 1, (B,), dtype=torch.int32, device=self.device, generator=self.generator)
            if self.sampling == "uniform":
                entries = torch.randint(0, len(c), (B,), dtype=torch.int32, device=self.device, generator=self.generator)
            else:
                entries = self.order[k * B:(k + 1) * B]
            out = torch.empty((T, B) + tuple(c.frames.shape[1:]), dtype=torch.float32, device=self.device)
            self.K.video_windows(c.frames, c.clip_first, c.clip_len, entries, draws, c.paired_flips, c.max_seq_len, out)
        self._advance()
        return out


def _check_pose_lengths(lengths, need):
    short = next((e for e, n in enumerate(lengths) if n < need), None)
    if short is not None:
        raise ValueError(f"entry {short}: {lengths[short]} frames, fewer than speed_hi * max_seq_len = {need}: the reference "
                         "would raise from np.random.randint when it draws this entry")


class PoseClips:
    """Human3.6M pose sequences held on the device: ``pose_2d`` fp32 [F, J, 2] and ``pose_3d`` fp32 [F, J, 3]; entry e is
    frames ``seq_first[e] .. seq_first[e] + seq_len[e]`` of both (``lengths``: the same lengths on the host).
    ``camera_view`` (CPU int64) is the dataset's camera-view list, and entry e reports ``camera_view[e]``. ``max_seq_len`` is
    the window length L.

    Built from ``Human36mDataset``'s own normalised float64 lists ``data['pose']['2d' | '3d']`` and ``data['camera_view']``
    (data/human36m/human36m.py:26-65) by a casting upload.  Each value is rounded to fp32 exactly as the reference's
    ``.float()`` of its collated float64 batch rounds it.  The camera-view list is taken as the dataset holds it:
    ``reformat_data`` appends [0, 1, 2, 3] per annotation but keeps one view of the poses, and the length filter does not
    touch it, so it is longer than the entries, and ``__getitem__(e)`` reports its e-th value.

    Raises ValueError naming the entry for arrays that are not [n, J, 2] / [n, J, 3] with one J, for 2d and 3d lengths that
    differ, and for an entry shorter than ``speed_hi * max_seq_len``.  Known deviation: the reference accepts such a short
    entry and raises from ``np.random.randint`` only when it draws it."""

    def __init__(self, pose_2d, pose_3d, camera_view, max_seq_len, speed_hi=1, device="cuda"):
        if len(pose_2d) != len(pose_3d):
            raise ValueError(f"{len(pose_2d)} 2d entries but {len(pose_3d)} 3d entries")
        if len(pose_2d) == 0:
            raise ValueError("no pose entries")
        if len(camera_view) < len(pose_2d):
            raise ValueError(f"{len(camera_view)} camera views for {len(pose_2d)} entries")
        pose_2d, pose_3d = [np.asarray(a) for a in pose_2d], [np.asarray(a) for a in pose_3d]
        J = pose_2d[0].shape[1] if pose_2d[0].ndim == 3 else None
        for e, (a, b) in enumerate(zip(pose_2d, pose_3d)):
            if a.ndim != 3 or b.ndim != 3 or a.shape[1:] != (J, 2) or b.shape[1:] != (J, 3):
                raise ValueError(f"entry {e}: pose arrays {a.shape} and {b.shape}, expected [n, {J}, 2] and [n, {J}, 3]")
            if len(a) != len(b):
                raise ValueError(f"entry {e}: {len(a)} 2d frames but {len(b)} 3d frames")
        self.lengths = [len(a) for a in pose_2d]
        _check_pose_lengths(self.lengths, int(speed_hi) * int(max_seq_len))
        F = sum(self.lengths)
        first = np.concatenate([[0], np.cumsum(self.lengths)[:-1]])
        host_2d, host_3d = torch.empty(F, J, 2), torch.empty(F, J, 3)
        for a, b, f, n in zip(pose_2d, pose_3d, first, self.lengths):
            host_2d[f:f + n] = torch.from_numpy(np.ascontiguousarray(a))     # float64 -> fp32, round to nearest
            host_3d[f:f + n] = torch.from_numpy(np.ascontiguousarray(b))
        self.pose_2d, self.pose_3d = host_2d.to(device), host_3d.to(device)
        self.seq_first = torch.tensor(first, dtype=torch.int64, device=device)
        self.seq_len = torch.tensor(self.lengths, dtype=torch.int32, device=device)
        self.camera_view = torch.as_tensor(np.asarray(camera_view), dtype=torch.int64)
        self.max_seq_len = int(max_seq_len)

    def __len__(self):
        return len(self.lengths)

    def to(self, device):
        out = object.__new__(PoseClips)
        out.__dict__.update(self.__dict__)
        for k in ("pose_2d", "pose_3d", "seq_first", "seq_len"):
            setattr(out, k, getattr(self, k).to(device))
        return out


class PoseBatches(_EpochBatches):
    """Endless iterator of Human3.6M batches ``(pose_2d, pose_3d, camera_view)`` gathered from ``clips``
    (``p2pvg_pose_windows``): fp32 [T, B, J, 2] and [T, B, J, 3] on the device, time-major, and the CPU int64 [B] camera views
    of the rows' entries. This is what the reference's ``get_h36m_generator`` yields (data/data_utils.py:94-109).

    Per batch, ``T = np.random.randint(lo, hi + 1)`` is drawn from NumPy's global stream where ``get_h36m_generator`` calls
    ``get_seq_len()``.  The entries follow ``DataLoader(shuffle=True, drop_last=True)``: a fresh permutation every epoch of
    ``len(clips) // B`` batches.  It is drawn on the host with torch's global CPU generator, from which the reference's
    sampler also seeds itself once per epoch, and uploaded once per epoch, so the camera views are read on the host.  Each
    row's window start and speed are drawn on the device from ``generator`` (a CUDA generator), in place of the reference's
    worker-process NumPy stream: the same distributions, other values.  ``next()`` never waits for the device.  Only the
    constant-speed crop is implemented: the breakpoint / acceleration branch of ``__getitem__`` is never enabled by
    ``load_dataset``.  Each batch is a fresh pair of tensors, never written again."""

    def __init__(self, clips, batch_size, seq_len, speed_range, device="cuda", generator=None):
        from ._lib import kernels_for
        lo, hi = (int(v) for v in speed_range)
        if not 1 <= lo <= hi:
            raise ValueError(f"speed_range = ({lo}, {hi}): needs 1 <= speed_lo <= speed_hi")
        super().__init__(batch_size, seq_len, clips.max_seq_len, len(clips))
        _check_pose_lengths(clips.lengths, hi * clips.max_seq_len)
        self.K = kernels_for(device)
        self.device = self.K.device
        self.clips = clips.to(self.device)
        self.speed_range, self.generator = (lo, hi), generator
        self.order = self.order_host = None

    def __next__(self):
        T = self._draw_seq_len()
        B, k, c = self.batch_size, self.k, self.clips
        J = c.pose_2d.shape[1]
        with torch.cuda.device(self.device):
            if k == 0:
                self.order_host = torch.randperm(len(c))[:self.epoch_batches * B]
                self.order = self.order_host.to(torch.int32).pin_memory().to(self.device, non_blocking=True)
            draws = torch.randint(0, 2 ** 31 - 1, (2, B), dtype=torch.int32, device=self.device, generator=self.generator)
            out_2d = torch.empty((T, B, J, 2), dtype=torch.float32, device=self.device)
            out_3d = torch.empty((T, B, J, 3), dtype=torch.float32, device=self.device)
            self.K.pose_windows(c.pose_2d, c.pose_3d, c.seq_first, c.seq_len, self.order[k * B:(k + 1) * B], draws,
                                self.speed_range, c.max_seq_len, out_2d, out_3d)
        camera_view = c.camera_view[self.order_host[k * B:(k + 1) * B]]
        self._advance()
        return out_2d, out_3d, camera_view


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
