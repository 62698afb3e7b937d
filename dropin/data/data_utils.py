"""Drop-in for the reference's ``data/data_utils.py``: the ``mnist`` branches of ``load_dataset`` and ``get_data_generator``
render Moving MNIST batches on the GPU (``p2pvg_b200.data.MovingMNIST``), the ``weizmann`` and ``bair`` branches cut them
from clips decoded once into device memory (``p2pvg_b200.data.ClipBatches``), and the ``h36m`` branches gather them from pose
sequences uploaded once into device memory (``p2pvg_b200.data.PoseBatches``); every other call is delegated unchanged to the
reference's own module, loaded from the reference's ``data/`` directory.  For Human3.6M, reading ``annot.h5`` and normalising
still happen in the reference's own ``Human36mDataset``, called through its ``load_dataset``.

The generator yields what the reference's ``get_generator`` yields, fp32 [T, B, 1, S, S] on the device, and draws T from
NumPy's global stream at the same point; the digit trajectories are drawn on the device (torch's CUDA generator, seeded by
``train.py``'s ``torch.cuda.manual_seed_all``) instead of in a loader worker process.  MNIST is read from torchvision's raw
files under ``<data_root>/MNIST/raw`` and never downloaded."""
import importlib.util
import os

import numpy as np

import data as _pkg
from p2pvg_b200.data import (ClipBatches, MovingMNIST, PoseBatches, PoseClips, load_bair_clips, load_mnist_digits,
                             load_weizmann_clips)

_here = os.path.dirname(os.path.abspath(__file__))
_ref = None


def _reference():
    global _ref
    if _ref is None:
        for d in _pkg.__path__:
            f = os.path.join(d, "data_utils.py")
            if os.path.abspath(d) != _here and os.path.isfile(f):
                spec = importlib.util.spec_from_file_location("data._reference_data_utils", f)
                mod = importlib.util.module_from_spec(spec)
                spec.loader.exec_module(mod)
                _ref = mod
                break
        else:
            raise ImportError("the reference's data/data_utils.py was not found: set P2PVG_REF to the reference checkout")
    return _ref


def __getattr__(name):
    if name.startswith("__"):
        raise AttributeError(name)
    return getattr(_reference(), name)


class MovingMNISTDigits:
    """Stands in for ``DynamicLengthMovingMNIST`` (data/moving_mnist.py:7-49) wherever ``train.py`` and ``get_generator`` use
    the dataset object; the frames themselves come from ``MovingMNIST``."""

    def __init__(self, data_root, train, max_seq_len, delta_len, image_size, num_digits, deterministic):
        self.data_root, self.train = data_root, train
        self.max_seq_len, self.delta_len, self.image_size = max_seq_len, delta_len, image_size
        self.num_digits, self.deterministic = num_digits, deterministic
        self.channels, self.digit_size = 1, 32
        self.digits = load_mnist_digits(data_root, train=train)
        self.N = len(self.digits)

    def get_seq_len(self):
        return np.random.randint(low=self.max_seq_len - self.delta_len * 2, high=self.max_seq_len + 1)

    def __len__(self):
        return self.N


class VideoClipSet:
    """Stands in for ``WeizmannDataset`` (data/weizmann.py) or ``BairRobotPush`` (data/bair.py) wherever ``train.py`` and
    ``get_generator`` use the dataset object: the same ``get_seq_len`` bounds and ``__len__``; the frames are the device clip
    store ``clips`` (a ``p2pvg_b200.data.VideoClips``), cut into batches by ``ClipBatches`` with ``sampling``."""

    def __init__(self, clips, train, seq_len, sampling, length):
        self.clips, self.train, self.seq_len, self.sampling, self.length = clips, train, seq_len, sampling, length
        self.max_seq_len, self.channels, self.image_size = clips.max_seq_len, 3, clips.frames.shape[-1]

    def get_seq_len(self):
        return np.random.randint(low=self.seq_len[0], high=self.seq_len[1] + 1)

    def __len__(self):
        return self.length


class PoseSet:
    """Stands in for ``Human36mDataset`` (data/human36m/human36m.py) wherever ``train.py`` and ``get_h36m_generator`` use the
    dataset object: the same ``get_seq_len`` bounds, ``__len__``, ``max_seq_len``, ``delta_len`` and ``speed_range``, and the
    dataset's own ``skeleton``.  The poses are the device stores ``clips`` (a ``p2pvg_b200.data.PoseClips``) uploaded from the
    dataset's normalised lists; the dataset itself, with its float64 lists and raw annotations, is not kept."""

    def __init__(self, ds):
        if ds.n_breakpoints > 0:
            raise NotImplementedError("device pose batches implement the constant-speed crop only (n_breakpoints = 0)")
        self.max_seq_len, self.delta_len, self.speed_range = ds.max_seq_len, ds.delta_len, list(ds.speed_range)
        self.skeleton, self.length = ds.skeleton, len(ds)
        self.clips = PoseClips(ds.data["pose"]["2d"], ds.data["pose"]["3d"], ds.data["camera_view"], ds.max_seq_len,
                               ds.speed_range[1], device="cuda")

    def get_seq_len(self):
        return np.random.randint(low=self.max_seq_len - 2 * self.delta_len, high=self.max_seq_len + 1)

    def __len__(self):
        return self.length


def _weizmann(opt, train):
    L = 18 if train else 10    # data_utils.py: train_max_seq_len / test_max_seq_len
    clips = load_weizmann_clips(opt.data_root, train, L, opt.image_width)
    return VideoClipSet(clips, train, (10 if train else 6, L), "permutation", len(clips))


def _bair(opt, train):
    clips = load_bair_clips(opt.data_root, train, opt.max_seq_len, opt.image_width)
    return VideoClipSet(clips, train, (opt.max_seq_len - 2 * opt.delta_len, opt.max_seq_len),
                        "uniform" if train else "ordered", 10000)


def load_dataset(opt, eval=False, eval_len=None, id_act=None):
    if opt.dataset in ("weizmann", "bair"):
        assert opt.channels == 3, "=> %s has 3 channels, but opt.channels = %d" % (opt.dataset, opt.channels)
        make = _weizmann if opt.dataset == "weizmann" else _bair
        return make(opt, True), make(opt, False)
    if opt.dataset == "h36m":
        train, test = _reference().load_dataset(opt, eval=eval, eval_len=eval_len, id_act=id_act)
        return PoseSet(train), PoseSet(test)
    if opt.dataset != "mnist":
        return _reference().load_dataset(opt, eval=eval, eval_len=eval_len, id_act=id_act)
    kw = dict(data_root=opt.data_root, max_seq_len=opt.max_seq_len, delta_len=opt.delta_len, image_size=opt.image_width,
              num_digits=opt.num_digits, deterministic=False)
    return MovingMNISTDigits(train=True, **kw), MovingMNISTDigits(train=False, **kw)


def get_data_generator(data, train=True, dynamic_length=True, opt=None):
    if opt.dataset in ("weizmann", "bair"):
        if not dynamic_length:
            raise NotImplementedError("device clip batches always have the dynamic length get_seq_len() draws")
        return ClipBatches(data.clips, opt.batch_size, data.sampling, data.seq_len, device="cuda")
    if opt.dataset == "h36m":
        if not dynamic_length:
            raise NotImplementedError("device pose batches always have the dynamic length get_seq_len() draws")
        L = data.max_seq_len
        return PoseBatches(data.clips, opt.batch_size if train else 10, (L - 2 * data.delta_len, L), data.speed_range,
                           device="cuda")
    if opt.dataset != "mnist":
        return _reference().get_data_generator(data, train=train, dynamic_length=dynamic_length, opt=opt)
    if not dynamic_length:
        raise NotImplementedError("GPU-rendered Moving MNIST batches always have the dynamic length get_seq_len() draws")
    return MovingMNIST(data.digits, opt.batch_size, data.max_seq_len, data.delta_len, image_size=data.image_size,
                       num_digits=data.num_digits, deterministic=data.deterministic, device="cuda")
