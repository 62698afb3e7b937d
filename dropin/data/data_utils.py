"""Drop-in for the reference's ``data/data_utils.py``: the ``mnist`` branches of ``load_dataset`` and ``get_data_generator``
render Moving MNIST batches on the GPU (``p2pvg_b200.data.MovingMNIST``); every other call and dataset is delegated
unchanged to the reference's own module, loaded from the reference's ``data/`` directory.

The generator yields what the reference's ``get_generator`` yields, fp32 [T, B, 1, S, S] on the device, and draws T from
NumPy's global stream at the same point; the digit trajectories are drawn on the device (torch's CUDA generator, seeded by
``train.py``'s ``torch.cuda.manual_seed_all``) instead of in a loader worker process.  MNIST is read from torchvision's raw
files under ``<data_root>/MNIST/raw`` and never downloaded."""
import importlib.util
import os

import numpy as np

import data as _pkg
from p2pvg_b200.data import MovingMNIST, load_mnist_digits

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


def load_dataset(opt, eval=False, eval_len=None, id_act=None):
    if opt.dataset != "mnist":
        return _reference().load_dataset(opt, eval=eval, eval_len=eval_len, id_act=id_act)
    kw = dict(data_root=opt.data_root, max_seq_len=opt.max_seq_len, delta_len=opt.delta_len, image_size=opt.image_width,
              num_digits=opt.num_digits, deterministic=False)
    return MovingMNISTDigits(train=True, **kw), MovingMNISTDigits(train=False, **kw)


def get_data_generator(data, train=True, dynamic_length=True, opt=None):
    if opt.dataset != "mnist":
        return _reference().get_data_generator(data, train=train, dynamic_length=dynamic_length, opt=opt)
    if not dynamic_length:
        raise NotImplementedError("GPU-rendered Moving MNIST batches always have the dynamic length get_seq_len() draws")
    return MovingMNIST(data.digits, opt.batch_size, data.max_seq_len, data.delta_len, image_size=data.image_size,
                       num_digits=data.num_digits, deterministic=data.deterministic, device="cuda")
