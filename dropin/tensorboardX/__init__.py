"""Shadow of the ``tensorboardX`` package for the reference's ``train.py`` (``from tensorboardX import SummaryWriter``): only
``SummaryWriter`` is replaced, by a subclass whose ``add_histogram`` computes fp32 / fp64 histograms on the GPU
(``p2pvg_b200.tboard.HistogramWriterMixin``) and whose ``add_image`` encodes 3-channel float32 / uint8 images as PNG on the
GPU (``p2pvg_b200.tboard.add_image_gpu``: the same pixels, other compressed bytes).  Scalars, videos and every other call
are the base class's.

The real tensorboardX is the next ``tensorboardX`` directory on sys.path after this one: its ``__init__.py`` runs in this
module with ``__path__`` pointing at its directory, so every submodule and every other name is the real one.  When no
real tensorboardX is installed, ``SummaryWriter`` derives from ``torch.utils.tensorboard.SummaryWriter`` (which takes the
``log_dir=`` keyword ``train.py`` passes) and nothing else is exported."""
import os
import sys

from p2pvg_b200.tboard import HistogramWriterMixin as _Mixin
from p2pvg_b200.tboard import add_image_gpu as _add_image_gpu

_here = os.path.dirname(os.path.abspath(__file__))
_real = None
for _p in sys.path:
    _cand = os.path.join(_p or os.getcwd(), "tensorboardX")
    if os.path.abspath(_cand) != _here and os.path.isfile(os.path.join(_cand, "__init__.py")):
        _real = os.path.abspath(_cand)
        break

if _real is not None:
    __path__ = [_real]
    with open(os.path.join(_real, "__init__.py")) as _f:
        exec(compile(_f.read(), os.path.join(_real, "__init__.py"), "exec"))
    _Base = SummaryWriter  # noqa: F821 -- defined by the real package's __init__
else:
    from torch.utils.tensorboard import SummaryWriter as _Base


class SummaryWriter(_Mixin, _Base):
    __doc__ = _Base.__doc__

    def add_image(self, tag, img_tensor, global_step=None, walltime=None, dataformats='CHW'):
        if not _add_image_gpu(self, tag, img_tensor, global_step, walltime, dataformats):
            return super().add_image(tag, img_tensor, global_step=global_step, walltime=walltime, dataformats=dataformats)
