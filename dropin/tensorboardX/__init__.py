"""Shadow of the ``tensorboardX`` package for the reference's ``train.py`` (``from tensorboardX import SummaryWriter``): only
``SummaryWriter`` is replaced, by a subclass whose ``add_histogram`` computes fp32 / fp64 histograms on the GPU
(``p2pvg_b200.tboard.HistogramWriterMixin``) and whose ``add_image`` encodes 3-channel float32 / uint8 images as PNG on the
GPU (``p2pvg_b200.tboard.add_image_gpu``: the same pixels, other compressed bytes), whose ``add_video`` encodes one
3-channel float32 / uint8 video as a GIF on the GPU (``p2pvg_b200.tboard.add_video_gpu``), and whose event records are
framed with the library's native CRC-32C (``p2pvg_b200.tboard.native_record_crc``: the same bytes).  Scalars and every
other call are the base class's.

The real tensorboardX is the next ``tensorboardX`` directory on sys.path after this one: its ``__init__.py`` runs in this
module with ``__path__`` pointing at its directory, so every submodule and every other name is the real one.  When no
real tensorboardX is installed, ``SummaryWriter`` derives from ``torch.utils.tensorboard.SummaryWriter`` (which takes the
``log_dir=`` keyword ``train.py`` passes) and nothing else is exported."""
import os
import sys

from p2pvg_b200.tboard import HistogramWriterMixin as _Mixin
from p2pvg_b200.tboard import add_image_gpu as _add_image_gpu
from p2pvg_b200.tboard import add_video_gpu as _add_video_gpu
from p2pvg_b200.tboard import native_record_crc as _native_record_crc

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

    def add_video(self, tag, vid_tensor, global_step=None, fps=4, walltime=None):
        if not _add_video_gpu(self, tag, vid_tensor, global_step, fps, walltime):
            return super().add_video(tag, vid_tensor, global_step=global_step, fps=fps, walltime=walltime)

    def _get_file_writer(self):
        fw = super()._get_file_writer()
        _native_record_crc(fw)
        return fw
