"""Drop-in for the reference's ``misc/visualize.py``: ``vis_seq`` runs ``p2pvg_b200.visualize.vis_seq`` (only the displayed
rows generated, all samples in one CUDA-graph replay, the pictures composed in one launch, the PNG file encoded on the GPU by
``p2pvg_b200.png.save_image`` and the GIF file by ``p2pvg_b200.gif.save_gif``) whenever
``p2pvg_b200.visualize.check_vis_seq`` accepts the call, and the reference's own ``vis_seq`` otherwise.  Every other name
(``add_gt_cp_border``, ``add_samples_cp_border``, ``save_utils``, ...) is the reference's, from its module loaded from the
reference's ``misc/`` directory."""
import importlib.util
import os

import misc as _pkg
from p2pvg_b200 import gif as _gif
from p2pvg_b200 import png as _png
from p2pvg_b200 import visualize as _fast

_here = os.path.dirname(os.path.abspath(__file__))
_ref = None


def _reference():
    global _ref
    if _ref is None:
        for d in _pkg.__path__:
            f = os.path.join(d, "visualize.py")
            if os.path.abspath(d) != _here and os.path.isfile(f):
                spec = importlib.util.spec_from_file_location("misc._reference_visualize", f)
                mod = importlib.util.module_from_spec(spec)
                spec.loader.exec_module(mod)
                _ref = mod
                break
        else:
            raise ImportError("the reference's misc/visualize.py was not found: set P2PVG_REF to the reference checkout")
    return _ref


def __getattr__(name):
    if name.startswith("__"):
        raise AttributeError(name)
    return getattr(_reference(), name)


def vis_seq(model, x, epoch, output_len, model_mode='full', recon_mode=None, skip_frame=True, h36m_visualizer=None, writer=None,
            opt=None):
    try:
        _fast.check_vis_seq(model, x, output_len, model_mode, skip_frame, opt)
    except ValueError:
        return _reference().vis_seq(model, x, epoch, output_len, model_mode=model_mode, recon_mode=recon_mode,
                                    skip_frame=skip_frame, h36m_visualizer=h36m_visualizer, writer=writer, opt=opt)
    _fast.vis_seq(model, x, epoch, output_len, model_mode=model_mode, recon_mode=recon_mode, skip_frame=skip_frame,
                  h36m_visualizer=h36m_visualizer, writer=writer, opt=opt, save_png=_png.save_image,
                  save_gif=_gif.save_gif)
