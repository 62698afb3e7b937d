"""Drop-in for the reference's ``data/human36m/human36m.py``, which ``train.py``'s ``from human36m import
Skeleton3DVisualizer, STD_SCALE`` reaches when ``dropin/`` comes first on sys.path: ``Skeleton3DVisualizer`` is
``p2pvg_b200.skeleton.Skeleton3DVisualizer`` (the skeletons drawn on the GPU, no matplotlib), ``STD_SCALE`` is the
reference's 3, and every other name (``Human36mDataset``, ``fig2img``, ...) is the reference's, from its module loaded by
path out of $P2PVG_REF/data/human36m or a ``data/human36m`` directory on sys.path (that directory is put on sys.path for the
module's own ``from skeleton import Skeleton``)."""
import importlib.util
import os
import sys

from p2pvg_b200.skeleton import Skeleton3DVisualizer  # noqa: F401

STD_SCALE = 3

_here = os.path.dirname(os.path.abspath(__file__))
_ref = None


def _reference_dir():
    roots = [os.environ.get("P2PVG_REF", "")] + list(sys.path)
    for p in roots:
        for d in ((os.path.join(p, "data", "human36m"), p) if p else ()):
            if os.path.abspath(d) != _here and os.path.isfile(os.path.join(d, "human36m.py")) and \
                    os.path.basename(os.path.normpath(os.path.abspath(d))) == "human36m":
                return d
    raise ImportError("the reference's data/human36m/human36m.py was not found: set P2PVG_REF to the reference checkout")


def _reference():
    global _ref
    if _ref is None:
        d = _reference_dir()
        if d not in sys.path:
            sys.path.append(d)
        spec = importlib.util.spec_from_file_location("_reference_human36m", os.path.join(d, "human36m.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        _ref = mod
    return _ref


def __getattr__(name):
    if name.startswith("__"):
        raise AttributeError(name)
    return getattr(_reference(), name)
