"""Shadow of the reference's ``data`` package: ``data.data_utils`` comes from here (Moving MNIST, Weizmann, BAIR and
Human3.6M batches made on the GPU), every other submodule (``data.moving_mnist``, ``data.weizmann``, ``data.bair``, ...) keeps resolving to the
reference checkout named by $P2PVG_REF (or any later ``data`` directory on sys.path)."""
import os
import sys

_here = os.path.dirname(os.path.abspath(__file__))
for _p in [os.environ.get("P2PVG_REF", "")] + list(sys.path):
    _cand = os.path.join(_p, "data") if _p else ""
    if _cand and os.path.isdir(_cand) and os.path.abspath(_cand) != _here and _cand not in __path__:
        __path__.append(_cand)
