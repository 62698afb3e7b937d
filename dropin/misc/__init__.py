"""Shadow of the reference's ``misc`` package: ``misc.criterion`` comes from p2pvg_b200, ``misc.visualize`` runs ``vis_seq`` on
the graphed generator (every other name in it is the reference's), and every other submodule (``misc.utils``,
``misc.metrics``) keeps resolving to the reference checkout named by $P2PVG_REF (or any later ``misc`` directory on
sys.path)."""
import os
import sys

_here = os.path.dirname(os.path.abspath(__file__))
for _p in [os.environ.get("P2PVG_REF", "")] + list(sys.path):
    _cand = os.path.join(_p, "misc") if _p else ""
    if _cand and os.path.isdir(_cand) and os.path.abspath(_cand) != _here and _cand not in __path__:
        __path__.append(_cand)
