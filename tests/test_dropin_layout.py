"""`dropin/` shadows the reference's package names (CPU: import wiring and exported C symbols only)."""
import ctypes
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_dropin_packages_resolve_to_the_kernel_backed_modules():
    code = ("import models.dcgan_64 as b, models.dcgan_128, models.vgg_64, models.vgg_128, models.h36m_mlp, models.lstm as l; from models.p2p_model import P2PModel; "
            "from misc import criterion; import p2pvg_b200.models.p2p_model as impl; "
            "assert P2PModel is impl.P2PModel and hasattr(b, 'encoder') and hasattr(l, 'gaussian_lstm'); "
            "assert criterion.KLCriterion.__module__.startswith('p2pvg_b200'); print('ok')")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "dropin"), ROOT]))
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd="/")
    assert out.returncode == 0 and "ok" in out.stdout, out.stderr


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "p2pvg_b200.h")).read()
    names = set(re.findall(r"\b(p2pvg_[a-z0-9_]+)\s*\(", hdr))
    assert len(names) > 30
    lib = ctypes.CDLL(os.path.join(ROOT, "p2pvg_b200", "libp2pvg_b200.so"))
    missing = [n for n in sorted(names) if not hasattr(lib, n)]
    assert not missing, missing
    assert lib.p2pvg_version() >= 100
    # and the other way round: every entry point the ctypes binding calls is declared in the header
    called = set(re.findall(r"lib\.(p2pvg_[a-z0-9_]+)", open(os.path.join(ROOT, "p2pvg_b200", "_lib.py")).read()))
    assert len(called) > 30
    undeclared = sorted(called - names)
    assert not undeclared, undeclared
