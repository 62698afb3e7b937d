"""p2pvg_b200.tboard's host side: TensorBoard's default edges, histogram_fields against make_histogram from np.histogram's
counts, and the tensorboardX drop-in's name resolution (no GPU needed)."""
import importlib.util
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from torch.utils.tensorboard import SummaryWriter
from torch.utils.tensorboard.summary import make_histogram

from p2pvg_b200 import tboard

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_default_bins_are_the_writers(tmp_path):
    w = SummaryWriter(log_dir=str(tmp_path))
    want = np.array(w.default_bins, dtype=np.float64)
    w.close()
    assert tboard.DEFAULT_BINS.shape == want.shape == (1549,)
    assert tboard.DEFAULT_BINS.tobytes() == want.tobytes()
    assert (tboard.DEFAULT_BINS < 0).sum() == 774 and (tboard.DEFAULT_BINS > 0).sum() == 774


def inputs():
    r = np.random.RandomState(0)
    E = tboard.DEFAULT_BINS
    return [
        ("normal_weights", 0.02 * r.randn(5000), E),
        ("normal_grads", 1e-5 * r.randn(777), E),
        ("wide", 10.0 ** r.uniform(-15, 19, 3000) * np.sign(r.randn(3000)), E),
        ("all_zeros", np.zeros(100), E),
        ("first_bin", np.array([E[0], E[0], -1.0]), E),
        ("last_bin", np.array([E[-1], 3.0]), E),
        ("first_and_last", np.array([E[0], E[-1]]), E),
        ("single_value", np.array([0.5]), E),
        ("single_bin_table", r.rand(50), np.array([0.0, 1.0])),
        ("two_bins", np.array([0.25, 0.25, 1.0]), np.array([0.0, 0.5, 1.0])),
        ("integers", r.randint(-5, 5, 400).astype(np.float64), np.arange(-6.0, 7.0)),
        ("with_nan_inf", np.array([np.nan, np.inf, -np.inf, 0.1, -0.2]), E),
        ("out_of_range_one_bin", np.array([5.0, -3.0]), np.array([0.0, 1.0])),
    ]


def numpy_stats(v):
    return (v.min(), v.max(), v.size, v.sum(), v.dot(v))


@pytest.mark.parametrize("max_bins", [None, 1, 2, 7, 100, 774, 1000, 1548, 2000])
def test_histogram_fields_reproduce_make_histogram(max_bins):
    for name, v, edges in inputs():
        counts = np.histogram(v, bins=edges)[0]
        want = make_histogram(v, edges, max_bins)
        got = tboard.histogram_fields(counts, numpy_stats(v), edges, max_bins)
        assert got["bucket_limits"] == list(want.bucket_limit), name
        assert got["bucket_counts"] == list(want.bucket), name
        for k in ("min", "max", "num", "sum", "sum_squares"):
            a, b = got[k], getattr(want, k)
            assert a == b or (np.isnan(a) and np.isnan(b)), (name, k)


@pytest.mark.parametrize("max_bins", [None, 3])
def test_all_out_of_range_raises_like_make_histogram(max_bins):
    E = tboard.DEFAULT_BINS
    v = np.array([1e21, -1e21, np.nan])
    with pytest.raises(ValueError, match="The histogram is empty"):
        make_histogram(v, E, max_bins)
    with pytest.raises(ValueError, match="The histogram is empty"):
        tboard.histogram_fields(np.histogram(v, bins=E)[0], numpy_stats(v), E, max_bins)


def test_edge_checks():
    assert tboard.check_edges([0, 1, 2]).dtype == np.float64
    for bad in ([1.0], [0.0, 0.0], [1.0, 0.0], [0.0, np.inf], [np.nan, 1.0], np.arange(4097.0), [[0.0, 1.0]]):
        with pytest.raises(ValueError):
            tboard.check_edges(bad)


FAKE_WRITER = '''
CALLS = []


class SummaryWriter:
    def __init__(self, log_dir=None, **kw):
        CALLS.append(("init", log_dir))

    def add_scalar(self, tag, value, global_step=None, walltime=None):
        CALLS.append(("scalar", tag))

    def add_histogram(self, tag, values, global_step=None, bins="tensorflow", walltime=None, max_bins=None):
        CALLS.append(("histogram", tag))

    def add_histogram_raw(self, tag, min, max, num, sum, sum_squares, bucket_limits, bucket_counts, global_step=None,
                          walltime=None):
        CALLS.append(("histogram_raw", tag))
'''

PROBE = '''
import json, os, sys
import numpy as np
sys.path[:0] = [{root!r}, os.path.join({root!r}, "dropin")] + {extra!r}
import tensorboardX
out = dict(path=list(tensorboardX.__path__), file=tensorboardX.__file__,
           bases=[c.__module__ + "." + c.__name__ for c in tensorboardX.SummaryWriter.__mro__])
if {extra!r}:
    import tensorboardX.summary
    out["summary"] = tensorboardX.summary.__file__
    out["marker"] = tensorboardX.MARKER
    w = tensorboardX.SummaryWriter(log_dir="runs/x")
    w.add_scalar("a", 1.0, 3)
    w.add_histogram("ints", np.arange(5), 1)
    w.add_histogram("int_bins", np.arange(5.0), 1, bins=10)
    w.add_histogram("auto", np.arange(5.0), 1, bins="auto")
    from tensorboardX import writer
    out["calls"] = writer.CALLS
print(json.dumps(out))
'''


def probe(extra):
    r = subprocess.run([sys.executable, "-c", PROBE.format(root=ROOT, extra=extra)], capture_output=True, text=True,
                       cwd=ROOT, env={k: v for k, v in os.environ.items() if k != "PYTHONPATH"})
    assert r.returncode == 0, r.stderr
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_dropin_wraps_the_real_tensorboardx(tmp_path):
    real = tmp_path / "site" / "tensorboardX"
    real.mkdir(parents=True)
    (real / "__init__.py").write_text("from .writer import SummaryWriter\nMARKER = 'real'\n")
    (real / "writer.py").write_text(FAKE_WRITER)
    (real / "summary.py").write_text("X = 1\n")
    out = probe([str(tmp_path / "site")])
    assert out["path"] == [str(real)]
    assert os.path.dirname(out["file"]) == os.path.join(ROOT, "dropin", "tensorboardX")
    assert out["summary"] == str(real / "summary.py") and out["marker"] == "real"
    assert out["bases"][1:3] == ["p2pvg_b200.tboard.HistogramWriterMixin", "tensorboardX.writer.SummaryWriter"]
    # the constructor, scalars, other dtypes and int / string bins reach the real class unchanged
    assert out["calls"] == [["init", "runs/x"], ["scalar", "a"], ["histogram", "ints"], ["histogram", "int_bins"],
                            ["histogram", "auto"]]


def test_dropin_falls_back_to_torch_writer():
    if importlib.util.find_spec("tensorboardX") is not None:
        pytest.skip("a real tensorboardX is installed")
    out = probe([])
    assert out["path"] == [os.path.join(ROOT, "dropin", "tensorboardX")]
    assert out["bases"][1:3] == ["p2pvg_b200.tboard.HistogramWriterMixin", "torch.utils.tensorboard.writer.SummaryWriter"]


def test_mixin_sends_other_inputs_to_the_base(tmp_path):
    calls = []

    class Base:
        def add_histogram(self, tag, values, global_step=None, bins="tensorflow", walltime=None, max_bins=None):
            calls.append(tag)

    class W(tboard.HistogramWriterMixin, Base):
        pass

    w = W()
    w.add_histogram("ints", np.arange(4), 0)
    w.add_histogram("int_bins", np.arange(4.0), 0, bins=3)
    w.add_histogram("string_bins", torch.arange(4.0), 0, bins="fd")
    w.add_histogram("half", torch.zeros(3, dtype=torch.float16), 0)
    w.add_histogram("empty", np.zeros(0, np.float32), 0)
    w.add_histogram("bad_edges", np.arange(4.0), 0, bins=[1.0, 0.0])
    assert calls == ["ints", "int_bins", "string_bins", "half", "empty", "bad_edges"]
    if not torch.cuda.is_available():
        w.add_histogram("no_gpu", np.arange(4.0), 0)
        assert calls[-1] == "no_gpu"
