"""p2pvg_histograms (csrc/histogram.cu) and p2pvg_b200.tboard on the GPU: counts bit for bit against np.histogram, the
statistics against NumPy, bit-identical results whatever shares the launch, the wrapper's input checks, and train.py's
histogram block end to end against stock add_histogram for dcgan_64, vgg_64 and h36m_mlp."""
import ctypes
import importlib
import os
import sys
import types

import numpy as np
import pytest
import torch

from p2pvg_b200 import tboard
from p2pvg_b200._lib import kernels_for

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E = tboard.DEFAULT_BINS


def ref_hist(v, edges=E):
    v64 = np.asarray(v).astype(np.float64).reshape(-1)
    return np.histogram(v64, bins=edges)[0], v64


def check_stats(st, v64):
    mn, mx, num, sm, sq = st
    assert num == v64.size
    assert (np.isnan(mn) and np.isnan(v64.min())) or mn == v64.min()
    assert (np.isnan(mx) and np.isnan(v64.max())) or mx == v64.max()
    for got, want, scale in ((sm, v64.sum(), np.abs(v64).sum()), (sq, v64.dot(v64), v64.dot(v64))):
        if not np.isfinite(want):
            assert got == want or (np.isnan(got) and np.isnan(want))
        else:
            assert abs(got - want) <= 1e-12 * scale


def cases():
    r = np.random.RandomState(0)
    edge_vals = np.concatenate([E, np.nextafter(E, -np.inf), np.nextafter(E, np.inf)])
    sub = np.array([1e-45, -1e-45, 1e-40, -1e-40, 1.17549e-38, -1.17549e-38], dtype=np.float32)
    spec = np.array([np.inf, -np.inf, np.nan, 9.93e19, -9.93e19, 1e30, -1e30, E[0], E[-1], 0.5], dtype=np.float64)
    return {
        "weights_f32": (0.02 * r.randn(100_003)).astype(np.float32),
        "grads_f32": np.where(r.rand(70_001) < 0.1, 0, 1e-4 * r.randn(70_001)).astype(np.float32),
        "weights_f64": 0.05 * r.randn(40_000),
        "zeros_pm_f32": np.tile(np.array([0.0, -0.0], dtype=np.float32), 20_000),
        "zeros_pm_f64": np.tile(np.array([0.0, -0.0]), 777),
        "subnormal_f32": np.tile(sub, 5000),
        "edges_f64": edge_vals,
        "edges_f32": E.astype(np.float32),
        "special_f64": np.tile(spec, 300),
        "special_f32": np.tile(spec.astype(np.float32), 301),
        "inf_only_f32": np.array([np.inf, -np.inf, 1.0], dtype=np.float32),
        "one_f32": np.array([-3.5e-7], dtype=np.float32),
        "one_f64": np.array([2.0]),
        "all_zero_f32": np.zeros(300_000, dtype=np.float32),
    }


def run(arrays, edges=E):
    ts = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]
    return tboard.histograms(ts, edges)


def test_counts_and_stats_match_numpy_in_one_launch():
    cs = cases()
    res = run(list(cs.values()))
    for (name, a), (counts, st) in zip(cs.items(), res):
        want, v64 = ref_hist(a)
        assert np.array_equal(counts, want), name
        check_stats(st, v64)


def test_subnormal_edges_and_single_bin():
    a = np.array([-1e-40, -1e-42, -0.0, 0.0, 1e-45, 1e-41, 1e-39, -1e-39, 3e-39], dtype=np.float32).repeat(33)
    for edges in ([-1e-39, -1e-41, 0.0, 1e-41, 1e-39], [-1e-39, 1e-39], [0.0, 1e-41]):
        (counts, st), = run([a], edges)
        want, v64 = ref_hist(a, edges)
        assert np.array_equal(counts, want), edges
        check_stats(st, v64)


def test_large_segment_and_many_segments():
    r = np.random.RandomState(1)
    big = (0.01 * r.randn((1 << 24) + 12345)).astype(np.float32)
    many = [(r.randn(int(n)) * 10.0 ** r.randint(-6, 3)).astype(np.float32 if k % 3 else np.float64)
            for k, n in enumerate(r.randint(1, 3000, size=1100))]
    res = run([big] + many)
    for a, (counts, st) in zip([big] + many, res):
        want, v64 = ref_hist(a)
        assert np.array_equal(counts, want)
        check_stats(st, v64)


def test_integer_valued_sums_are_exact():
    r = np.random.RandomState(2)
    arrs = [r.randint(-1000, 1000, size=n).astype(dt) for n, dt in ((50_000, np.float32), (123_457, np.float64), (1, np.float32))]
    for a, (counts, st) in zip(arrs, run(arrs)):
        v64 = a.astype(np.float64)
        assert st[3] == v64.sum() and st[4] == v64.dot(v64)


def _bits(res):
    return [(c.tobytes(), np.array(s, dtype=np.float64).tobytes()) for c, s in res]


def test_bit_identical_across_launches_orders_and_compositions():
    cs = list(cases().values())
    r = np.random.RandomState(3)
    extra = [(r.randn(n)).astype(np.float32) for n in (5, 70_000, 16384, 16385)]
    arrs = cs + extra
    base = _bits(run(arrs))
    assert _bits(run(arrs)) == base
    perm = r.permutation(len(arrs))
    got = _bits(run([arrs[i] for i in perm]))
    assert [got[list(perm).index(i)] for i in range(len(arrs))] == base
    for i in (0, 3, len(arrs) - 1):
        assert _bits(run([arrs[i]])) == [base[i]]
    assert _bits(run(arrs[::2] + [np.ones(10 ** 6, np.float32)]))[:len(arrs[::2])] == base[::2]


def test_wrapper_rejects_before_any_launch():
    K = kernels_for("cuda")
    n0 = K.launches
    good = torch.randn(10, device="cuda")
    bad_inputs = [
        [good, torch.randn(10)],                               # CPU tensor
        [torch.randn(4, 6, device="cuda").t()],                # non-contiguous
        [torch.arange(5, device="cuda")],                      # int64
        [torch.randn(5, device="cuda", dtype=torch.bfloat16)],
        [torch.empty(0, device="cuda")],
    ]
    for ts in bad_inputs:
        with pytest.raises(ValueError):
            tboard.histograms(ts)
    for edges in ([0.0, 1.0, 1.0], [1.0, 0.0], [0.0, np.inf], [0.0, np.nan, 1.0], np.arange(4097.0), [1.0]):
        with pytest.raises(ValueError):
            tboard.histograms([good], edges)
    assert K.launches == n0


def test_abi_rejections_and_empty_launch():
    K = kernels_for("cuda")
    lib = K.lib
    t = torch.randn(100, device="cuda")
    edges = np.ascontiguousarray(E)
    out = torch.zeros(2 * len(E), dtype=torch.int64, device="cuda")
    st = torch.zeros(10, dtype=torch.float64, device="cuda")
    ws = torch.empty(1 << 16, dtype=torch.uint8, device="cuda")
    s = K._stream()

    def call(segs, n_seg, ws_bytes=ws.numel(), e=edges, ne=len(E)):
        return lib.p2pvg_histograms(ctypes.c_void_p(segs.ctypes.data), n_seg, ctypes.c_void_p(e.ctypes.data), ne,
                                    ctypes.c_void_p(ws.data_ptr()), ctypes.c_size_t(ws_bytes), ctypes.c_void_p(out.data_ptr()),
                                    ctypes.c_void_p(st.data_ptr()), s)

    assert lib.p2pvg_histograms(None, 0, None, 0, None, ctypes.c_size_t(0), None, None, s) == 0
    ok = np.array([[t.data_ptr(), 100, 0]], dtype=np.int64)
    assert call(ok, 1) == 0
    assert call(np.array([[t.data_ptr(), 100, 1]], dtype=np.int64), 1) == -1          # bf16 is not taken
    assert call(np.array([[t.data_ptr(), 0, 0]], dtype=np.int64), 1) == -1            # empty segment
    assert call(np.array([[t.data_ptr() + 2, 10, 0]], dtype=np.int64), 1) == -1       # misaligned
    assert call(ok, 1, ws_bytes=64) == -4
    bad = edges.copy()
    bad[5] = bad[4]
    assert call(ok, 1, e=bad) == -1
    big = np.arange(4097.0)
    assert call(ok, 1, e=big, ne=4097) == -2
    torch.cuda.synchronize()


# ---- train.py's block end to end ----------------------------------------------------------------------------------------

# dataset, channels, width, rnn_size, batch, sequence length
CONFIGS = {"dcgan_64": ("mnist", 1, 64, 256, 8, 6), "vgg_64": ("weizmann", 3, 64, 256, 8, 6),
           "h36m_mlp": ("h36m", 1, None, 512, 16, 8)}


def make_model(backbone):
    dataset, C, width, rnn, B, _ = CONFIGS[backbone]
    os.environ["P2PVG_PRECISION"] = "bf16"
    os.environ["P2PVG_GRAPH"] = "1"
    torch.manual_seed(1)
    net = importlib.import_module(f"p2pvg_b200.models.{backbone}")
    opt = types.SimpleNamespace(dataset=dataset, backbone_net=net, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0,
                                weight_align=0.5, skip_prob=0.0, n_past=1, last_frame_skip=False, batch_size=B)
    from p2pvg_b200.models.p2p_model import P2PModel
    return P2PModel(B, C, 128, 10, rnn, 1, 1, 2, opt=opt).cuda().train()


def batch(backbone, seed):
    _, C, width, _, B, T = CONFIGS[backbone]
    g = torch.Generator().manual_seed(seed)
    if width is None:
        return (None, (3 * torch.randn(T, B, 17, 3, generator=g)).cuda(), None)
    return torch.rand(T, B, C, width, width, generator=g).cuda()


def step(model, backbone, seed):
    torch.manual_seed(100 + seed)
    np.random.seed(seed)
    T = CONFIGS[backbone][5]
    return np.array(model(batch(backbone, seed), 0, T - 1))


class Recorder:
    def __init__(self):
        self.rows = []

    def add_summary(self, summary, global_step=None, walltime=None):
        for v in summary.value:
            self.rows.append((v.tag, global_step, v.histo))


def recording(cls, log_dir):
    class Rec(cls):
        def _get_file_writer(self):
            if not hasattr(self, "_rec"):
                self._rec = Recorder()
            return self._rec
    return Rec(log_dir=str(log_dir))


def dropin_writer_class(monkeypatch):
    monkeypatch.syspath_prepend(os.path.join(ROOT, "dropin"))
    monkeypatch.delitem(sys.modules, "tensorboardX", raising=False)
    mod = importlib.import_module("tensorboardX")
    assert os.path.dirname(mod.__file__) == os.path.join(ROOT, "dropin", "tensorboardX")
    return mod.SummaryWriter


def stock_block(writer, model, step_, abs_sums):
    """train.py:225-233 verbatim, plus the sum of |v| of every logged tensor (the scale of the sum's tolerance)."""
    for name, param in model.named_parameters():
        if param.requires_grad:
            name = name.replace('.', '/')
            writer.add_histogram(name, param.data.cpu().numpy(), step_)
            abs_sums.append(np.abs(param.data.cpu().numpy().astype(np.float64)).sum())
            try:
                writer.add_histogram(name + '/grad', param.grad.data.cpu().numpy(), step_)
                abs_sums.append(np.abs(param.grad.data.cpu().numpy().astype(np.float64)).sum())
            except Exception:
                pass


def same_protos(got, want, abs_sums):
    assert [(t, s) for t, s, _ in got] == [(t, s) for t, s, _ in want]
    assert len(abs_sums) == len(want)
    for (tag, _, g), (_, _, w), a in zip(got, want, abs_sums):
        assert list(g.bucket) == list(w.bucket), tag
        assert list(g.bucket_limit) == list(w.bucket_limit), tag
        assert g.num == w.num and g.min == w.min and g.max == w.max, tag
        assert abs(g.sum - w.sum) <= 1e-12 * a, tag
        assert abs(g.sum_squares - w.sum_squares) <= 1e-12 * w.sum_squares, tag


@pytest.mark.parametrize("backbone", ["dcgan_64", "vgg_64", "h36m_mlp"])
def test_param_histograms_match_stock_add_histogram(backbone, tmp_path, monkeypatch):
    from torch.utils.tensorboard import SummaryWriter
    model = make_model(backbone)
    # before the first forward: plain parameters, no gradients yet
    stock, fast = recording(SummaryWriter, tmp_path / "a"), recording(SummaryWriter, tmp_path / "b")
    a0 = []
    stock_block(stock, model, 0, a0)
    tboard.add_param_histograms(fast, model, 0)
    assert not any(t.endswith("/grad") for t, _, _ in stock._rec.rows)
    same_protos(fast._rec.rows, stock._rec.rows, a0)
    # after seeded training steps: arena views, .grad set
    drop = recording(dropin_writer_class(monkeypatch), tmp_path / "c")
    a1 = []
    for k in (1, 2):
        step(model, backbone, k)
        stock_block(stock, model, k, a1)
        tboard.add_param_histograms(fast, model, k)
        stock_block(drop, model, k, [])
    assert any(t.endswith("/grad") for t, _, _ in stock._rec.rows)
    same_protos(fast._rec.rows, stock._rec.rows, a0 + a1)
    same_protos(drop._rec.rows, stock._rec.rows[len(a0):], a1)
    stock.close(), fast.close(), drop.close()


@pytest.mark.parametrize("backbone", ["dcgan_64", "vgg_64", "h36m_mlp"])
def test_logging_leaves_the_next_step_unchanged(backbone, tmp_path):
    from torch.utils.tensorboard import SummaryWriter
    losses = []
    for log in (False, True):
        model = make_model(backbone)
        w = recording(SummaryWriter, tmp_path / str(log))
        step(model, backbone, 1)
        if log:
            tboard.add_param_histograms(w, model, 1)
        losses.append(np.stack([step(model, backbone, k) for k in (2, 3)]))
        w.close()
    assert losses[0].tobytes() == losses[1].tobytes()


def test_dropin_writer_takes_the_gpu_path_for_tensors_and_arrays(tmp_path, monkeypatch):
    from torch.utils.tensorboard import SummaryWriter
    cls = dropin_writer_class(monkeypatch)
    drop, stock = recording(cls, tmp_path / "a"), recording(SummaryWriter, tmp_path / "b")
    K = kernels_for("cuda")
    r = np.random.RandomState(4)
    vals = [r.randn(1000).astype(np.float32), 0.3 * r.randn(77), torch.randn(3, 50, device="cuda"), torch.randn(64)]
    abs_sums = []
    for i, v in enumerate(vals):
        a = v.cpu().numpy() if torch.is_tensor(v) else v
        for kw in (dict(), dict(max_bins=10), dict(bins=[-1.0, 0.0, 0.5, 2.0])):
            n0 = K.launches
            drop.add_histogram(f"t{i}", v, i, **kw)
            assert K.launches == n0 + 1
            stock.add_histogram(f"t{i}", a, i, **kw)
            abs_sums.append(np.abs(a.astype(np.float64)).sum())
    n0 = K.launches
    drop.add_histogram("ints", np.arange(10), 0)                   # other dtypes, int and string bins: the base class
    drop.add_histogram("auto", vals[0], 0, bins="auto")
    drop.add_histogram("int_bins", vals[0], 0, bins=7)
    stock.add_histogram("ints", np.arange(10), 0)
    stock.add_histogram("auto", vals[0], 0, bins="auto")
    stock.add_histogram("int_bins", vals[0], 0, bins=7)
    assert K.launches == n0
    abs_sums += [np.arange(10).sum()] + [np.abs(vals[0].astype(np.float64)).sum()] * 2
    same_protos(drop._rec.rows, stock._rec.rows, abs_sums)
