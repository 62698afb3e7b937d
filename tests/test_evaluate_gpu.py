"""Split-level evaluation on the GPU: P2PModel.p2p_evaluate_lengths against looped p2p_evaluate calls for every graphed
backbone in both P2PVG_PRECISION modes; p2pvg_metrics_fold alone against its float64 restatement (tests/eval_ref.py), bit for
bit; evaluate_split against float64 host aggregation of looped p2p_evaluate results; and python -m p2pvg_b200.evaluate end to
end on a synthetic Weizmann tree.

Tolerances against the looped calls as test_generate_lengths_gpu.py (rtol 1e-4 + atol 2e-5), with its models."""
import json
import math

import numpy as np
import pytest
import torch

from tests.eval_ref import fold_ref, fold_results, new_totals
from tests.test_generate_engine_gpu import precision, run
from tests.test_generate_lengths_gpu import CONFIGS, draws_for
from tests.test_multi_cp_gpu import clip, config_model

pytestmark = pytest.mark.gpu
RTOL, ATOL = 1e-4, 2e-5


def close(a, b):
    return a.shape == b.shape and torch.allclose(a.double().cpu(), b.double().cpu(), rtol=RTOL, atol=ATOL, equal_nan=True)


def assert_same_results(got, ref, names, what):
    assert len(got) == len(ref), what
    for k, (g, r) in enumerate(zip(got, ref)):
        assert g["frames"] == r["frames"], (what, k)
        for n in names:
            assert close(g[n], r[n]), f"{what} length {k} {n}: {(g[n] - r[n]).abs().max().item():.3e}"
            assert torch.equal(g["best"][n][0].cpu(), r["best"][n][0].cpu()), (what, k, n)
            assert close(g["best"][n][1], r["best"][n][1]), (what, k, n)


# ---- 1. p2p_evaluate_lengths against looped p2p_evaluate ---------------------------------------------------------------------
@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("backbone,C,n_past,lfs", CONFIGS, ids=[f"{b}-C{c}-np{n}{'-lfs' if l else ''}" for b, c, n, l in CONFIGS])
def test_evaluate_lengths_equals_looped_evaluate(backbone, C, n_past, lfs, prec):
    """Lengths below, equal to and above len(x), unsorted; nsample 1 and 3.  Same scores and best samples, and NumPy's and
    torch's CUDA generator left in the same state."""
    from p2pvg_b200 import metrics
    T, B = 6, 2
    lens = [4, 9, 6]
    with precision(prec):
        model = config_model(backbone, C, n_past, lfs, B)
        names = metrics.POSE_METRICS if model.is_pose else metrics.FRAME_METRICS
        x = clip(model, T, B, seed=T + n_past)
        for ns in (1, 3):
            what = f"{backbone} {prec} nsample={ns}"
            draws = draws_for(lens, ns * B, model.z_dim, seed=ns)
            torch.cuda.manual_seed(11)
            got = run(lambda: model.p2p_evaluate_lengths(x, lens, nsample=ns), 5, draws)
            np_after, rng_after = np.random.get_state(), torch.cuda.get_rng_state()
            torch.cuda.manual_seed(11)
            ref = run(lambda: [model.p2p_evaluate(x, ns, len_output=L) for L in lens], 5, draws)
            np_ref = np.random.get_state()
            assert np_after[2] == np_ref[2] and np.array_equal(np_after[1], np_ref[1]), what
            assert torch.equal(rng_after, torch.cuda.get_rng_state()), what
            assert [r["frames"] for r in got] == [[3], [8], list(range(n_past, 6))], what
            assert_same_results(got, ref, names, what)


def test_evaluate_lengths_rejects_before_any_draw():
    model = config_model("dcgan_64", 1, 2, False, 2)
    x = clip(model, 5, 2, seed=1)
    for bad, kw in (([2, 5], {}), ([], {}), ([5, 1], {}), ([5], dict(data_range=0.0)), ([5], dict(model_mode="both")),
                    ([5], dict(nsample=0))):
        st, rng = np.random.get_state(), torch.cuda.get_rng_state()
        with pytest.raises(ValueError):
            model.p2p_evaluate_lengths(x, bad, **kw)
        assert np.random.get_state()[2] == st[2] and np.array_equal(np.random.get_state()[1], st[1])
        assert torch.equal(torch.cuda.get_rng_state(), rng)


# ---- 2. the fold kernel alone ------------------------------------------------------------------------------------------------
def synthetic(n_pairs, nm, seed):
    """Scores on a grid of quarters (exact ties between sample means), with +inf, -inf and NaN sprinkled in."""
    rs = np.random.RandomState(seed)
    s = rs.randint(0, 8, (n_pairs, nm)).astype(np.float64) / 4
    s[rs.rand(n_pairs, nm) < 0.08] = math.inf
    s[rs.rand(n_pairs, nm) < 0.04] = math.nan
    s[rs.rand(n_pairs, nm) < 0.02] = -math.inf
    return s


def fold_dev(K, scores, segs, col_bin, B, ns, mask, n_bins, dev, times=1, tot=None):
    nm = scores.shape[1]
    if tot is None:
        tot = dict(sums=torch.zeros(n_bins, nm, 3, dtype=torch.float64, device=dev),
                   counts=torch.zeros(n_bins, nm, 4, dtype=torch.int64, device=dev),
                   rows=torch.zeros(n_bins, dtype=torch.int64, device=dev))
    sc = torch.from_numpy(scores).to(dev)
    sg = torch.tensor(segs, dtype=torch.int32, device=dev)
    cb = torch.tensor(col_bin, dtype=torch.int32, device=dev)
    pv = torch.empty(len(col_bin) * B * nm * 2, dtype=torch.float64, device=dev)
    pc = torch.empty(len(col_bin) * B * nm * 2, dtype=torch.int32, device=dev)
    counter = torch.zeros(1, dtype=torch.int32, device=dev)
    for _ in range(times):
        K.metrics_fold(sc, mask, B, ns, sg, cb, pv, pc, counter, tot["sums"], tot["counts"], tot["rows"])
    assert counter.item() == 0, "the ticket counter is left zero"
    return {k: v.cpu().numpy() for k, v in tot.items()}


def same_bits(a, b):
    return all(np.array_equal(a[k].view(np.int64) if a[k].dtype == np.float64 else a[k],
                              b[k].view(np.int64) if b[k].dtype == np.float64 else b[k]) for k in ("sums", "counts", "rows"))


@pytest.mark.parametrize("B,ns,nm", [(5, 4, 3), (300, 2, 3), (7, 1, 2)])
def test_fold_kernel_bit_identical_to_restatement(B, ns, nm):
    from p2pvg_b200._lib import kernels_for
    dev = torch.device("cuda")
    K = kernels_for(dev)
    # three segments (lengths) of 1, 4 and 3 frames; the third repeats the second's first bins (a duplicate length)
    Fs = [1, 4, 3]
    segs, off, c0 = [], 0, 0
    for F in Fs:
        segs.append((off, c0, F))
        off += F * B * ns
        c0 += F
    col_bin = [0, 1, 2, 3, 4, 1, 2, 5]
    n_bins = 7   # bin 6 stays empty
    mask = 0b110 if nm == 3 else 0
    s = synthetic(off, nm, seed=B + ns)
    got = fold_dev(K, s, segs, col_bin, B, ns, mask, n_bins, dev)
    ref = fold_ref(new_totals(n_bins, nm), s, segs, col_bin, B, ns, mask)
    assert same_bits(got, ref)
    assert got["counts"].sum() > 0 and got["rows"].tolist() == [B, 2 * B, 2 * B, B, B, B, 0]
    # two launches: the restatement applied twice, and run-to-run identical
    twice = fold_dev(K, s, segs, col_bin, B, ns, mask, n_bins, dev, times=2)
    assert same_bits(twice, fold_ref(fold_ref(new_totals(n_bins, nm), s, segs, col_bin, B, ns, mask), s, segs, col_bin, B, ns, mask))
    assert same_bits(twice, fold_dev(K, s, segs, col_bin, B, ns, mask, n_bins, dev, times=2))
    # the bins of the first segment folded without the others: the same bits for those bins
    alone = fold_dev(K, s[:Fs[0] * B * ns], segs[:1], col_bin[:1], B, ns, mask, n_bins, dev)
    for k in ("sums", "counts", "rows"):
        assert np.array_equal(alone[k][0], got[k][0])
        assert not alone[k][1:].any()


# ---- 3. evaluate_split against host aggregation of looped p2p_evaluate --------------------------------------------------------
def split_draws(Ts, lens_of, B, ns, z, seed):
    return [d for i, T in enumerate(Ts) for d in draws_for(lens_of(T), ns * B, z, seed + i)]


@pytest.mark.parametrize("len_outputs", [None, [4, 6]], ids=["own-length", "fixed"])
def test_evaluate_split_equals_looped_aggregation(len_outputs):
    from p2pvg_b200 import evaluate, metrics
    B, ns = 2, 3
    Ts = [6, 5, 6, 7]
    lens_of = (lambda T: [T]) if len_outputs is None else (lambda T: list(len_outputs))
    with precision("fp32"):
        model = config_model("dcgan_64", 1, 1, False, B)
        batches = [clip(model, T, B, seed=20 + i) for i, T in enumerate(Ts)]
        draws = split_draws(Ts, lens_of, B, ns, model.z_dim, seed=3)
        before = {k: v.clone() for k, v in model.state_dict().items()}
        rep = run(lambda: evaluate.evaluate_split(model, iter(batches), len(Ts), len_outputs, ns, seed=7), 4, list(draws))
        eng = model._graphed_engine()
        graphs = list(eng._graphs.items())
        again = run(lambda: evaluate.evaluate_split(model, batches, len(Ts), len_outputs, ns, seed=7), 4, list(draws))
        assert json.dumps(again) == json.dumps(rep), "two runs from the same draws give the same report"
        assert list(eng._graphs.items()) == graphs and all(G.ws_gen == eng.K.ws_gen for _, G in graphs), "no recapture"
        for k, v in model.state_dict().items():
            assert torch.equal(v, before[k]), k
        # the looped calls, aggregated on the host in float64
        names = metrics.FRAME_METRICS
        np.random.seed(4)
        tot, index = new_totals(0, 3), {}
        from p2pvg_b200.infer import eps_stream
        with eps_stream(list(draws)):
            for x, T in zip(batches, Ts):
                res = [model.p2p_evaluate(x, ns, len_output=L) for L in lens_of(T)]
                fold_results(tot, index, res, lens_of(T), ns, names)
    keys = sorted(index, key=index.get)
    ref = evaluate.build_report(keys, tot["sums"], tot["counts"], tot["rows"], names, ns, rep["config"])
    assert rep["config"]["rows"] == B * len(Ts) and rep["config"]["seed"] == 7 and rep["config"]["backbone"] == "dcgan_64"
    assert [(e["length"], e["frame"], e["rows"]) for e in rep["bins"]] == [(e["length"], e["frame"], e["rows"]) for e in ref["bins"]]
    for a, b in zip(rep["bins"] + rep["lengths"], ref["bins"] + ref["lengths"]):
        for k in names:
            for q, va in a[k].items():
                vb = b[k][q]
                assert (va is None and vb is None) or math.isclose(va, vb, rel_tol=1e-4, abs_tol=2e-5), (a["length"], k, q, va, vb)


# ---- 4. the command line --------------------------------------------------------------------------------------------------
def test_cli_on_a_weizmann_tree(tmp_path):
    from p2pvg_b200 import evaluate
    from p2pvg_b200.models.p2p_model import P2PModel
    from tests.video_tree import write_weizmann_tree
    write_weizmann_tree(str(tmp_path / "data"))
    model = config_model("dcgan_64", 3, 1, False, 2)
    o = model.opt
    o.dataset, o.data_root, o.backbone, o.image_width, o.channels = "weizmann", str(tmp_path / "data"), "dcgan", 64, 3
    for k, v in dict(g_dim=128, z_dim=10, rnn_size=256, prior_rnn_layers=1, posterior_rnn_layers=1, predictor_rnn_layers=2,
                     max_seq_len=10, delta_len=2).items():
        setattr(o, k, v)
    ckpt = str(tmp_path / "model.pth")
    model.save(ckpt, 0)
    argv = ["--ckpt", ckpt, "--nsample", "2", "--n_batches", "3", "--batch_size", "2", "--seed", "5"]
    evaluate.main(argv + ["--out", str(tmp_path / "a.json")])
    evaluate.main(argv + ["--out", str(tmp_path / "b.json")])
    a, b = (tmp_path / "a.json").read_bytes(), (tmp_path / "b.json").read_bytes()
    assert a == b, "two runs with one seed write the same report"
    # the same seed through the Python API
    states = torch.load(ckpt, weights_only=False)
    opt = states["opt"]
    from p2pvg_b200.generate import backbone_of
    opt.backbone_net = backbone_of(opt)
    m = P2PModel(2, 3, 128, 10, 256, 1, 1, 2, opt=opt).cuda()
    m.load(states=states)
    m.eval()
    import random
    random.seed(5)
    np.random.seed(5)
    torch.manual_seed(5)
    torch.cuda.manual_seed_all(5)
    batches, n = evaluate.split_batches(opt, opt.data_root, 2)
    assert n == 3   # 3 test clips long enough, 6 entries with their mirrored copies
    rep = evaluate.evaluate_split(m, batches, 3, None, 2, seed=5)
    assert json.loads(a) == json.loads(json.dumps(rep))
    assert rep["config"]["batches"] == 3 and rep["config"]["rows"] == 6
    assert {e["length"] for e in rep["lengths"]} <= set(range(6, 11))
