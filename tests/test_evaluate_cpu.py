"""evaluate_split's host side without a GPU: the pair plan over the lengths engine's layout (metrics.plan_pairs_lengths)
against looped plan_pairs calls, the fold's bin tables for dynamic-length batch sequences, the float64 restatement of
p2pvg_metrics_fold (tests/eval_ref.py) on +inf, NaN and ties, the report built from restated totals, and the command
line's rejections."""
import argparse
import json
import math

import numpy as np
import pytest
import torch

from p2pvg_b200 import evaluate, metrics
from tests.eval_ref import best_ref, fold_ref, new_totals


# ---- the pair plan over the lengths layout ---------------------------------------------------------------------------------
@pytest.mark.parametrize("nsample", [1, 5])
@pytest.mark.parametrize("n_past", [1, 2])
@pytest.mark.parametrize("lens", [[6], [4, 6, 9], [9, 3, 6, 9], [3, 4]], ids=["T", "below-T-above", "dup", "below"])
def test_plan_pairs_lengths_selects_the_looped_rows(lens, n_past, nsample):
    """For every (length, frame, row, sample): the output row the lengths replay decodes that frame into, and the same
    ground-truth row, as the looped plan_pairs call on its own one-length store."""
    T, B = 6, 3
    lens = [L for L in lens if L > n_past]
    grows = nsample * B
    rows = len(lens) * grows
    # row group of each caller index: longest first, ties in caller order (written out independently of lengths_order)
    group = {k: sum(1 for q in range(len(lens)) if lens[q] > lens[k] or (lens[q] == lens[k] and q < k)) for k in range(len(lens))}
    frames, pairs, offsets = metrics.plan_pairs_lengths(lens, T, n_past, nsample, B)
    assert pairs.dtype == torch.int32 and offsets[0] == 0
    n = 0
    for k, L in enumerate(lens):
        fk, pk = metrics.plan_pairs(L, T, n_past, nsample, B)
        assert frames[k] == fk and offsets[k] == n
        got = pairs[n:n + len(pk)]
        n += len(pk)
        assert torch.equal(got[:, 1], pk[:, 1])
        for (r_loop, _), (r_len, _) in zip(pk.tolist(), got.tolist()):
            f, s, b = r_loop // grows, r_loop % grows // B, r_loop % B
            assert r_len == f * rows + group[k] * grows + s * B + b
            i = f + n_past   # the decode step: every group whose length exceeds i is active, a prefix of the rows
            assert i < L and r_len % rows < grows * sum(1 for L2 in lens if L2 > i)
    assert n == len(pairs)


# ---- the bin tables --------------------------------------------------------------------------------------------------------
def tables_for(seq, len_outputs, n_past=1, nsample=2, B=2):
    index, out = {}, []
    for T in seq:
        lens = [T] if len_outputs is None else list(len_outputs)
        frames, pairs, offsets = metrics.plan_pairs_lengths(lens, T, n_past, nsample, B)
        segs, col_bin = evaluate.plan_bins(lens, frames, offsets, index)
        out.append((lens, frames, segs, col_bin, len(pairs)))
    return index, out


def test_bins_of_dynamic_length_batches_own_length():
    index, out = tables_for([8, 6, 8, 7], None)
    assert list(index) == [(8, f) for f in range(1, 8)] + [(6, f) for f in range(1, 6)] + [(7, f) for f in range(1, 7)]
    assert list(index.values()) == list(range(len(index)))
    for lens, frames, segs, col_bin, n_pairs in out:
        (T,) = lens
        assert segs == [(0, 0, T - 1)] and col_bin == [index[(T, f)] for f in range(1, T)] and n_pairs == (T - 1) * 2 * 2
    assert out[0][3] == out[2][3], "a repeated T folds into the same bins"


def test_bins_of_fixed_lengths_over_dynamic_batches():
    """A length equal to the batch's T scores its frames; otherwise only its control point, in the bin (L, L - 1), which
    the full scoring of that length shares."""
    index, out = tables_for([8, 6, 5], [5, 8], nsample=3, B=2)
    lens, frames, segs, col_bin, n_pairs = out[0]   # T = 8: 5 control point only, 8 every frame
    assert frames == [[4], list(range(1, 8))]
    assert segs == [(0, 0, 1), (1 * 2 * 3, 1, 7)] and n_pairs == 8 * 2 * 3
    assert col_bin == [index[(5, 4)]] + [index[(8, f)] for f in range(1, 8)]
    _, frames, segs, col_bin, _ = out[1]             # T = 6: both control point only
    assert frames == [[4], [7]] and col_bin == [index[(5, 4)], index[(8, 7)]]
    _, frames, _, col_bin, _ = out[2]                # T = 5: 5 every frame
    assert frames == [[1, 2, 3, 4], [7]]
    assert col_bin == [index[(5, f)] for f in range(1, 5)] + [index[(8, 7)]]
    assert len(index) == 1 + 7 + 3


def test_duplicate_lengths_share_bins():
    index, out = tables_for([6], [6, 6, 4])
    _, frames, segs, col_bin, _ = out[0]
    assert col_bin[:5] == col_bin[5:10] and len(index) == 6


# ---- the restatement -------------------------------------------------------------------------------------------------------
def test_best_ref_is_best_of_on_ties_inf_and_nan():
    """best_ref against metrics.best_of (torch's argmax / argmin) on values whose sums are exact: ties, +inf means, NaN
    means, and -inf meeting +inf."""
    rs = np.random.RandomState(0)
    inf, nan = math.inf, math.nan
    for trial in range(200):
        ns, F, B = rs.randint(1, 6), rs.randint(1, 5), 4
        v = rs.randint(0, 4, (ns, F, B)).astype(np.float64) / 4
        if trial % 3 == 0:
            v[rs.rand(ns, F, B) < 0.15] = inf
        if trial % 5 == 0:
            v[rs.rand(ns, F, B) < 0.1] = nan
        if trial % 7 == 0:
            v[rs.rand(ns, F, B) < 0.1] = -inf
        t = torch.from_numpy(v)
        for k in ("psnr", "mse"):
            idx, _ = metrics.best_of({k: t}, [k])[k]
            for b in range(B):
                assert best_ref(v[:, :, b].tolist(), metrics.HIGHER_IS_BETTER[k]) == int(idx[b]), (trial, k, b)


def test_fold_ref_counts_inf_and_nan_apart():
    ns, B, F = 2, 2, 2
    # pairs (frame j, row b, sample s) at (j * B + b) * ns + s; one metric (psnr, higher is better)
    v = np.array([[10.0], [math.inf], [12.0], [11.0], [math.nan], [14.0], [13.0], [15.0]])
    tot = fold_ref(new_totals(2, 1), v, [(0, 0, F)], [0, 1], B, ns, 1)
    # row 0: sample means (10 + nan) / 2 = nan, (inf + 14) / 2 = inf -> the NaN mean wins: sample 0
    # row 1: (12 + 13) / 2 = 12.5, (11 + 15) / 2 = 13 -> sample 1
    assert tot["rows"].tolist() == [2, 2]
    assert tot["sums"][0, 0].tolist() == [10.0 + 11.0, 10.0 ** 2 + 11.0 ** 2, 10.0 + 12.0 + 11.0]
    assert tot["counts"][0, 0].tolist() == [0, 0, 1, 0]
    assert tot["sums"][1, 0].tolist() == [15.0, 225.0, 14.0 + 13.0 + 15.0]
    assert tot["counts"][1, 0].tolist() == [0, 1, 0, 1]


def test_fold_ref_is_order_fixed_and_bins_independent():
    """Two bins folded in one launch or one each: the same totals, bit for bit."""
    rs = np.random.RandomState(1)
    ns, B = 3, 4
    s = rs.rand(2 * B * ns + 3 * B * ns, 2)
    segs = [(0, 0, 2), (2 * B * ns, 2, 3)]
    both = fold_ref(new_totals(5, 2), s, segs, [0, 1, 2, 3, 4], B, ns, 2)
    a = fold_ref(new_totals(5, 2), s, segs[:1], [0, 1], B, ns, 2)
    b = fold_ref(new_totals(5, 2), s[2 * B * ns:], [(0, 0, 3)], [2, 3, 4], B, ns, 2)
    for k in ("sums", "counts", "rows"):
        assert np.array_equal(both[k][:2], a[k][:2]) and np.array_equal(both[k][2:], b[k][2:])


# ---- the report ------------------------------------------------------------------------------------------------------------
def test_report_from_restated_totals():
    ns, B = 2, 3
    names = metrics.FRAME_METRICS
    index = {}
    frames, pairs, offsets = metrics.plan_pairs_lengths([4, 6], 6, 1, ns, B)
    segs, col_bin = evaluate.plan_bins([4, 6], frames, offsets, index)
    rs = np.random.RandomState(2)
    s = rs.rand(len(pairs), 3)
    s[0, 1] = s[1, 1] = math.inf   # row 0 of length 4's control point: both samples identical to the ground truth
    tot = fold_ref(new_totals(len(index), 3), s, segs, col_bin, B, ns, evaluate.higher_mask(names))
    keys = sorted(index, key=index.get)
    cfg = dict(nsample=ns, lengths=[4, 6])
    rep = evaluate.build_report(keys, tot["sums"], tot["counts"], tot["rows"], names, ns, cfg)
    json.dumps(rep, allow_nan=False)
    assert rep["config"] == cfg and rep["metrics"] == list(names)
    assert [(e["length"], e["frame"]) for e in rep["bins"]] == [(4, 3)] + [(6, f) for f in range(1, 6)]
    cp4 = rep["bins"][0]
    u = index[(4, 3)]
    assert cp4["rows"] == B and cp4["psnr"]["best_inf_share"] == 1 / B and cp4["psnr"]["inf_share"] == 2 / (B * ns)
    assert cp4["psnr"]["best_mean"] == tot["sums"][u, 1, 0] / (B - 1)
    m = tot["sums"][u, 0, 0] / B
    sem = math.sqrt(max((tot["sums"][u, 0, 1] - tot["sums"][u, 0, 0] * m) / (B - 1), 0) / B)
    assert cp4["mse"]["best_mean"] == m and math.isclose(cp4["mse"]["best_sem"], sem, rel_tol=1e-12)
    assert cp4["mse"]["mean"] == tot["sums"][u, 0, 2] / (B * ns)
    L6 = rep["lengths"][1]
    us = [index[(6, f)] for f in range(1, 6)]
    assert L6["frames"] == list(range(1, 6))
    assert L6["ssim"]["best_mean_over_frames"] == sum(float(tot["sums"][q, 2, 0]) for q in us) / (5 * B)
    assert L6["ssim"]["control_point"] == rep["bins"][-1]["ssim"]["best_mean"]
    assert rep["lengths"][0]["psnr"]["control_point"] == cp4["psnr"]["best_mean"]
    assert rep["psnr_inf_share"] == dict(best=1 / (6 * B), samples=2 / (6 * B * ns))


def test_report_without_finite_values_gives_none():
    tot = new_totals(1, 1)
    tot["rows"][0] = 2
    tot["counts"][0, 0] = [2, 0, 4, 0]
    rep = evaluate.build_report([(5, 4)], tot["sums"], tot["counts"], tot["rows"], ("psnr",), 2, {})
    e = rep["bins"][0]["psnr"]
    assert e["best_mean"] is None and e["best_sem"] is None and e["mean"] is None and e["best_inf_share"] == 1.0
    json.dumps(rep, allow_nan=False)


# ---- the command line ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("argv", [[], ["--ckpt", "m.pth", "--nsample", "0"], ["--ckpt", "m.pth", "--n_batches", "0"],
                                  ["--ckpt", "m.pth", "--batch_size", "-1"], ["--ckpt", "m.pth", "--lengths", "1", "5"],
                                  ["--ckpt", "m.pth", "--lengths"], ["--ckpt", "m.pth", "--seed", "x"]])
def test_cli_rejects_bad_arguments(argv, capsys):
    with pytest.raises(SystemExit) as e:
        evaluate.parse_args(argv)
    assert e.value.code == 2


def test_cli_defaults():
    a = evaluate.parse_args(["--ckpt", "m.pth"])
    assert (a.nsample, a.lengths, a.n_batches, a.batch_size, a.seed, a.out) == (20, None, None, None, 1, "report.json")
    assert evaluate.parse_args(["--ckpt", "m.pth", "--lengths", "10", "20", "30"]).lengths == [10, 20, 30]


def test_cli_refuses_h36m_and_names_the_python_api(tmp_path):
    ckpt = str(tmp_path / "h36m.pth")
    torch.save(dict(opt=argparse.Namespace(dataset="h36m")), ckpt)
    with pytest.raises(SystemExit) as e:
        evaluate.main(["--ckpt", ckpt, "--out", str(tmp_path / "r.json")])
    assert "evaluate_split" in str(e.value) and "PoseBatches" in str(e.value)
    assert not (tmp_path / "r.json").exists()
    with pytest.raises(ValueError, match="unknown dataset"):
        evaluate.check_dataset(argparse.Namespace(dataset="kth"))


def test_evaluate_split_rejects_bad_counts():
    for kw in (dict(n_batches=0), dict(n_batches=1.5), dict(n_batches=2, nsample=0), dict(n_batches=True)):
        with pytest.raises(ValueError):
            evaluate.evaluate_split(None, iter([]), **kw)
