"""Host side of P2PModel.p2p_generate_multi_cp and p2p_evaluate(cp_ixs=...) (p2pvg_b200/gen_engine.py, metrics.py), no GPU
needed: the multi-segment slot planner against plan_slots per segment, every per-slot table entry against the looped
calls' own tables, the scored-pair plan, and the ValueErrors raised before any draw or launch."""
import types

import numpy as np
import pytest
import torch

from p2pvg_b200 import metrics
from p2pvg_b200.gen_engine import check_cp_ixs, plan_segments, plan_slots


def single_call_tables(slots, T, n_past, len_output, model_mode):
    """The per-slot tables one generate call on x_k (len(x_k) = T) builds: (tab_i, tab_h, tab_z, glob, tuc, dt) with the
    autoregressive h row numbered T."""
    n_tf = min(n_past - 1, len_output - 1)
    tab_h = [s if s <= n_tf else T for s in range(len(slots))]
    tab_i = [t if t >= 0 else tab_h[s] for s, (_, _, _, t) in enumerate(slots)]
    tab_z = [0 if (model_mode == "posterior" or (s < n_tf and model_mode == "full")) else 1 for s in range(len(slots))]
    return tab_i, tab_h, tab_z, T - 1, [t for (_, t, _, _) in slots], [d for (_, _, d, _) in slots]


@pytest.mark.parametrize("model_mode", ["full", "posterior", "prior"])
@pytest.mark.parametrize("skip_frame", [False, True])
@pytest.mark.parametrize("n_past", [1, 2, 3])
def test_plan_segments_is_the_concatenation_of_plan_slots(n_past, skip_frame, model_mode):
    rng = np.random.RandomState(10 * n_past + skip_frame)
    for _ in range(100):
        K = int(rng.randint(1, 5))
        T_k = [int(rng.randint(max(n_past, 2), 9)) for _ in range(K)]
        cps = [0]
        for t in T_k:
            cps.append(cps[-1] + t - 1)
        T = cps[-1] + 1 + int(rng.randint(0, 3))
        L_k = [t if rng.rand() < 0.5 else int(rng.randint(max(2, min(n_past, t)), 12)) for t in T_k]
        L_k = [max(L, 2) if t >= min(n_past, L) else t for L, t in zip(L_k, T_k)]
        segs = check_cp_ixs(cps, T, L_k, n_past)
        assert [(o, Tk, Lk) for (o, Tk, Lk, _) in segs] == list(zip(cps, T_k, L_k))
        skip_prob = float(rng.choice([0.0, 0.5, 0.9]))
        probs = [rng.uniform(0, 1, Lk - 1) for Lk in L_k]
        Tc = cps[-1] + 1
        slots, ints, fl = plan_segments(segs, Tc, probs, skip_prob, n_past, skip_frame, model_mode)
        S = sum(len(s) for s in slots)
        assert len(ints) == 4 * S and len(fl) == 2 * S
        tab = [ints[j * S:(j + 1) * S] for j in range(4)]
        tuc, dt = fl[:S], fl[S:]
        s0 = 0
        for k, (o, Tk, Lk, cp) in enumerate(segs):
            ref = plan_slots(Lk, Tk, probs[k], skip_prob, n_past, skip_frame, Lk - 1)
            assert cp == Lk - 1 and slots[k] == ref
            ri, rh, rz, rg, rt, rd = single_call_tables(ref, Tk, n_past, Lk, model_mode)
            n = len(ref)
            sl = slice(s0, s0 + n)
            # clip frame o + f for a ground-truth frame f of x_k; the autoregressive row T_k of the single call is Tc here
            clip = [Tc if v == Tk else o + v for v in rh]
            assert tab[1][sl] == clip, k
            assert tab[0][sl] == [Tc if v == Tk else o + v for v in ri], k
            assert tab[2][sl] == rz, k
            assert tab[3][sl] == [o + rg] * n, k
            assert [a.hex() for a in tuc[sl]] == [a.hex() for a in rt] and [a.hex() for a in dt[sl]] == [a.hex() for a in rd]
            s0 += n
        assert s0 == S


def test_one_segment_tables_equal_the_single_call():
    probs = np.random.RandomState(3).uniform(0, 1, 8)
    slots, ints, fl = plan_segments([(0, 6, 9, 7)], 6, [probs], 0.5, 2, True, "full")
    ref = plan_slots(9, 6, probs, 0.5, 2, True, 7)
    ri, rh, rz, rg, rt, rd = single_call_tables(ref, 6, 2, 9, "full")
    S = len(ref)
    assert slots == [ref] and ints == ri + rh + rz + [rg] * S and fl == rt + rd


@pytest.mark.parametrize("n_past", [1, 2])
def test_plan_pairs_multi_cp(n_past):
    cps, ns, B = [0, 3, 4 + n_past, 9], 2, 3
    frames, pairs = metrics.plan_pairs_multi_cp(cps, n_past, ns, B)
    want = [i + a for a, b in zip(cps, cps[1:]) for i in range(n_past, b - a + 1)]
    assert frames == sorted(frames) == want and set(cps[1:]) <= set(frames)
    p = pairs.view(len(frames), B, ns, 2)
    for fi, f in enumerate(frames):
        for b in range(B):
            for s in range(ns):
                assert p[fi, b, s, 1].item() == f * B + b
                assert p[fi, b, s, 0].item() == (fi * ns + s) * B + b   # decodes in chain order
    # one segment is plan_pairs of the whole clip
    f1, p1 = metrics.plan_pairs_multi_cp([0, 6], n_past, ns, B)
    f2, p2 = metrics.plan_pairs(7, 7, n_past, ns, B)
    assert f1 == f2 and torch.equal(p1, p2)
    with pytest.raises(ValueError):
        metrics.plan_pairs_multi_cp([0, n_past - 1, 8], n_past, ns, B)   # a first segment of n_past frames


@pytest.mark.parametrize("cp_ixs,len_outputs,n_past", [
    ([0], None, 1), ([], None, 1), ([1, 4], None, 1), ([0, 2, 2], None, 1), ([0, 3, 2], None, 1), ([0, 6], None, 1),
    ([0, 2.5], None, 1), ([0, True], None, 1), ("04", None, 1), (None, None, 1),
    ([0, 2, 5], [4], 1), ([0, 2, 5], [4, 1], 1), ([0, 2, 5], [4, 3, 3], 1), ([0, 2, 5], [4, 2.5], 1),
    ([0, 1, 5], [4, 5], 3),   # segment 0 has 2 frames, min(n_past, L_0) = 3
    ([0, 3, 5], None, 0)])
def test_check_cp_ixs_rejects(cp_ixs, len_outputs, n_past):
    with pytest.raises(ValueError):
        check_cp_ixs(cp_ixs, 6, len_outputs, n_past)


def test_check_cp_ixs_accepts():
    assert check_cp_ixs(range(4), 4, None, 1) == [(0, 2, 2, 1), (1, 2, 2, 1), (2, 2, 2, 1)]
    assert check_cp_ixs(np.array([0, 2, 5]), 8, [9, 2], 2) == [(0, 3, 9, 8), (2, 4, 2, 1)]


def _model(n_past=1, train=False):
    from p2pvg_b200.models import dcgan_64
    from p2pvg_b200.models.p2p_model import P2PModel
    opt = types.SimpleNamespace(dataset="mnist", backbone_net=dcgan_64, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0,
                                weight_align=0.5, skip_prob=0.5, n_past=n_past, last_frame_skip=False, batch_size=2)
    model = P2PModel(2, 1, 128, 10, 64, 1, 1, 2, opt=opt)
    return model.train() if train else model.eval()


@pytest.mark.parametrize("kw", [dict(cp_ixs=[0, 2, 2]), dict(cp_ixs=[0, 7]), dict(cp_ixs=[0, 3], len_outputs=[1]),
                                dict(cp_ixs=[0, 1, 4], len_outputs=[3]), dict(cp_ixs=[0, 2], model_mode="nope"),
                                dict(cp_ixs=[0, 2], nsample=0)])
def test_generate_multi_cp_rejects_before_drawing(kw):
    """Bad arguments raise ValueError before the NumPy draw (the global stream is unchanged) and before any device work
    (the model lives on the CPU)."""
    model = _model()
    x = [torch.zeros(2, 1, 64, 64) for _ in range(5)]
    np.random.seed(0)
    with pytest.raises(ValueError):
        model.p2p_generate_multi_cp(x, **kw)
    assert np.random.uniform() == np.random.RandomState(0).uniform()


def test_generate_multi_cp_rejects_model_and_frames():
    x = [torch.zeros(2, 1, 64, 64) for _ in range(5)]
    with pytest.raises(ValueError, match="eval mode"):
        _model(train=True).p2p_generate_multi_cp(x, [0, 2, 4])
    with pytest.raises(ValueError, match="do not fit"):
        _model().p2p_generate_multi_cp([torch.zeros(2, 1, 32, 32) for _ in range(5)], [0, 2, 4])
    # a segment shorter than min(n_past, L_k)
    with pytest.raises(ValueError, match="segment 1"):
        _model(n_past=3).p2p_generate_multi_cp(x, [0, 3, 4], len_outputs=[4, 5])


def test_evaluate_cp_ixs_rejections():
    model = _model(n_past=2)
    x = torch.zeros(6, 2, 1, 64, 64)
    for kw in (dict(cp_ixs=[0, 3, 5], len_output=6),   # both
               dict(cp_ixs=[0, 1, 5]),                 # segment [0, 1] has 2 frames <= n_past: nothing to score
               dict(cp_ixs=[0, 3, 5], data_range=0.0), dict(cp_ixs=[0, 5, 3])):
        np.random.seed(1)
        with pytest.raises(ValueError):
            model.p2p_evaluate(x, **kw)
        assert np.random.uniform() == np.random.RandomState(1).uniform()
