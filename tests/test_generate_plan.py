"""Host side of P2PModel.p2p_generate_graphed (p2pvg_b200/gen_engine.py), no GPU needed: the slot planner against a
direct transcription of the reference's skip predicate (models/p2p_model.py:126-138), and the ValueError for models the
graphed path does not cover."""
import types

import numpy as np
import pytest
import torch

from p2pvg_b200.gen_engine import plan_slots


def reference_steps(len_output, len_x, probs, skip_prob, n_past, skip_frame, eval_cp_ix):
    """The generation loop's bookkeeping, statement by statement: which i execute, time_until_cp, delta_time and
    whether the posterior sees a ground-truth target."""
    prev_i, skip_count, out = 0, 0, []
    max_skip_count = len_x * skip_prob
    for i in range(1, len_output):
        if probs[i - 1] <= skip_prob and i >= n_past and skip_count < max_skip_count and i != 1 and i != (len_output - 1) and skip_frame:
            skip_count += 1
            continue
        time_until_cp = (eval_cp_ix - i + 1) / eval_cp_ix
        delta_time = (i - prev_i) / eval_cp_ix
        prev_i = i
        out.append((i, time_until_cp, delta_time, i if i < len_x else -1))
    return out


@pytest.mark.parametrize("skip_frame", [False, True])
@pytest.mark.parametrize("n_past", [1, 2, 3])
def test_plan_slots_matches_reference_predicate(n_past, skip_frame):
    rng = np.random.RandomState(100 * n_past + skip_frame)
    for _ in range(200):
        len_x = int(rng.randint(max(n_past, 2), 12))
        len_output = int(rng.randint(2, 16))
        eval_cp_ix = int(rng.randint(1, 16))
        skip_prob = float(rng.choice([0.0, 0.1, 0.5, 0.9]))
        probs = rng.uniform(0, 1, len_output - 1)
        got = plan_slots(len_output, len_x, probs, skip_prob, n_past, skip_frame, eval_cp_ix)
        ref = reference_steps(len_output, len_x, probs, skip_prob, n_past, skip_frame, eval_cp_ix)
        assert len(got) == len(ref)
        for g, r in zip(got, ref):
            assert g[0] == r[0] and g[3] == r[3]
            # bit-exact as Python doubles
            assert g[1].hex() == r[1].hex() and g[2].hex() == r[2].hex()
        # teacher-forced steps are never skipped: the first min(n_past - 1, len_output - 1) slots are i = 1, 2, ...
        n_tf = min(n_past - 1, len_output - 1)
        assert [g[0] for g in got[:n_tf]] == list(range(1, n_tf + 1))


def _model(backbone, dataset="mnist"):
    from p2pvg_b200.models.p2p_model import P2PModel
    opt = types.SimpleNamespace(dataset=dataset, backbone_net=backbone, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0,
                                weight_align=0.5, skip_prob=0.5, n_past=1, last_frame_skip=False, batch_size=2)
    return P2PModel(2, 1, 128, 10, 64, 1, 1, 2, opt=opt)


@pytest.mark.parametrize("which", ["vgg_64", "h36m_mlp", "training"])
def test_unsupported_models_raise(which):
    from p2pvg_b200.models import dcgan_64, h36m_mlp, vgg_64
    if which == "vgg_64":
        model = _model(vgg_64).eval()
    elif which == "h36m_mlp":
        model = _model(h36m_mlp, dataset="h36m").eval()
    else:
        model = _model(dcgan_64).train()
    x = [torch.zeros(2, 1, 64, 64) for _ in range(3)]
    with pytest.raises(ValueError, match="p2p_generate"):
        model.p2p_generate_graphed(x, 4, 3)
