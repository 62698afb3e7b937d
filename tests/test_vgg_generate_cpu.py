"""vgg generation without a GPU: the CPU oracle's p2p_generate(width="vgg") against the frames the reference's own
P2PModel.p2p_generate wrote (tests/golden/vgg_gen.pt: vgg_64 and vgg_128, eval-mode BatchNorm on warmed running statistics),
and the checks p2p_generate_graphed makes before any device work.

Tolerance: both sides are fp32 PyTorch on the CPU with the same weights and draws; only convolution summation orders may
differ, so frames in [0, 1] agree to 1e-5 absolute.  Skipped frames are exact zeros."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import p2p_oracle as O

GOLD = os.path.join(os.path.dirname(__file__), "golden")
FIX = os.path.join(GOLD, "vgg_gen.pt")
ATOL = 1e-5


def load():
    return torch.load(FIX, weights_only=False)


def case_frames(c):
    """The case's input frames (the fixture stores their seed: make_golden_vgg_gen.frames)."""
    g = torch.Generator().manual_seed(c["x_seed"])
    return torch.rand(*c["x_shape"], generator=g)


def case_state(c):
    """The reference's initial weights (same init seed) with the fixture's BatchNorm buffers."""
    state = O.build_state(c["cfg"], seed=c["init_seed"])
    for m, bufs in c["bn_buffers"].items():
        for k, v in bufs.items():
            state[m][k].copy_(v)
    return state


def full_frames(seq, r):
    """(generated, reference) pairs of the frames the run stores in full: the middle and last frame of the model_mode="full",
    skip_frame=False run of each case (every other frame is checked through its digest)."""
    return ((seq[-1], r["last"]), (seq[len(seq) // 2], r["mid"])) if "last" in r else ()


@pytest.mark.parametrize("case", range(3))
def test_oracle_reproduces_reference_vgg_generation(case):
    c = load()["cases"][case]
    state, x, L = case_state(c), case_frames(c), c["len_output"]
    for r in c["runs"]:
        got = O.p2p_generate(state, list(x), L, c["eval_cp_ix"], c["opt"], "vgg", r["eps"], r["probs"].numpy(),
                             model_mode=r["model_mode"], skip_frame=r["skip_frame"])
        what = f"{c['case']} {r['model_mode']}/skip_frame={r['skip_frame']}"
        assert len(got) == L, what
        assert [bool((f == 0).all()) for f in got] == r["zero_frames"], what
        for i, (f, d) in enumerate(zip(got, r["digests"])):
            v = f.double().reshape(-1)
            assert v.numel() == d["numel"], what
            assert (v[d["idx"]] - d["samples"]).abs().max().item() <= ATOL, f"{what} frame {i}"
        for f, ref in full_frames(got, r):
            assert (f - ref).abs().max().item() <= ATOL, f"{what}: {(f - ref).abs().max().item():.3e}"


def test_fixture_covers_the_issue_cases():
    cases = load()["cases"]
    shapes = {(c["cfg"]["vgg_width"], c["cfg"]["channels"], c["opt"]["n_past"], c["opt"]["last_frame_skip"]) for c in cases}
    assert {(64, 3, 1, False), (64, 1, 2, True), (128, 1, 1, False)} <= shapes
    for c in cases:
        assert {(r["model_mode"], r["skip_frame"]) for r in c["runs"]} == {(m, s) for m in ("full", "posterior", "prior")
                                                                           for s in (False, True)}
    assert any(c["len_output"] > c["x_shape"][0] for c in cases), "no case runs past the ground truth"
    assert all(sum("last" in r for r in c["runs"]) == 1 for c in cases), "each case stores one run's frames in full"
    assert any(any(r["zero_frames"]) for c in cases for r in c["runs"]), "no run skips a frame"


def _model(rnn_size=64, channels=1, width=64):
    from p2pvg_b200.models import vgg_64, vgg_128
    from p2pvg_b200.models.p2p_model import P2PModel
    opt = types.SimpleNamespace(dataset="mnist", backbone_net=vgg_128 if width == 128 else vgg_64, lr=1e-3, beta1=0.9, beta=1e-4,
                                weight_cpc=100.0, weight_align=0.5, skip_prob=0.5, n_past=1, last_frame_skip=False, batch_size=2)
    return P2PModel(2, channels, 32, 4, rnn_size, 1, 1, 2, opt=opt)


@pytest.mark.parametrize("which,match", [("training", "training mode"), ("rnn_size_32", "rnn_size"), ("rnn_size_516", "rnn_size"),
                                         ("rnn_size_520", "rnn_size"), ("channels_5", "image channels"),
                                         ("cpu", "CUDA device.*model.cuda")])
def test_graphed_vgg_generation_rejects_before_device_work(which, match):
    """Every model p2p_generate_graphed cannot run raises ValueError naming p2p_generate_graphed before any device work and
    before the NumPy skip draw (the global NumPy state is unchanged).  The models live on the CPU, so the device check
    comes last: every other rejection fires first."""
    channels = 5 if which == "channels_5" else 1
    model = _model(rnn_size=int(which.split("_")[-1]) if which.startswith("rnn_size") else 64, channels=channels)
    model.train() if which == "training" else model.eval()
    x = [torch.zeros(2, channels, 64, 64) for _ in range(3)]
    np.random.seed(17)
    before = np.random.get_state()
    with pytest.raises(ValueError, match="^p2p_generate_graphed") as e:
        model.p2p_generate_graphed(x, 4, 3, skip_frame=True)
    assert e.match(match)
    after = np.random.get_state()
    assert before[0] == after[0] and np.array_equal(before[1], after[1]) and before[2:] == after[2:]
