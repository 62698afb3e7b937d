"""Pose generation without a GPU: the CPU oracle's p2p_generate(width="mlp") against the poses the reference's own
P2PModel.p2p_generate wrote (tests/golden/pose_gen_h36m.pt, h36m_mlp backbone, rnn_size 512), and the ctypes mirrors of the
p2pvg_pose_mlp argument structs against include/p2pvg_b200.h.

Tolerance: both sides are fp32 PyTorch on the CPU with the same weights and draws; only summation orders may differ, so
generated poses (std about 3 at the input, about 0.3 at the decoder output) agree to 1e-5 absolute.  Skipped frames are
exact zeros and teacher-forced / first frames are the inputs themselves."""
import os

import pytest
import torch

from oracle import p2p_oracle as O
from p2pvg_b200 import _lib
from tests.test_c_abi_layout import test_ctypes_struct_matches_the_header as struct_matches_header
from tests.test_oracle_golden import check_digest

GOLD = os.path.join(os.path.dirname(__file__), "golden")
FIX = os.path.join(GOLD, "pose_gen_h36m.pt")
ATOL = 1e-5


def load():
    return torch.load(FIX, weights_only=False)


def oracle_state(fix):
    return O.build_state(fix["cfg"], seed=fix["init_seed"])


@pytest.mark.parametrize("case", range(2))
def test_oracle_reproduces_reference_pose_generation(case):
    fix = load()
    c = fix["cases"][case]
    state = oracle_state(fix)
    for m, digs in c["init_digest"].items():   # same seed -> the reference's initial weights
        for k, d in digs.items():
            check_digest(state[m][k], d, 0.0, 0.0, f"{m}.{k}")
    x, L = c["x"], c["len_output"]
    assert L > len(x), "the fixture must run past the ground truth (posterior on h_cpaw)"
    for r in c["runs"]:
        got = O.p2p_generate(state, list(x), L, c["eval_cp_ix"], c["opt"], "mlp", r["eps"], r["probs"].numpy(),
                             model_mode=r["model_mode"], skip_frame=r["skip_frame"])
        what = f"{c['case']} {r['model_mode']}/skip_frame={r['skip_frame']}"
        assert len(got) == L == r["poses"].shape[0], what
        for i, (a, b) in enumerate(zip(got, r["poses"])):
            if r["zero_frames"][i]:
                assert torch.equal(a, torch.zeros_like(a)), f"{what} frame {i}"
            else:
                assert (a - b).abs().max().item() <= ATOL, f"{what} frame {i}: {(a - b).abs().max().item():.3e}"
        assert torch.equal(got[0], x[0])


def test_fixture_covers_the_issue_cases():
    fix = load()
    assert fix["cfg"]["g_dim"] == 128 and fix["cfg"]["z_dim"] == 10 and fix["cfg"]["rnn_size"] == 512
    seen = {(c["opt"]["n_past"], c["opt"]["last_frame_skip"], r["model_mode"], r["skip_frame"]) for c in fix["cases"] for r in c["runs"]}
    for n_past, lfs in ((1, False), (2, True)):
        for mode in ("full", "posterior", "prior"):
            for skip in (False, True):
                assert (n_past, lfs, mode, skip) in seen
    assert any(any(r["zero_frames"]) for c in fix["cases"] for r in c["runs"]), "no run skips a frame"


@pytest.mark.parametrize("c_name,py_struct", [("p2pvg_pose_residual", _lib.PoseResidual), ("p2pvg_pose_mlp_args", _lib.PoseMlpArgs)])
def test_pose_mlp_structs_match_the_header(tmp_path, c_name, py_struct):
    struct_matches_header(tmp_path, c_name, py_struct)


def _model(backbone, rnn_size=64, dataset="h36m"):
    import types
    from p2pvg_b200.models.p2p_model import P2PModel
    opt = types.SimpleNamespace(dataset=dataset, backbone_net=backbone, lr=1e-3, beta1=0.9, beta=1e-4, weight_cpc=100.0,
                                weight_align=0.5, skip_prob=0.5, n_past=1, last_frame_skip=False, batch_size=2)
    return P2PModel(2, 1, 32, 4, rnn_size, 1, 1, 2, opt=opt)


@pytest.mark.parametrize("which", ["vgg_64", "training", "image_frames", "flat_frames", "rnn_size_32", "rnn_size_516",
                                   "rnn_size_520"])
def test_graphed_pose_generation_rejects_before_capture(which):
    """Everything p2p_generate_graphed cannot run raises ValueError naming p2p_generate before any device work (these
    models live on the CPU, so anything later would fail differently)."""
    from p2pvg_b200.models import h36m_mlp, vgg_64
    poses = [torch.zeros(2, 17, 3) for _ in range(3)]
    x = poses
    if which == "vgg_64":
        model = _model(vgg_64, dataset="mnist").eval()
    elif which == "training":
        model = _model(h36m_mlp).train()
    elif which.startswith("rnn_size"):
        model = _model(h36m_mlp, rnn_size=int(which.split("_")[-1])).eval()
    else:
        model = _model(h36m_mlp).eval()
        x = [torch.zeros(2, 1, 64, 64)] * 3 if which == "image_frames" else [torch.zeros(2, 51)] * 3
    with pytest.raises(ValueError, match="p2p_generate"):
        model.p2p_generate_graphed((None, x, None) if which == "training" else x, 4, 3)
