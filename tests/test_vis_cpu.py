"""p2pvg_b200.visualize without a GPU: the tile planner and a torch statement of p2pvg_vis_canvas (tests/vis_ref.py) against
the reference's own vis_seq pictures (tests/golden/vis_seq.pt, written by make_golden_vis.py), bit for bit, for every case
whose samples the fixture can redraw (the composition cases and the poses); the NumPy draws the planner makes; and the drop-in
misc/visualize.py's name resolution."""
import hashlib
import importlib
import os
import sys
import types

import numpy as np
import pytest
import torch

from p2pvg_b200 import visualize as V
from tests.vis_ref import FrameSource, PoseStub, case_input, compose_ref, compose_tiles

FIX = os.path.join(os.path.dirname(__file__), "golden", "vis_seq.pt")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.fixture(scope="module")
def fix():
    return torch.load(FIX, weights_only=False)


def refs(c):
    """(gt_ref, sample_ref) of a fixture case as vis_seq lays out its stores: for poses one store of the sample images, then
    the ground truth's; for frames the ground truth in store 0 and the samples [nsample, L, n_block] in store 1."""
    ns, L, nb = c["nsample"], c["spec"]["L"], c["n_block"]
    if c["spec"]["net"] == "mlp":
        g0 = ns * L * nb
        return (lambda t: (0, g0 + t * nb)), (lambda s, t: (0, (s * L + t) * nb))
    return (lambda t: (0, t * nb)), (lambda s, t: (1, (s * L + t) * nb))


def stores(c):
    """(store0, store1, C, H) of a case whose samples the fixture redraws: the poses' rendered images, or the FrameSource
    frames of a composition case."""
    ns, L, nb, T = c["nsample"], c["spec"]["L"], c["n_block"], c["spec"]["T"]
    x = case_input(c["spec"])
    if c["spec"]["net"] == "mlp":
        stub = PoseStub()
        imgs = [stub.set_data(p, v) for p, v in c["set_data"]]          # samples (s, b), then the ground truth (b)
        a = lambda ims: np.stack(ims, 1).astype(np.float64) / 255.     # noqa: E731  [T, nb, S, S, 3]
        per = [a(imgs[s * nb:(s + 1) * nb]) for s in range(ns)] + [a(imgs[ns * nb:])]
        store = torch.cat([torch.from_numpy(p.astype(np.float32)).permute(0, 1, 4, 2, 3).reshape(-1, 3, *p.shape[2:4])
                           for p in per]).contiguous()
        return store, None, 3, int(store.shape[-1])
    C = c["spec"]["channels"]
    s0 = x[:, :nb].reshape(T * nb, C, 64, 64).contiguous()
    smp = FrameSource(c["spec"]["src_seed"], c["spec"]["zero"]).samples(x, ns, L)
    s1 = smp[:, :, :nb].reshape(ns * L * nb, C, 64, 64).contiguous()
    return s0, s1, C, 64


def exact_cases(fix):
    return [c for c in fix["cases"] if c["spec"]["net"] in ("mlp", "source")]


def plan(c, gt_ref, sample_ref):
    np.random.seed(c["np_seed"])
    for _ in range(c["nsample"]):
        np.random.uniform(0, 1, c["spec"]["L"] - 1)
    return V.plan_tiles(c["spec"]["T"], c["spec"]["L"], c["n_block"], c["nsample"], gt_ref, sample_ref)


def test_planner_and_kernel_statement_match_reference(fix):
    assert len(exact_cases(fix)) == 4
    for c in exact_cases(fix):
        s0, s1, C, H = stores(c)
        tiles = plan(c, *refs(c))
        canvas, video, gif = compose_tiles(s0, s1, tiles, C, H)
        assert tuple(canvas.shape) == c["canvas"]["shape"] and sha(canvas.numpy()) == c["canvas"]["sha"], c["case"]
        assert (1, *video.shape) == c["video"]["shape"] and sha(video.numpy()) == c["video"]["sha"], c["case"]
        assert gif.shape == c["gif"]["shape"] and gif.dtype == np.uint8 and sha(gif) == c["gif"]["sha"], c["case"]


def test_restated_composition_matches_reference(fix):
    """compose_ref (the GPU tests' and the benchmark's reference) against the fixture."""
    for c in exact_cases(fix):
        s0, s1, C, H = stores(c)
        ns, L, nb, T = c["nsample"], c["spec"]["L"], c["n_block"], c["spec"]["T"]
        if s1 is None:
            gt = s0[ns * L * nb:].view(-1, nb, C, H, H)[:T]
            smp = s0[:ns * L * nb].view(ns, L, nb, C, H, H)
        else:
            gt, smp = s0.view(T, nb, C, H, H), s1.view(ns, L, nb, C, H, H)
        canvas, video, gif = compose_ref(gt, smp, T, L, c["s_lists"])
        assert sha(canvas.numpy()) == c["canvas"]["sha"] and sha(video.numpy()) == c["video"]["sha"] and sha(gif) == c["gif"]["sha"]


def test_planner_draws(fix):
    """One randint(nsample, size=4) per block, in block order, after the nsample skip draws: the s_lists and the NumPy state
    afterwards are the reference's, for every case."""
    for c in fix["cases"]:
        gt_ref, sample_ref = refs(c)
        tiles = plan(c, gt_ref, sample_ref)
        st = np.random.get_state()
        ref = c["np_state_after"]
        assert st[0] == ref[0] and np.array_equal(st[1], ref[1]) and st[2:] == ref[2:]
        L = c["spec"]["L"]
        for i, sl in enumerate(c["s_lists"]):
            for j, s in enumerate(sl):
                want = sample_ref(s, 0)
                assert tuple(tiles[0, i, j + 1, :2]) == (want[0], want[1] + i)
                want = sample_ref(s, L - 1)
                assert tuple(tiles[-1, i, j + 1, :2]) == (want[0], want[1] + i)


def test_names_and_tags(fix):
    for c in fix["cases"]:
        opt = types.SimpleNamespace(log_dir="LOGDIR")
        assert V.file_names(opt, 7, c["spec"]["L"], c["spec"]["mode"], c["spec"]["recon"]) == c["names"]
        assert V.tags(c["spec"]["L"], c["spec"]["mode"], c["spec"]["recon"]) == c["tags"]
        assert c["steps"] == (7, 7) and c["fps"] == 2


def test_plan_tiles_layout():
    """Borders and padding: gt red from seq_len - 1 on, samples red from output_len - 1 on, zero frames as frame -1."""
    np.random.seed(0)
    t = V.plan_tiles(4, 6, 1, 2, lambda f: (0, 10 * f), lambda s, f: None if f == 2 else (1, 100 * s + f))
    assert [tuple(v) for v in t[:, 0, 0]] == [(0, 0, 1), (0, 10, 0), (0, 20, 0), (0, 30, 2), (0, 30, 2), (0, 30, 2)]
    assert tuple(t[2, 0, 1]) == (0, -1, 0) and tuple(t[5, 0, 1]) == (1, 105, 2) and tuple(t[0, 0, 1]) == (1, 100, 1)
    np.random.seed(0)
    t = V.plan_tiles(6, 4, 1, 2, lambda f: (0, f), lambda s, f: (1, f))
    assert t.shape == (6, 1, 6, 3)
    assert [tuple(v) for v in t[:, 0, 1]] == [(1, 0, 1), (1, 1, 0), (1, 2, 0), (1, 3, 2), (1, 3, 2), (1, 3, 2)]
    assert [int(v) for v in t[:, 0, 0, 2]] == [1, 0, 0, 0, 0, 2]


def test_dropin_resolves_names(tmp_path, monkeypatch):
    """vis_seq is the drop-in's; every other name comes from the reference's file, loaded by path."""
    ref = tmp_path / "ref" / "misc"
    ref.mkdir(parents=True)
    (ref / "__init__.py").write_text("")
    (ref / "visualize.py").write_text("def vis_seq(*a, **k):\n    return 'reference'\n\ndef add_gt_cp_border(s, *a):\n"
                                      "    return 'gt'\n\ndef save_utils(*a, **k):\n    return 'save'\n")
    monkeypatch.setenv("P2PVG_REF", str(tmp_path / "ref"))
    monkeypatch.syspath_prepend(os.path.join(ROOT, "dropin"))
    for m in [m for m in sys.modules if m == "misc" or m.startswith("misc.")]:
        monkeypatch.delitem(sys.modules, m)
    vis = importlib.import_module("misc.visualize")
    assert os.path.dirname(vis.__file__) == os.path.join(ROOT, "dropin", "misc")
    assert vis.add_gt_cp_border(None) == "gt" and vis.save_utils() == "save"
    # a model the fast path rejects (no p2pvg_b200 P2PModel) goes to the reference's vis_seq
    model = types.SimpleNamespace(opt=types.SimpleNamespace(dataset="mnist", nsample=20, batch_size=4))
    assert vis.vis_seq(model, None, 0, 5, opt=model.opt) == "reference"
    assert vis.vis_seq.__module__ == "misc.visualize"
    for m in [m for m in sys.modules if m == "misc" or m.startswith("misc.")]:
        del sys.modules[m]
