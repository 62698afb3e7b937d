"""The skeleton renderer's spec on the host (no GPU): the oracle's anchors and axis reversal, p2pvg_b200.skeleton's camera
matrices against the oracle's, the parents against the loader's fixture, zero-length limbs, the fp32 levels, the argument
checks made before any launch, and the drop-in ``human36m`` module."""
import importlib
import os
import sys
import textwrap

import numpy as np
import pytest
import torch

from p2pvg_b200 import skeleton as S
from tests import skeleton_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_oracle_anchors():
    for limit in ((-6, 6), [-6.0, 6.0]):
        M = R.matrices(limit)
        for v in range(4):
            assert np.allclose(R.project_rc(M[v], (0, 0, 0)), (47.27, 50.73), atol=5e-3)
            assert np.allclose(R.project_rc(M[v], (0, -3, 0)), (30.45, 50.73), atol=5e-3)   # the head is up
            corners = np.array([R.project_rc(M[v], (x, y, z)) for x in (-6, 6) for y in (-6, 6) for z in (-6, 6)])
            assert (corners > 0).all() and (corners < R.OUT).all()


def test_world_matrix_reverses_x_and_z():
    W = R.world((-6, 6))
    to = lambda p: (W @ np.array([*p, 1.0]))[:3]  # noqa: E731
    assert np.allclose(to((6, -6, 6)), 0) and np.allclose(to((-6, 6, -6)), 1)
    assert np.allclose(to((0, 0, 0)), 0.5)
    assert W[0, 0] < 0 and W[1, 1] > 0 and W[2, 2] < 0


def test_camera_matrices_equal_the_oracles():
    for limit in ((-6, 6), (0.0, 1.0), (-2.5, 4)):
        assert np.allclose(S.camera_matrices(limit), R.matrices(limit), rtol=0, atol=1e-12)
    k = S.kernel_matrices((-6, 6))
    assert k.dtype == np.float32 and k.shape == (4, 3, 4)
    assert np.allclose(k, R.matrices((-6, 6))[:, [0, 1, 3]], rtol=1e-7, atol=1e-12)
    M = S.camera_matrices((-6, 6))
    assert np.array_equal(M[0], M[1]) and np.array_equal(M[2], M[3]) and not np.allclose(M[0], M[2])


def test_parents_are_the_loaders():
    fix = torch.load(os.path.join(ROOT, "tests", "golden", "pose_data_ref.pt"), weights_only=False)
    for split in ("train", "test"):
        assert list(S.H36M_PARENTS) == fix[split]["parents"] == R.PARENTS


def test_limb_colours():
    c = S.limb_colors(16)
    assert np.array_equal(c, R.colors(16))
    assert [tuple(c[l]) for l in (0, 3, 6, 13)] == [(1, 0, 0), (0, 0, 1), (0, 0.5, 0), (1, 0, 0)]


def test_zero_length_limbs_draw_nothing():
    u8, f = R.render(np.zeros((2, 17, 3)), [0, 2])
    assert (u8 == 255).all() and (f == 1).all()
    assert R.coverage(np.array([40.0, 60.0]), np.array([40.0, 60.0 + 5e-7])) is None
    k = R.coverage(np.array([40.0, 60.0]), np.array([40.0, 60.0 + 1e-3]))
    assert k is not None and k.sum() > 0   # a dot: the projecting caps make a square of side 2h


def test_coverage_of_a_horizontal_limb():
    # from display (40, 60) to (60, 60): the rectangle x in [40 - h, 60 + h], y in [60 - h, 60 + h]
    # h = 4/3: a pixel whose samples lie 1 + (i + .5) / 8 from an edge has 3 of 8 sample lines inside
    k = R.coverage(np.array([40.0, 60.0]), np.array([60.0, 60.0]))
    r = R.FIG - 1 - 60 - R.CROP                         # the row covering y in [60, 61)
    c = 50 - R.CROP
    assert [k[r + d, c] for d in (-2, -1, 0, 1, 2, 3)] == [0, 24, 64, 64, 24, 0]
    assert [k[r, x - R.CROP] for x in (37, 38, 39, 40, 60, 61, 62)] == [0, 24, 64, 64, 64, 24, 0]
    assert k.sum() == 182 * 22   # sample columns 38 + 5/8 .. 61 + 3/8 by sample rows 58 + 5/8 .. 61 + 3/8


def test_levels_are_float32_of_q_over_255():
    q = np.arange(256)
    want = np.array([np.float32(v / 255.) for v in q])
    assert np.array_equal(R.levels(), want)
    # what the reference's pictures become in vis_seq: uint8 -> float64 / 255 -> float32
    assert np.array_equal((q.astype(np.uint8).astype(np.float64) / 255.).astype(np.float32), want)


def test_argument_checks():
    with pytest.raises(ValueError, match="joints"):
        S.check_parents([-1] + list(range(32)))                   # J = 33
    for bad in ([0, 0, 1], [-1, 1, 1], [-1, 0, 2], [-1, -1, 0], [-1]):
        with pytest.raises(ValueError):
            S.check_parents(bad)
    assert S.check_parents(S.H36M_PARENTS).dtype == np.int32
    with pytest.raises(ValueError, match="autoscaling"):
        S.Skeleton3DVisualizer(S.H36M_PARENTS, plot_3d_limit=None)
    vis = S.Skeleton3DVisualizer(S.H36M_PARENTS, plot_3d_limit=[-6, 6])
    vis.plot_3d_limit = None
    with pytest.raises(ValueError, match="autoscaling"):
        vis.set_data(np.zeros((2, 17, 3)), 0)
    with pytest.raises(ValueError, match="autoscaling"):
        S.camera_matrices(None)
    with pytest.raises(ValueError):
        S.camera_matrices((1, 1))
    vis = S.Skeleton3DVisualizer(S.H36M_PARENTS, plot_3d_limit=[-6, 6], show_joint=True)
    with pytest.raises(NotImplementedError):
        vis.set_data(np.zeros((2, 17, 3)), 0)
    vis = S.Skeleton3DVisualizer(S.H36M_PARENTS, plot_3d_limit=[-6, 6])
    for view in (-1, 4, 7):
        with pytest.raises(ValueError, match="camera_view"):
            vis.set_data(np.zeros((2, 17, 3)), view)
    for views in ([0, 4], np.array([-1, 0])):
        with pytest.raises(ValueError, match="views"):
            S._views(views, 2, "cpu")
    with pytest.raises(ValueError, match="views"):
        S._views(torch.tensor([0, 5]), 2, "cpu")
    with pytest.raises(ValueError, match="CUDA"):
        S.render_poses(torch.zeros(2, 17, 3), [0, 1])
    # the reference's constructor signature and attributes
    v = S.Skeleton3DVisualizer([-1, 0, 1])
    assert v.plot_3d_limit == [0.0, 1.0] and v.show_joint is False and v.show_ticks is False and v.render is False
    assert v.camera_azimuth == [70, 70, 110, 110] and v.parents == [-1, 0, 1]


@pytest.fixture
def fake_reference(tmp_path, monkeypatch):
    d = tmp_path / "data" / "human36m"
    d.mkdir(parents=True)
    (d / "skeleton.py").write_text("class Skeleton:\n    pass\n")
    (d / "human36m.py").write_text(textwrap.dedent("""\
        from skeleton import Skeleton
        STD_SCALE = 3
        class Human36mDataset:
            skeleton_class = Skeleton
        def fig2img(fig):
            return 'fake fig2img'
        class Skeleton3DVisualizer:
            pass
        """))
    monkeypatch.setenv("P2PVG_REF", str(tmp_path))
    monkeypatch.syspath_prepend(os.path.join(ROOT, "dropin"))
    for m in ("human36m", "skeleton"):
        monkeypatch.delitem(sys.modules, m, raising=False)
    path = list(sys.path)
    yield d
    for m in ("human36m", "skeleton"):
        sys.modules.pop(m, None)
    sys.path[:] = path


def test_dropin_human36m(fake_reference):
    h36m = importlib.import_module("human36m")
    assert h36m.__file__ == os.path.join(ROOT, "dropin", "human36m.py")
    assert h36m.Skeleton3DVisualizer is S.Skeleton3DVisualizer and h36m.STD_SCALE == 3
    assert h36m.Human36mDataset.__module__ == "_reference_human36m"
    assert h36m.Human36mDataset.skeleton_class.__name__ == "Skeleton" and h36m.fig2img(None) == "fake fig2img"
    with pytest.raises(AttributeError):
        h36m.__wrapped__


def test_dropin_human36m_through_sys_path(fake_reference, monkeypatch):
    monkeypatch.setenv("P2PVG_REF", "")
    monkeypatch.syspath_prepend(str(fake_reference.parent.parent))   # the reference's root, as train.py runs from it
    monkeypatch.syspath_prepend(os.path.join(ROOT, "dropin"))
    h36m = importlib.import_module("human36m")
    assert h36m.Skeleton3DVisualizer is S.Skeleton3DVisualizer
    assert h36m.Human36mDataset.skeleton_class.__name__ == "Skeleton"
