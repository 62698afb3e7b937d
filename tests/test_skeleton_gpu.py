"""p2pvg_skeleton_render on the GPU against the float64 NumPy oracle (tests/skeleton_ref.py), the drop-in
Skeleton3DVisualizer, and vis_seq's device pose path against the host path drawn by the oracle."""
import sys
import types

import numpy as np
import pytest
import torch

from p2pvg_b200 import skeleton as S
from p2pvg_b200 import visualize as V
from p2pvg_b200._lib import CudaKernels, KernelError, kernels_for
from tests import skeleton_ref as R
from tests.test_generate_engine_gpu import precision
from tests.test_vis_gpu import bench_input, bench_model, fixture_model, inject_eps
from tests.vis_ref import Recorder, case_input

pytestmark = pytest.mark.gpu
ROWS = S.kernel_matrices((-6, 6))
STEP = 1 / 255 + 1e-6


def render_both(poses, views):
    f, u = S.render_poses(torch.as_tensor(np.asarray(poses, np.float32)).cuda(), torch.as_tensor(np.asarray(views)).cuda(),
                          out="both")
    torch.cuda.synchronize()
    return f.cpu().numpy(), u.cpu().numpy()


def hand_made():
    """(poses [n, 17, 3], views): limbs partly and fully outside the crop, overlapping limbs of different colours, zeros."""
    rs = np.random.RandomState(7)
    out = []
    p = 3 * rs.randn(17, 3)
    p[1] = (40, 0, 0)                    # limbs 0 and 1 reach far outside the crop
    p[2:4] = (60, 0, 60), (80, 10, 70)   # limbs 1, 2 wholly outside
    out.append(p)
    p = np.zeros((17, 3))
    p[1] = p[4] = (3, 0, 0)              # limb 0 (red) and limb 3 (blue) on the same segment: blue drawn over red
    p[7] = (0, -3, 0)
    p[8] = (0, -4, 1)                    # limb 6 (green) and limb 10 (blue, joint 11 -> 8) crossing
    p[11] = (2, -4, -2)
    out.append(p)
    out.append(np.zeros((17, 3)))        # a skipped frame: nothing drawn
    out.append(20 * rs.randn(17, 3))     # mostly outside
    p = 3 * rs.randn(17, 3)
    p[5] = (0, 0, 1e4)                   # a joint far behind the scene
    out.append(p)
    return np.stack(out)


def compare(got_u8, got_f, want_u8):
    d = np.abs(got_u8.astype(np.int32) - want_u8.astype(np.int32))
    assert d.max() <= 1 and (d == 0).mean() >= 0.999, (d.max(), (d == 0).mean())
    assert np.array_equal(got_f, R.levels()[got_u8].transpose(0, 3, 1, 2))


def test_kernel_matches_the_oracle_on_loader_scale_poses():
    rs = np.random.RandomState(0)
    poses = (3 * rs.randn(256, 17, 3)).astype(np.float32)   # N(0, 3^2) per coordinate, the loader's scale
    views = np.arange(256) % 4
    f, u = render_both(poses, views)
    want, _ = R.render(poses, views, rows=ROWS)
    compare(u, f, want)
    assert len(np.unique(u)) == 256          # every quantised level appears, and its fp32 value is float32(q / 255.)
    assert (u < 255).mean() > 0.05


def test_kernel_matches_the_oracle_on_hand_made_cases():
    poses = hand_made()
    for view in range(4):
        views = np.full(len(poses), view)
        f, u = render_both(poses, views)
        want, _ = R.render(poses, views, rows=ROWS)
        compare(u, f, want)
        assert (u[2] == 255).all()
        # the overlap: along the shared segment the last limb drawn (blue) covers the red one completely
        X, Y = R.display(poses[1], ROWS[view])
        mid = (X[1] + X[0]) / 2, (Y[1] + Y[0]) / 2
        r, c = R.FIG - 1 - int(np.floor(mid[1])) - R.CROP, int(np.floor(mid[0])) - R.CROP
        assert tuple(u[1, r, c]) == (0, 0, 255)
        assert tuple(want[1, r, c]) == (0, 0, 255)


def test_uint8_is_the_rounded_fp32():
    rs = np.random.RandomState(1)
    f, u = render_both(3 * rs.randn(64, 17, 3), rs.randint(0, 4, 64))
    assert np.array_equal(np.round(f.astype(np.float64) * 255).astype(np.uint8).transpose(0, 2, 3, 1), u)


def test_batched_equals_single_launches_and_runs_repeat():
    rs = np.random.RandomState(2)
    poses = torch.from_numpy((3 * rs.randn(48, 17, 3)).astype(np.float32)).cuda()
    views = torch.from_numpy(rs.randint(0, 4, 48)).cuda()
    a = S.render_poses(poses, views)
    b = S.render_poses(poses, views)
    one = torch.cat([S.render_poses(poses[i:i + 1], views[i:i + 1]) for i in range(48)])
    torch.cuda.synchronize()
    assert torch.equal(a, b) and torch.equal(a, one)


def test_set_data_returns_the_references_arrays():
    rs = np.random.RandomState(3)
    vis = S.Skeleton3DVisualizer(S.H36M_PARENTS, plot_3d_limit=[-6, 6])
    pose = 3 * rs.randn(7, 17, 3)
    for view in range(4):
        img = vis.set_data(pose, view)
        assert isinstance(img, np.ndarray) and img.dtype == np.uint8 and img.shape == (7, 98, 98, 3)
        want, _ = R.render(pose, [view] * 7, rows=ROWS)
        d = np.abs(img.astype(np.int32) - want)
        assert d.max() <= 1 and (d == 0).mean() >= 0.999
    assert np.array_equal(vis.set_data(pose, 2), S.render_poses(torch.from_numpy(pose).float().cuda(), 2, out="uint8")
                          .cpu().numpy())


def test_library_rejects_malformed_arguments():
    K = kernels_for(torch.device("cuda"))
    col, mats = S.limb_colors(16).astype(np.float32), S.kernel_matrices((-6, 6))
    poses, views = torch.zeros(2, 17, 3, device="cuda"), torch.zeros(2, dtype=torch.int32, device="cuda")
    f = torch.empty(2, 3, 98, 98, device="cuda")
    par = np.array(S.H36M_PARENTS, np.int32)
    K.skeleton_render(poses, views, par, col, mats, f, None)
    for bad in ([0] + list(par[1:]), [-1, 0, 2] + list(par[3:]), [-1, 0, -1] + list(par[3:])):
        with pytest.raises(KernelError, match="parents"):
            K.skeleton_render(poses, views, np.array(bad, np.int32), col, mats, f, None)
    p33 = torch.zeros(2, 33, 3, device="cuda")
    with pytest.raises(KernelError, match="J = 33"):
        K.skeleton_render(p33, views, np.array([-1] + list(range(32)), np.int32), np.zeros((32, 3), np.float32), mats, None,
                          torch.empty(2, 98, 98, 3, device="cuda", dtype=torch.uint8))
    with pytest.raises(KernelError, match="colour"):
        K.skeleton_render(poses, views, par, col * 2, mats, f, None)
    with pytest.raises(KernelError, match="outputs"):
        K.skeleton_render(poses, views, par, col, mats, None, None)


# vis_seq ------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def rec(monkeypatch):
    r = Recorder()
    monkeypatch.setitem(sys.modules, "imageio", r.imageio)
    tv = types.ModuleType("torchvision")
    tv.utils = r.vutils
    monkeypatch.setitem(sys.modules, "torchvision", tv)
    monkeypatch.setitem(sys.modules, "torchvision.utils", r.vutils)
    return r


class OracleVis:
    """The host path's visualizer: set_data draws with the oracle (any object but Skeleton3DVisualizer takes that path)."""

    def __init__(self):
        self.calls = 0

    def set_data(self, pose_3d, camera_view):
        self.calls += 1
        return R.render(pose_3d, [camera_view] * len(pose_3d), rows=ROWS)[0]


class CountingVis(S.Skeleton3DVisualizer):
    def set_data(self, pose_3d, camera_view):
        raise AssertionError("the device path must not call set_data")


def run_both(monkeypatch, run):
    """run(vis) on the host path (OracleVis) and on the device path (CountingVis), each from the same seeds: returns
    [(outputs, numpy state, cuda rng state)] and the device path's render launches."""
    launches = []
    orig = CudaKernels.skeleton_render

    def counted(self, *a, **k):
        launches.append(1)
        return orig(self, *a, **k)
    monkeypatch.setattr(CudaKernels, "skeleton_render", counted)
    res = []
    for vis in (OracleVis(), CountingVis(S.H36M_PARENTS, plot_3d_limit=[-6, 6])):
        if isinstance(vis, CountingVis):
            monkeypatch.setattr(V, "_render", lambda *a: pytest.fail("poses went to the host"))
            launches.clear()
        out = run(vis)
        torch.cuda.synchronize()
        res.append((out, np.random.get_state(), torch.cuda.get_rng_state()))
    return res, len(launches)


def check_same(res, rec):
    (a, sa, ca), (b, sb, cb) = res
    assert sa[0] == sb[0] and np.array_equal(sa[1], sb[1]) and sa[2:] == sb[2:]
    assert torch.equal(ca, cb)
    for x, y in zip(a[:2], b[:2]):
        assert x.shape == y.shape and (x - y).abs().max().item() <= STEP
    assert a[2].shape == b[2].shape and (a[2].int() - b[2].int()).abs().max().item() <= 1
    assert rec.saved[0][0] == rec.saved[1][0] and rec.gifs[0][0] == rec.gifs[1][0]
    assert [i[0] for i in rec.images[:1]] == [i[0] for i in rec.images[1:]] and rec.images[0][2] == rec.images[1][2]
    assert (rec.videos[0][0], rec.videos[0][2], rec.videos[0][3]) == (rec.videos[1][0], rec.videos[1][2], rec.videos[1][3])


@pytest.mark.parametrize("T,L,skip_frame", [(10, 12, False), (10, 8, True)])
def test_vis_seq_device_path_matches_the_host_path(rec, monkeypatch, T, L, skip_frame):
    model, C = bench_model("pose", 10, 20)
    x = bench_input("pose", T, 10, C)

    def run(vis):
        np.random.seed(11)
        torch.cuda.manual_seed(12)
        return V.vis_seq(model, x, 3, L, model_mode="full", recon_mode="test", skip_frame=skip_frame, h36m_visualizer=vis,
                         writer=rec, opt=model.opt)
    res, launches = run_both(monkeypatch, run)
    assert launches == 1
    check_same(res, rec)
    assert res[1][0][0].shape[1] == 5 * 6 * 98                  # 5 row blocks of 6 rows of 98-pixel pictures


def test_vis_seq_device_path_on_the_fixture_case(rec, monkeypatch):
    import os
    fix = torch.load(os.path.join(os.path.dirname(__file__), "golden", "vis_seq.pt"), weights_only=False)
    c = next(c for c in fix["cases"] if c["case"] == "h36m")
    sp = c["spec"]
    with precision("fp32"):
        model = fixture_model(c)
        x = tuple(t.cuda() for t in case_input(sp))

        def run(vis):
            pos = inject_eps(monkeypatch, c["eps"])
            np.random.seed(c["np_seed"])
            out = V.vis_seq(model, x, 7, sp["L"], model_mode=sp["mode"], recon_mode=sp["recon"], skip_frame=sp["skip"],
                            h36m_visualizer=vis, writer=rec, opt=model.opt)
            assert pos[0] == c["n_calls"]
            return out
        res, launches = run_both(monkeypatch, run)
    assert launches == 1
    check_same(res, rec)
    assert (rec.saved[1][0], rec.gifs[1][0]) == c["names"] and (rec.images[1][0], rec.videos[1][0]) == c["tags"]
    st, ref = res[1][1], c["np_state_after"]
    assert st[0] == ref[0] and np.array_equal(st[1], ref[1]) and st[2:] == ref[2:]
