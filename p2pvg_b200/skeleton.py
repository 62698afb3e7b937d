"""Human3.6M skeletons drawn on the GPU as the reference's ``Skeleton3DVisualizer`` (data/human36m/human36m.py:290-388) draws
them with matplotlib: ``render_poses`` renders any number of poses in one ``p2pvg_skeleton_render`` launch, and
``Skeleton3DVisualizer`` stands in for the reference's class (same constructor, ``set_data`` returns the same uint8 arrays).

What is drawn (the kernel and the float64 NumPy oracle tests/skeleton_ref.py both implement this; it restates mplot3d's
``Axes3D.get_proj``, ``proj3d.view_transformation`` and ``persp_transformation`` of the matplotlib 3.0 era.  Parity with
matplotlib's raster is neither claimed nor tested):

  figure     2 x 2 in at 64 dpi (128 x 128 px), the axes fill it; each image is the 98 x 98 crop [15:113, 15:113], RGB on
             white.
  data       pose joint p[j] = (x, y, z) is plotted at (X, Y, Z) = (x, z, y) (human36m.py:357-359).
  limits     plot_3d_limit = [lo, hi] gives xlim3d = (hi, lo), ylim3d = (lo, hi), zlim3d = (hi, lo) (X and Z reversed); the
             world matrix W maps each axis by (v - a) / (b - a) for its limit pair (a, b).
  camera     elev 15 deg, azim (70, 70, 110, 110)[camera_view], dist 10, R = (.5, .5, .5),
             E = R + dist (cos az cos el, sin az cos el, sin el), V = (0, 0, 1); n = (E - R) / |E - R|, u = V x n / |V x n|,
             v = n x u; View = [u; v; n] . translate(-E).
  perspective P = [[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, a, b], [0, 0, -1, 0]] with zfront, zback = -10, 10 (a = 0, b = -10);
             M = P . View . W; (x2, y2) = (m0 / m3, m1 / m3) for m = M (X, Y, Z, 1).  M is computed per view in float64
             (``camera_matrices``) and handed to the kernel in fp32.
  pixels     the 2-D view window is [-0.095, 0.09] on both axes: display dx = (x2 + .095) / .185 * 128, dy likewise, y up;
             column c covers dx in [c, c + 1), row r covers dy in [127 - r, 128 - r).  The pose origin lands at cropped
             (row, col) = (47.27, 50.73) in every view, (0, -3, 0) at (30.45, 50.73) (head up), and the whole [-6, 6]^3 box
             inside the crop.
  limbs      limb l = 0 .. J-2 joins joint l + 1 to parents[l + 1], drawn in that order, later limbs over earlier ones;
             colour (1, 0, 0) for l in {0, 1, 2, 13, 14, 15}, (0, 0, 1) for l in {3, 4, 5, 10, 11, 12}, (0, .5, 0) otherwise
             (human36m.py:321-330).  H36M_PARENTS is the 17-joint Human3.6M skeleton the loader builds.
  stroke     3 pt wide (half-width h = 1.5 * 64 / 72 px) with projecting caps: the projected segment becomes a rectangle
             extended by h past both ends.  Coverage of a pixel is k / 64, k the number of the 8 x 8 sample points
             (c + (i + .5) / 8, 127 - r + (j + .5) / 8) inside the rectangle.  A limb shorter than 1e-6 px (the zero poses of
             skipped frames) or with a non-finite projected end draws nothing.
  blend      per channel in fp32, c <- c + (colour - c) k / 64; q = min(255, floor(255 c + 0.5)).  uint8 output: q as
             [N, 98, 98, 3] (what the reference's ``fig2img`` returns); fp32 output: float32(q / 255.) as [N, 3, 98, 98] (the
             reference's pictures as vis_seq scales them).

Not covered: axes decorations (panes, grid, axis lines, ticks); ``plot_3d_limit=None``, the reference's per-call
autoscaling (ValueError); ``show_joint=True`` (NotImplementedError, as the reference's ``set_data`` raises); views outside
0..3 (ValueError, on the host).
"""
from __future__ import annotations

import numpy as np
import torch

H36M_PARENTS = (-1, 0, 1, 2, 0, 4, 5, 0, 7, 8, 9, 8, 11, 12, 8, 14, 15)
AZIMUTHS = (70, 70, 110, 110)
ELEV = 15.0
SIZE = 98            # the cropped image: 128 - 2 * 15
MAX_JOINTS = 32
RED, BLUE, GREEN = (1.0, 0.0, 0.0), (0.0, 0.0, 1.0), (0.0, 0.5, 0.0)


def limb_colors(n_limbs):
    """[n_limbs, 3] float64: the reference's colour of each limb (human36m.py:321-330)."""
    return np.array([RED if l in (0, 1, 2, 13, 14, 15) else BLUE if l in (3, 4, 5, 10, 11, 12) else GREEN
                     for l in range(n_limbs)], np.float64).reshape(n_limbs, 3)


def _limit(limit):
    if limit is None:
        raise ValueError("plot_3d_limit=None (the reference's per-call autoscaling) is not supported: pass [lo, hi]")
    lo, hi = (float(v) for v in limit)
    if not (np.isfinite(lo) and np.isfinite(hi) and lo != hi):
        raise ValueError(f"plot_3d_limit must be two finite, different numbers (got {limit!r})")
    return lo, hi


def camera_matrices(limit, azimuths=AZIMUTHS, elev=ELEV):
    """[len(azimuths), 4, 4] float64: M = P . View . W of each view for plot_3d_limit = limit (module docstring)."""
    lo, hi = _limit(limit)
    W = np.eye(4)
    for k, (a, b) in enumerate(((hi, lo), (lo, hi), (hi, lo))):
        W[k, k], W[k, 3] = 1.0 / (b - a), -a / (b - a)
    dist, R, V = 10.0, np.array([0.5, 0.5, 0.5]), np.array([0.0, 0.0, 1.0])
    P = np.array([[1.0, 0, 0, 0], [0, 1, 0, 0], [0, 0, 0, -10.0], [0, 0, -1, 0]])
    el = np.deg2rad(float(elev))
    out = []
    for az in azimuths:
        az = np.deg2rad(float(az))
        E = R + dist * np.array([np.cos(az) * np.cos(el), np.sin(az) * np.cos(el), np.sin(el)])
        n = (E - R) / np.linalg.norm(E - R)
        u = np.cross(V, n)
        u = u / np.linalg.norm(u)
        v = np.cross(n, u)
        view = np.eye(4)
        view[:3, :3] = np.stack([u, v, n])
        view[:3, 3] = -view[:3, :3] @ E
        out.append(P @ view @ W)
    return np.stack(out)


def kernel_matrices(limit):
    """fp32 [4, 3, 4]: rows 0, 1 and 3 of each view's M, as p2pvg_skeleton_render takes them."""
    return np.ascontiguousarray(camera_matrices(limit)[:, [0, 1, 3]].astype(np.float32))


def check_parents(parents):
    """The parents as an int32 array; ValueError unless parents[0] = -1, 0 <= parents[j] < j and 2 <= J <= 32."""
    p = np.asarray(parents).astype(np.int64).reshape(-1)
    J = len(p)
    if not 2 <= J <= MAX_JOINTS:
        raise ValueError(f"the skeleton has {J} joints; the renderer draws 2..{MAX_JOINTS}")
    if p[0] != -1 or any(not 0 <= p[j] < j for j in range(1, J)):
        raise ValueError(f"parents must start with -1 and have 0 <= parents[j] < j (got {p.tolist()})")
    return p.astype(np.int32)


def _views(views, n, dev):
    """int32 [n] views on dev; ValueError for a view outside 0..3."""
    if torch.is_tensor(views):
        v = views.reshape(-1)
        if v.numel() == 1 and n != 1:
            v = v.expand(n)
        if v.numel() != n:
            raise ValueError(f"{v.numel()} views for {n} poses")
        v = v.to(device=dev, dtype=torch.int32).contiguous()
        if n and bool(((v < 0) | (v > 3)).any()):
            raise ValueError("camera views must be 0..3")
        return v
    a = np.asarray(views).reshape(-1).astype(np.int64)
    if a.size == 1 and n != 1:
        a = np.full(n, a[0])
    if a.size != n:
        raise ValueError(f"{a.size} views for {n} poses")
    if n and (a.min() < 0 or a.max() > 3):
        raise ValueError(f"camera views must be 0..3 (got {sorted(set(a.tolist()))})")
    return torch.from_numpy(a.astype(np.int32)).to(dev)


def render_poses(poses, views, parents=H36M_PARENTS, limit=(-6, 6), out="float"):
    """Skeleton pictures of CUDA poses [N, J, 3] (any float dtype; drawn from their fp32 values) in one launch:
    out="float" -> fp32 [N, 3, 98, 98], out="uint8" -> uint8 [N, 98, 98, 3], out="both" -> (fp32, uint8).  views: one camera
    view 0..3 per pose (a CUDA / host tensor, a sequence or one int for all).  ValueError before any launch for a bad
    shape, view, parents or limit."""
    from ._lib import kernels_for
    if out not in ("float", "uint8", "both"):
        raise ValueError(f"out must be 'float', 'uint8' or 'both' (got {out!r})")
    if not torch.is_tensor(poses) or poses.device.type != "cuda" or poses.dim() != 3 or poses.shape[2] != 3:
        raise ValueError("render_poses takes CUDA poses [N, J, 3]")
    par = check_parents(parents)
    N, J = int(poses.shape[0]), int(poses.shape[1])
    if J != len(par):
        raise ValueError(f"poses have {J} joints but the skeleton has {len(par)}")
    mats = kernel_matrices(limit)
    dev = poses.device
    v = _views(views, N, dev)
    p = poses.to(torch.float32).contiguous()
    f = torch.empty(N, 3, SIZE, SIZE, device=dev) if out != "uint8" else None
    u = torch.empty(N, SIZE, SIZE, 3, device=dev, dtype=torch.uint8) if out != "float" else None
    colors = np.ascontiguousarray(limb_colors(J - 1).astype(np.float32))
    kernels_for(dev).skeleton_render(p, v, par, colors, mats, f, u)
    return f if out == "float" else u if out == "uint8" else (f, u)


class Skeleton3DVisualizer:
    """The reference's Skeleton3DVisualizer (same constructor) drawn by p2pvg_skeleton_render on the current CUDA device.
    ``show_ticks`` and ``render`` are accepted and have no effect: no axes are drawn and no window is shown."""

    def __init__(self, parents, plot_3d_limit=[0.0, 1.0], show_joint=False, show_ticks=False, render=False):
        self.parents = parents
        self.plot_3d_limit = plot_3d_limit
        self.camera_azimuth = list(AZIMUTHS)
        self.show_joint = show_joint
        self.show_ticks = show_ticks
        self.render = render
        self._parents = check_parents(parents)
        _limit(plot_3d_limit)

    def _check(self):
        if self.show_joint:
            raise NotImplementedError("show_joint is not drawn (the reference's set_data raises NotImplementedError too)")
        _limit(self.plot_3d_limit)

    def render_device(self, poses, views):
        """fp32 [N, 3, 98, 98] pictures of CUDA poses [N, J, 3] with one camera view each, in one launch (vis_seq's path)."""
        self._check()
        return render_poses(poses, views, self._parents, self.plot_3d_limit, out="float")

    def set_data(self, pose_3d, camera_view):
        """uint8 [T, 98, 98, 3] NumPy pictures of the host poses pose_3d [T, J, 3] seen from camera_view, as the reference's
        set_data returns them; drawn in one launch on the current CUDA device."""
        self._check()
        if camera_view not in range(4):
            raise ValueError(f"camera_view must be 0..3 (got {camera_view!r})")
        p = torch.as_tensor(np.asarray(pose_3d, dtype=np.float32))
        if p.dim() != 3 or p.shape[2] != 3:
            raise ValueError(f"set_data takes poses [T, J, 3] (got {tuple(p.shape)})")
        dev = torch.device("cuda", torch.cuda.current_device())
        return render_poses(p.to(dev), int(camera_view), self._parents, self.plot_3d_limit, out="uint8").cpu().numpy()
