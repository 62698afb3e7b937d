"""Float64 NumPy oracle of the skeleton pictures (the spec in p2pvg_b200/skeleton.py's module docstring), restated here
without p2pvg_b200: the camera matrices, the projection of every joint, each limb's rectangle and the 8 x 8 sample count of
every pixel, the fp32 blend and the quantisation.

The projection and the edge functions are written out one float64 operation at a time in the order the kernel evaluates
them (it rounds every operation the same way and contracts none), from the fp32 matrices the kernel is handed, so the
sample counts are the kernel's exactly; the blend and the quantisation are NumPy float32, as the spec states them.
``project_rc`` is the same projection in continuous cropped (row, col) coordinates, for the anchors."""
import numpy as np

PARENTS = [-1, 0, 1, 2, 0, 4, 5, 0, 7, 8, 9, 8, 11, 12, 8, 14, 15]
FIG, CROP, OUT = 128, 15, 98
HALF = 1.5 * 64 / 72
AZIM = (70, 70, 110, 110)


def world(limit):
    lo, hi = limit
    W = np.eye(4)
    for k, (a, b) in enumerate(((hi, lo), (lo, hi), (hi, lo))):   # xlim3d = (hi, lo), ylim3d = (lo, hi), zlim3d = (hi, lo)
        W[k, k] = 1.0 / (b - a)
        W[k, 3] = -a / (b - a)
    return W


def camera(limit, azim, elev=15.0, dist=10.0):
    """mplot3d's get_proj: P . View . W, float64 [4, 4]."""
    el, az = np.pi * elev / 180, np.pi * azim / 180
    R = np.array([0.5, 0.5, 0.5])
    E = R + dist * np.array([np.cos(az) * np.cos(el), np.sin(az) * np.cos(el), np.sin(el)])
    V = np.array([0.0, 0.0, 1.0])
    n = (E - R) / np.sqrt(((E - R) ** 2).sum())
    u = np.cross(V, n)
    u = u / np.sqrt((u ** 2).sum())
    v = np.cross(n, u)
    Mr = np.eye(4)
    Mr[0, :3], Mr[1, :3], Mr[2, :3] = u, v, n
    Mt = np.eye(4)
    Mt[:3, 3] = -E
    zf, zb = -dist, dist
    a, b = (zf + zb) / (zf - zb), -2 * (zf * zb) / (zf - zb)
    P = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, a, b], [0, 0, -1, 0]], np.float64)
    return P @ (Mr @ Mt) @ world(limit)


def matrices(limit):
    return np.stack([camera(limit, az) for az in AZIM])


def project_rc(M, p):
    """Continuous cropped (row, col) of pose point p = (x, y, z) under the float64 M."""
    m = M @ np.array([p[0], p[2], p[1], 1.0])
    dx = (m[0] / m[3] + 0.095) / 0.185 * 128
    dy = (m[1] / m[3] + 0.095) / 0.185 * 128
    return FIG - dy - CROP, dx - CROP


def colors(n_limbs):
    return np.array([(1, 0, 0) if l in (0, 1, 2, 13, 14, 15) else (0, 0, 1) if l in (3, 4, 5, 10, 11, 12) else (0, 0.5, 0)
                     for l in range(n_limbs)], np.float32).reshape(n_limbs, 3)


def levels():
    """float32(q / 255.) for q = 0..255: the fp32 picture of quantised value q."""
    return (np.arange(256, dtype=np.float64) / 255.).astype(np.float32)


def display(pose, rows32):
    """Display (dx, dy) float64 [J] of pose [J, 3] under the fp32 rows 0, 1, 3 of M, in the kernel's operation order."""
    p = np.asarray(pose, np.float32).astype(np.float64)
    X, Y, Z = p[:, 0], p[:, 2], p[:, 1]
    R = rows32.astype(np.float64)
    m = [((R[r, 0] * X + R[r, 1] * Y) + R[r, 2] * Z) + R[r, 3] for r in range(3)]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        x2, y2 = m[0] / m[2], m[1] / m[2]
        return (x2 + 0.095) / 0.185 * 128.0, (y2 + 0.095) / 0.185 * 128.0


def coverage(p0, p1):
    """(k [98, 98] int sample counts, or None when the limb draws nothing) of the limb from display point p0 to p1."""
    with np.errstate(over="ignore", invalid="ignore"):
        dx, dy = p1[0] - p0[0], p1[1] - p0[1]
        length = np.sqrt(dx * dx + dy * dy)
    if not (np.isfinite(p0).all() and np.isfinite(p1).all() and np.isfinite(length) and length >= 1e-6):
        return None
    ux, uy = dx / length, dy / length
    lenh = length + HALF
    k = np.zeros((OUT, OUT), np.int64)
    # bounding box (any box holding the rectangle gives the same counts; the caps reach sqrt(2) h past an end)
    pad = 2 * HALF
    xlo, xhi = min(p0[0], p1[0]) - pad, max(p0[0], p1[0]) + pad
    ylo, yhi = min(p0[1], p1[1]) - pad, max(p0[1], p1[1]) + pad
    c0, c1 = max(0, int(np.floor(max(xlo, -4096))) - CROP), min(OUT - 1, int(np.floor(min(xhi, 4096))) - CROP)
    r0, r1 = max(0, FIG - 1 - int(np.floor(min(yhi, 4096))) - CROP), min(OUT - 1, FIG - 1 - int(np.floor(max(ylo, -4096))) - CROP)
    if c0 > c1 or r0 > r1:
        return k
    off = (np.arange(8) + 0.5) / 8
    qx = (np.arange(c0, c1 + 1) + CROP)[:, None] + off[None, :]                  # [nc, 8 (i)]
    qy = (FIG - 1 - (np.arange(r0, r1 + 1) + CROP))[:, None] + off[None, :]     # [nr, 8 (j)]
    ex, ey = qx - p0[0], qy - p0[1]
    along = (ux * ex)[None, :, None, :] + (uy * ey)[:, None, :, None]          # [nr, nc, j, i]
    across = (ux * ey)[:, None, :, None] - (uy * ex)[None, :, None, :]
    inside = (along >= -HALF) & (along <= lenh) & (np.abs(across) <= HALF)
    k[r0:r1 + 1, c0:c1 + 1] = inside.sum((2, 3))
    return k


def render(poses, views, parents=PARENTS, limit=(-6, 6), rows=None):
    """(uint8 [N, 98, 98, 3], fp32 [N, 3, 98, 98]) pictures of poses [N, J, 3] with views [N].  rows: the fp32 [4, 3, 4]
    rows 0, 1, 3 of each view's M the kernel was handed (default: this module's M rounded to fp32; the two float64
    restatements agree to 1e-15, but an entry may round to a neighbouring fp32 value)."""
    poses = np.asarray(poses, np.float32)
    N, J = poses.shape[:2]
    rows = matrices(limit)[:, [0, 1, 3]].astype(np.float32) if rows is None else np.asarray(rows, np.float32)
    col = colors(J - 1)
    u8 = np.empty((N, OUT, OUT, 3), np.uint8)
    for n in range(N):
        X, Y = display(poses[n], rows[int(views[n])])
        c = np.ones((OUT, OUT, 3), np.float32)
        for l in range(J - 1):
            a, b = l + 1, parents[l + 1]
            k = coverage(np.array([X[a], Y[a]]), np.array([X[b], Y[b]]))
            if k is None:
                continue
            w = (k.astype(np.float32) * np.float32(1 / 64))[..., None]
            c = c + (col[l] - c) * w
        u8[n] = np.minimum(255, np.floor(np.float32(255) * c + np.float32(0.5))).astype(np.uint8)
    return u8, levels()[u8].transpose(0, 3, 1, 2).copy()
