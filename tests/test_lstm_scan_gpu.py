"""LSTM scan kernels (p2pvg_lstm_scan_fwd / _bwd) against the step-by-step formulation.

The first tests run the recurrence free against float64 with loose tolerances, and check that a row's result does not depend on
the slab it lands in.  The tests after them check every kernel instance step by step against teacher-forced float64 references
with per-element bounds (tests/lstm_schedule.py), each on the schedule it states: the benchmark's launch shapes, every slab size
with a partial last slab, launches of several waves of resident clusters, and saturated gates.  Every case starts from a
nonzero h0 / c0, and its outputs start as NaN with a NaN tail: every in-range element must be written, and nothing past the end.
"""
import pytest
import torch

from tests.lstm_schedule import check_backward, check_forward, max_clusters, report, scan_schedule

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def K():
    from p2pvg_b200._lib import CudaKernels
    return CudaKernels("cuda")


@pytest.mark.parametrize("tf32", [False, True])
@pytest.mark.parametrize("S,B,R", [(5, 3, 64), (7, 70, 256), (30, 256, 256), (4, 100, 128), (6, 40, 512), (9, 256, 512), (1, 17, 512),
                                   (5, 128, 512), (7, 250, 512), (3, 300, 512)])
def test_scan_fwd_bwd(K, S, B, R, tf32):
    if R == 512 and not tf32 and B > 128:
        pytest.skip("exact-fp32 R=512 uses the per-step kernels at this batch (the cooperative grid does not fit)")
    tol = 3e-3 if tf32 else 1e-4
    torch.manual_seed(0)
    dev = "cuda"
    pre = torch.randn(S, B, 4 * R, device=dev) * 0.5
    whh = torch.randn(4 * R, R, device=dev) * (1.0 / R ** 0.5)
    bhh = torch.randn(4 * R, device=dev) * 0.1
    gates = torch.empty(S, B, 4 * R, device=dev)
    hs = torch.zeros(S + 1, B, R, device=dev)
    cs = torch.zeros(S + 1, B, R, device=dev)
    ctr = torch.zeros(4, dtype=torch.int32, device=dev)
    K.lstm_scan_fwd(pre, whh, bhh, gates, hs, cs, S, B, R, ctr, tf32=tf32)
    # reference recurrence
    h = torch.zeros(B, R, device=dev, dtype=torch.float64)
    c = torch.zeros_like(h)
    for s in range(S):
        z = pre[s].double() + bhh.double() + h @ whh.double().t()
        i, f, g, o = torch.sigmoid(z[:, :R]), torch.sigmoid(z[:, R:2 * R]), torch.tanh(z[:, 2 * R:3 * R]), torch.sigmoid(z[:, 3 * R:])
        c = f * c + i * g
        h = o * torch.tanh(c)
        assert torch.allclose(gates[s].double(), torch.cat([i, f, g, o], 1), rtol=tol, atol=tol), f"gates step {s}"
        assert torch.allclose(hs[s + 1].double(), h, rtol=tol, atol=tol), f"h step {s}"
        assert torch.allclose(cs[s + 1].double(), c, rtol=tol, atol=tol), f"c step {s}"
    # backward against autograd through the same recurrence
    pre_a = pre.double().requires_grad_(True)
    h = torch.zeros(B, R, device=dev, dtype=torch.float64)
    c = torch.zeros_like(h)
    outs = []
    for s in range(S):
        z = pre_a[s] + bhh.double() + h @ whh.double().t()
        i, f, g, o = torch.sigmoid(z[:, :R]), torch.sigmoid(z[:, R:2 * R]), torch.tanh(z[:, 2 * R:3 * R]), torch.sigmoid(z[:, 3 * R:])
        c = f * c + i * g
        h = o * torch.tanh(c)
        outs.append(h)
    dhtop = torch.randn(S, B, R, device=dev)
    (torch.stack(outs) * dhtop.double()).sum().backward()
    dG = torch.empty(S, B, 4 * R, device=dev)
    ctr.zero_()
    K.lstm_scan_bwd(dhtop, whh, gates, cs, dG, S, B, R, ctr, tf32=tf32)
    ref = pre_a.grad
    err = (dG.double() - ref).abs().max().item()
    assert err <= tol * ref.abs().max().item() + tol * 0.1, err


def test_scan512_slab_size_invariance(K):
    """The R=512 forward scan picks 16-, 32- or 48-row slabs per cluster from the batch size (one wave of resident clusters);
    a batch row's result must not depend on that choice: rows 0..39 of a 256-row launch (48-row slabs, partial sums aliased
    onto the consumed h slab) are bit-identical to the same rows launched alone (16-row slabs), and so are rows of a 128-row
    launch (32-row slabs)."""
    S, R = 6, 512
    torch.manual_seed(3)
    dev = "cuda"
    pre = torch.randn(S, 256, 4 * R, device=dev) * 0.5
    whh = torch.randn(4 * R, R, device=dev) * (1.0 / R ** 0.5)
    bhh = torch.randn(4 * R, device=dev) * 0.1
    c0 = torch.randn(256, R, device=dev) * 0.3
    h0 = torch.randn(256, R, device=dev) * 0.3

    def run(rows):
        B = len(rows)
        p = pre[:, rows].contiguous()
        gates = torch.empty(S, B, 4 * R, device=dev)
        hs = torch.zeros(S + 1, B, R, device=dev)
        cs = torch.zeros(S + 1, B, R, device=dev)
        hs[0], cs[0] = h0[rows], c0[rows]
        ctr = torch.zeros(4, dtype=torch.int32, device=dev)
        K.lstm_scan_fwd(p, whh, bhh, gates, hs, cs, S, B, R, ctr, tf32=True)
        return gates, hs, cs

    full = run(list(range(256)))
    for rows in (list(range(40)), list(range(100, 228)), list(range(216, 256))):
        part = run(rows)
        for a, b, nm in zip(full, part, ("gates", "h", "c")):
            assert torch.equal(a[:, rows], b), f"{nm}: rows {rows[0]}..{rows[-1]} depend on the slab size"


def test_scan512_backward_slab_size_invariance(K):
    """The R=512 backward scan runs in 16-row slabs, with the 16 partial products of every row summed in rank order, so the
    gradients of rows taken from a 256-row launch and from a 128-row launch must be bit-identical to those rows launched alone:
    a row's result must not depend on which slab or cluster it lands in."""
    S, R = 5, 512
    torch.manual_seed(4)
    dev = "cuda"
    Bf = 256
    whh = torch.randn(4 * R, R, device=dev) * (1.0 / R ** 0.5)
    gates = torch.rand(S, Bf, 4 * R, device=dev) * 0.8 + 0.1
    gates[:, :, 2 * R:3 * R] = gates[:, :, 2 * R:3 * R] * 2 - 1          # the g gate is a tanh
    cs = torch.randn(S + 1, Bf, R, device=dev) * 0.5
    dh = torch.randn(S, Bf, R, device=dev)

    def run(rows):
        B = len(rows)
        dG = torch.empty(S, B, 4 * R, device=dev)
        ctr = torch.zeros(4, dtype=torch.int32, device=dev)
        K.lstm_scan_bwd(dh[:, rows].contiguous(), whh, gates[:, rows].contiguous(), cs[:, rows].contiguous(), dG, S, B, R, ctr, tf32=True)
        return dG

    full = run(list(range(Bf)))                       # 6 clusters of 48 rows
    for rows in (list(range(40)), list(range(200, 256)), list(range(64, 192))):   # 16-row slabs, 16-row slabs, 32-row slabs
        part = run(rows)
        assert torch.equal(full[:, rows], part), f"rows {rows[0]}..{rows[-1]} depend on the slab size"


# ------------------------------------------------------------------ per-step float64 bounds on stated schedules

TAIL = 4096                                               # NaN canary elements after every output
BENCH = {"C2": (29, 256, 256), "C3": (29, 128, 256), "C4": (29, 64, 256), "C5": (59, 256, 512)}   # (S = T - 1, B, R)


@pytest.fixture(scope="module")
def maxc(K):
    return {R: max_clusters(K.lib, R) for R in (64, 128, 192, 256, 512)}


def _nan_out(shape):
    n = 1
    for d in shape:
        n *= d
    buf = torch.full((n + TAIL,), float("nan"), device="cuda")
    return buf, buf[:n].view(*shape)


def _canary(buf, shape, name):
    n = buf.numel() - TAIL
    assert torch.isnan(buf[n:]).all(), f"{name}: {int((~torch.isnan(buf[n:])).sum())} elements written past the end"
    bad = ~torch.isfinite(buf[:n].view(*shape))
    assert not bad.any(), f"{name}: {int(bad.sum())} in-range elements not written or not finite, first at {bad.nonzero()[0].tolist()}"


def run_checked(K, maxc, S, B, R, tf32, seed=0, pre_scale=0.5, fbias=0.0):
    """Forward then backward (on the forward's own gates / cs) from a nonzero initial state, canaries and teacher-forced checks.
    Returns the forward and backward schedules and the outputs."""
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(seed)
    pre = torch.randn(S, B, 4 * R, device=dev, generator=g) * pre_scale
    whh = torch.randn(4 * R, R, device=dev, generator=g) / R ** 0.5
    bhh = torch.randn(4 * R, device=dev, generator=g) * 0.1
    bhh[R:2 * R] += fbias
    gb, gates = _nan_out((S, B, 4 * R))
    hb, hs = _nan_out((S + 1, B, R))
    cb, cs = _nan_out((S + 1, B, R))
    hs[0] = torch.randn(B, R, device=dev, generator=g) * 0.5
    cs[0] = torch.randn(B, R, device=dev, generator=g) * 0.5
    ctr = torch.zeros(4, dtype=torch.int32, device=dev)
    K.lstm_scan_fwd(pre, whh, bhh, gates, hs, cs, S, B, R, ctr, tf32=tf32)
    for buf, t, nm in ((gb, gates, "gates"), (hb, hs, "hs"), (cb, cs, "cs")):
        _canary(buf, t.shape, nm)
    sf = scan_schedule(R, B, tf32, maxc[R])
    worst = check_forward(sf, pre, whh, bhh, gates, hs, cs)
    report(worst, sf)
    dhtop = torch.randn(S, B, R, device=dev, generator=g)
    db, dG = _nan_out((S, B, 4 * R))
    ctr.zero_()
    K.lstm_scan_bwd(dhtop, whh, gates, cs, dG, S, B, R, ctr, tf32=tf32)
    _canary(db, dG.shape, "dG")
    sb = scan_schedule(R, B, tf32, maxc[R], bwd=True)
    report(check_backward(sb, dhtop, whh, gates, cs, dG), sb)
    return sf, sb, dict(gates=gates, hs=hs, cs=cs, dG=dG)


def search_B(start, want, R, maxc, limit=4096):
    """First batch size from `start` whose forward and backward schedules satisfy want(fwd, bwd): the shape follows the
    device's resident-cluster counts instead of skipping on another device."""
    for B in range(start, limit):
        sf, sb = scan_schedule(R, B, True, maxc[R]), scan_schedule(R, B, True, maxc[R], bwd=True)
        if want(sf, sb):
            return B
    pytest.fail(f"no batch size in [{start}, {limit}) gives the schedule this case is written for (R={R}, {maxc[R]})")


def partial_slab(s):
    return 0 < s.last_rows < s.rows


def partial_wave(s):
    """More clusters than are resident, and a last wave that is not full."""
    return s.maxc is not None and s.maxc > 0 and s.slabs > s.maxc and s.slabs % s.maxc != 0


@pytest.mark.parametrize("cfg", sorted(BENCH))
def test_bench_shapes_bf16(K, maxc, cfg):
    """The launches of the bf16 engine at the benchmark configurations (skip_prob 0: S = T - 1)."""
    S, B, R = BENCH[cfg]
    sf, sb, _ = run_checked(K, maxc, S, B, R, True, seed=1)
    if R == 512:
        assert sf.family == sb.family == "cluster16" and sb.MT == 1
    else:
        assert sf.family == sb.family == "cluster8" and sf.MT == sb.MT == (2 if B > 128 else 1)


@pytest.mark.parametrize("cfg", ["C2", "C3", "C4"])
def test_bench_shapes_fp32(K, maxc, cfg):
    """The same R = 256 launches in the fp32 engine: the cooperative exact-fp32 scans."""
    S, B, R = BENCH[cfg]
    sf, sb, _ = run_checked(K, maxc, S, B, R, False, seed=2)
    assert sf.family == sb.family == "coop-exact" and sf.last_rows == 64


@pytest.mark.parametrize("R", [64, 128, 256])
@pytest.mark.parametrize("MT,B", [(1, 100), (2, 150)])
def test_cluster8_instances(K, maxc, R, MT, B):
    """Every cluster-8 instance, forward and backward, with a partial last slab (100 = 6 x 16 + 4, 150 = 4 x 32 + 22)."""
    sf, sb, _ = run_checked(K, maxc, 9, B, R, True, seed=R + MT)
    for s in (sf, sb):
        assert s.family == "cluster8" and s.MT == MT and partial_slab(s), s.describe()


R512_FWD = {   # case -> (search start, schedule the case is written for)
    "MT1": (40, lambda f, b: f.MT == 1 and partial_slab(f)),
    "MT2": (150, lambda f, b: f.MT == 2 and partial_slab(f)),
    "MT3 last 1-16": (250, lambda f, b: f.MT == 3 and f.waves == 1 and 1 <= f.last_rows <= 16),
    "MT3 last 17-32": (250, lambda f, b: f.MT == 3 and f.waves == 1 and 17 <= f.last_rows <= 32),
    "MT3 last 33-47": (250, lambda f, b: f.MT == 3 and f.waves == 1 and 33 <= f.last_rows <= 47),
    "MT3 waves": (400, lambda f, b: f.MT == 3 and partial_wave(f) and partial_slab(f)),
    "bwd waves": (100, lambda f, b: partial_wave(b) and partial_slab(b)),
}


@pytest.mark.parametrize("case", list(R512_FWD))
def test_cluster16_instances(K, maxc, case):
    """R = 512: the forward at 16-, 32- and 48-row slabs (the 48-row slab aliases its partial sums onto consumed h rows; its
    last slab is tried with 1-16, 17-32 and 33-47 valid rows), several waves of 48-row slabs, and the 16-row backward over
    several waves.  Every case also checks the backward at its batch size."""
    start, want = R512_FWD[case]
    B = search_B(start, want, 512, maxc)
    sf, sb, _ = run_checked(K, maxc, 5, B, 512, True, seed=B)
    assert sf.family == sb.family == "cluster16" and want(sf, sb), (sf.describe(), sb.describe())


def test_cluster8_several_waves(K, maxc):
    """R = 256 with 32-row slabs on more clusters than are resident, forward and backward, last wave and slab partial."""
    B = search_B(129, lambda f, b: all(partial_wave(s) and partial_slab(s) and s.MT == 2 for s in (f, b)), 256, maxc)
    sf, sb, _ = run_checked(K, maxc, 5, B, 256, True, seed=7)
    assert partial_wave(sf) and partial_wave(sb) and sf.waves > 1, (sf.describe(), sb.describe())


@pytest.mark.parametrize("R,tf32", [(192, True), (192, False), (64, False)])
def test_cooperative_instances(K, maxc, R, tf32):
    """The cooperative scans: TF32 at R = 192 (the bf16 engine's fused scan for a hidden size that is no cluster size) and exact
    fp32; 100 rows = one full 64-row block and one of 36."""
    sf, sb, _ = run_checked(K, maxc, 9, 100, R, tf32, seed=R)
    for s in (sf, sb):
        assert s.family == ("coop-tf32" if tf32 else "coop-exact") and s.last_rows == 36, s.describe()


@pytest.mark.parametrize("R,tf32", [(256, True), (512, True), (256, False)])
def test_saturation(K, maxc, R, tf32):
    """S = 59 with pre-activations x6 and a +3 forget bias: |c| grows, sigmoid and tanh saturate, nothing is non-finite (the
    canaries check that) and every step stays within its bound."""
    _, _, out = run_checked(K, maxc, 59, 40, R, tf32, seed=11, pre_scale=3.0, fbias=3.0)
    cmax = out["cs"].abs().max().item()
    f = out["gates"][:, :, R:2 * R]
    assert cmax > 4.0, f"max |c| = {cmax}: the case does not drive c out of tanh's linear range"
    assert (f > 0.999).float().mean().item() > 0.05, "forget gates do not saturate"


@pytest.mark.parametrize("R", [64, 128, 256])
def test_cluster8_slab_size_invariance(K, maxc, R):
    """Rows of a 200-row launch (32-row slabs) are bit-identical to the same rows launched alone at <= 128 rows (16-row slabs),
    forward and backward: both instances run the same per-row m16 chain and the same partial-sum order."""
    S, Bf = 6, 200
    torch.manual_seed(5)
    dev = "cuda"
    pre = torch.randn(S, Bf, 4 * R, device=dev) * 0.5
    whh = torch.randn(4 * R, R, device=dev) * (1.0 / R ** 0.5)
    bhh = torch.randn(4 * R, device=dev) * 0.1
    h0 = torch.randn(Bf, R, device=dev) * 0.5
    c0 = torch.randn(Bf, R, device=dev) * 0.5
    dh = torch.randn(S, Bf, R, device=dev)

    def run(rows, gates_in=None, cs_in=None):
        B = len(rows)
        assert scan_schedule(R, B, True, maxc[R]).MT == (2 if B > 128 else 1)
        ctr = torch.zeros(4, dtype=torch.int32, device=dev)
        gates = torch.empty(S, B, 4 * R, device=dev)
        hs = torch.zeros(S + 1, B, R, device=dev)
        cs = torch.zeros(S + 1, B, R, device=dev)
        hs[0], cs[0] = h0[rows], c0[rows]
        K.lstm_scan_fwd(pre[:, rows].contiguous(), whh, bhh, gates, hs, cs, S, B, R, ctr, tf32=True)
        dG = torch.empty(S, B, 4 * R, device=dev)
        ctr.zero_()
        g_in = gates if gates_in is None else gates_in[:, rows].contiguous()
        c_in = cs if cs_in is None else cs_in[:, rows].contiguous()
        K.lstm_scan_bwd(dh[:, rows].contiguous(), whh, g_in, c_in, dG, S, B, R, ctr, tf32=True)
        return gates, hs, cs, dG

    full = run(list(range(Bf)))
    for rows in (list(range(40)), list(range(72, 200))):
        part = run(rows, full[0], full[2])
        for a, b, nm in zip(full, part, ("gates", "h", "c", "dG")):
            assert torch.equal(a[:, rows], b), f"{nm}: rows {rows[0]}..{rows[-1]} depend on the slab size"
