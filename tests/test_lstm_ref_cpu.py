"""The LSTM scan checker (tests/lstm_schedule.py) on the CPU: a torch emulation of the TF32 cluster scan passes it, and each of a
set of small, deliberate corruptions of that emulation is rejected, so the bounds are sharp enough to catch them.  Also the
host-side schedule mirror and the benchmark's scan lengths."""
import numpy as np
import pytest
import torch

from tests.lstm_schedule import (check_backward, check_forward, fwd_slab_tiles, scan_schedule, tf32_rna)

S, B, R = 6, 21, 64          # one full 16-row slab and a partial one of 5 rows (cluster8, MT = 1)


def emulate_fwd(pre, whh, bhh, h0, c0, corrupt=None):
    """The cluster kernels' forward in torch: tf32_rna operands, the product accumulated exactly and rounded to fp32 (within
    the tensor cores' bound), fp32 pointwise.  Outputs start as NaN, as in the GPU canary tests."""
    W = tf32_rna(whh).double()
    if corrupt == "k8 block":
        W[:, 8:16] = 0
    b = bhh.clone()
    if corrupt == "b_hh gate":
        b[R:2 * R] = 0
    gates = torch.full((S, B, 4 * R), float("nan"))
    hs = torch.full((S + 1, B, R), float("nan"))
    cs = torch.full((S + 1, B, R), float("nan"))
    hs[0], cs[0] = h0, c0
    c = torch.zeros(B, R) if corrupt == "c0 ignored" else c0.clone()
    rows = 16 if corrupt == "partial slab unwritten" else B
    for s in range(S):
        hin = hs[s].clone()
        if corrupt == "h from slot s-1" and s == 3:
            hin[16:] = hs[s - 1][16:]
        acc = (tf32_rna(hin).double() @ W.t()).float()
        z = acc + (pre[s] + b)
        i, f, g, o = torch.sigmoid(z[:, :R]), torch.sigmoid(z[:, R:2 * R]), torch.tanh(z[:, 2 * R:3 * R]), torch.sigmoid(z[:, 3 * R:])
        c = f * c + i * g
        h = o * torch.tanh(c)
        gates[s, :rows] = torch.cat([i, f, g, o], 1)[:rows]
        cs[s + 1, :rows], hs[s + 1, :rows] = c[:rows], h[:rows]
    return gates, hs, cs


def emulate_bwd(dhtop, whh, gates, cs, corrupt=None):
    W = tf32_rna(whh).double()
    dG = torch.full((S, B, 4 * R), float("nan"))
    dc_reg = torch.zeros(B, R)
    for s in range(S - 1, -1, -1):
        dh = dhtop[s] if s == S - 1 else dhtop[s] + (tf32_rna(dG[s + 1]).double() @ W).float()
        i, f, g, o = gates[s].split(R, -1)
        tc = torch.tanh(cs[s + 1])
        dc = dh * o * (1 - tc * tc) + dc_reg
        dc_reg = dc if (corrupt == "f missing from dc" and s == 2) else dc * f
        dG[s] = torch.cat([dc * g * i * (1 - i), dc * cs[s] * f * (1 - f), dc * i * (1 - g * g), dh * tc * o * (1 - o)], 1)
    return dG


@pytest.fixture(scope="module")
def data():
    gen = torch.Generator().manual_seed(0)
    pre = torch.randn(S, B, 4 * R, generator=gen) * 0.5
    whh = torch.randn(4 * R, R, generator=gen) / R ** 0.5
    bhh = torch.randn(4 * R, generator=gen) * 0.1
    h0 = torch.randn(B, R, generator=gen) * 0.5
    c0 = torch.randn(B, R, generator=gen) * 0.5
    dhtop = torch.randn(S, B, R, generator=gen)
    return pre, whh, bhh, h0, c0, dhtop


def sched(bwd=False):
    s = scan_schedule(R, B, True, None, bwd=bwd)
    assert (s.family, s.MT, s.rows, s.slabs, s.last_rows) == ("cluster8", 1, 16, 2, 5), s.describe()
    return s


def test_emulation_passes(data):
    pre, whh, bhh, h0, c0, dhtop = data
    gates, hs, cs = emulate_fwd(pre, whh, bhh, h0, c0)
    worst = check_forward(sched(), pre, whh, bhh, gates, hs, cs)
    dG = emulate_bwd(dhtop, whh, gates, cs)
    check_backward(sched(True), dhtop, whh, gates, cs, dG, worst)
    print(worst)
    assert set(worst) == {"gates", "c", "h", "dG"}


@pytest.mark.parametrize("corrupt", ["b_hh gate", "k8 block", "h from slot s-1", "c0 ignored", "partial slab unwritten"])
def test_forward_corruption_rejected(data, corrupt):
    pre, whh, bhh, h0, c0, _ = data
    gates, hs, cs = emulate_fwd(pre, whh, bhh, h0, c0, corrupt)
    with pytest.raises(AssertionError) as ei:
        check_forward(sched(), pre, whh, bhh, gates, hs, cs)
    print(corrupt, "->", str(ei.value)[:200])


@pytest.mark.parametrize("corrupt", ["f missing from dc", "partial slab unwritten"])
def test_backward_corruption_rejected(data, corrupt):
    pre, whh, bhh, h0, c0, dhtop = data
    gates, hs, cs = emulate_fwd(pre, whh, bhh, h0, c0)
    dG = emulate_bwd(dhtop, whh, gates, cs, "f missing from dc" if corrupt == "f missing from dc" else None)
    if corrupt == "partial slab unwritten":
        dG[:, 16:] = float("nan")
    with pytest.raises(AssertionError) as ei:
        check_backward(sched(True), dhtop, whh, gates, cs, dG)
    print(corrupt, "->", str(ei.value)[:200])


def test_tf32_rna():
    """Round to nearest on the 10 kept mantissa bits, ties away from zero, sign-symmetric."""
    one = 1.0
    x = torch.tensor([one + 2 ** -11, one + 2 ** -11 - 2 ** -23, one + 3 * 2 ** -11, 1.5 + 2 ** -12, 3.0, 0.0])
    want = torch.tensor([one + 2 ** -10, one, one + 4 * 2 ** -11, 1.5, 3.0, 0.0])
    assert torch.equal(tf32_rna(x), want)
    assert torch.equal(tf32_rna(-x), -want)
    y = torch.randn(4096) * 100
    r = tf32_rna(y)
    assert torch.equal(r.view(torch.int32) & 0x1FFF, torch.zeros(4096, dtype=torch.int32))
    assert ((r - y).abs() <= y.abs() * 2.0 ** -11).all()


def test_schedule_mirror():
    """Slab sizes and the R = 512 cost model, for stated resident-cluster counts."""
    assert scan_schedule(256, 128, True, None).MT == 1 and scan_schedule(256, 129, True, None).MT == 2
    s = scan_schedule(256, 600, True, {1: 16})
    assert (s.family, s.MT, s.slabs, s.waves, s.last_rows) == ("cluster8", 2, 19, 2, 24)
    s = scan_schedule(192, 100, True, None, bwd=True)
    assert (s.family, s.cs, s.slabs, s.last_rows, s.waves) == ("coop-tf32", 24, 2, 36, 1)
    assert scan_schedule(256, 100, False, None).family == "coop-exact"
    # cost waves * (1.5 + 2.8 MT) with 8 resident clusters: 1 wave of 16-row slabs up to 128 rows, then 32-row slabs (one
    # wave beats two), 48-row slabs between 257 and 384 rows, 32-row slabs again at 385..512 (2 waves of 7.1 < 2 of 9.9)
    assert [fwd_slab_tiles(b, 8) for b in (128, 129, 256, 257, 384, 385, 512)] == [1, 2, 2, 3, 3, 2, 2]
    assert fwd_slab_tiles(300, 0) == fwd_slab_tiles(300, 7)
    s = scan_schedule(512, 300, True, {0: 8, 1: 8, 3: 8, 2: 8})
    assert (s.family, s.MT, s.rows, s.slabs, s.last_rows) == ("cluster16", 3, 48, 7, 12)
    assert scan_schedule(512, 300, True, {1: 8}, bwd=True).rows == 16


@pytest.mark.parametrize("T,S", [(30, 29), (60, 59)])
def test_benchmark_scan_lengths(T, S):
    """The scan lengths the GPU tests use for the benchmark configurations (C2-C4: T = 30, C5: T = 60) at skip_prob 0."""
    from p2pvg_b200.engine import StepPlan
    probs = np.random.RandomState(0).uniform(0, 1, T - 1)
    assert StepPlan(T, probs, dict(skip_prob=0.0, n_past=1, last_frame_skip=False)).S == S
