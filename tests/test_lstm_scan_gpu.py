"""Persistent cooperative LSTM scan kernels (p2pvg_lstm_scan_fwd / _bwd) against the step-by-step formulation."""
import pytest
import torch

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
