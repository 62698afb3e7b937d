"""BatchNorm backward (bn.cu) the way the training step calls it, against float64.

TrainEngine.bn_backward calls bn_bwd with y = None (the LeakyReLU slope is recomputed from sign(fmaf(x, scale, shift))), with
scale / shift passed and dx aliasing dy.  Shapes (G groups, R rows, C channels) are the step's: C in {64, 128, 256, 512}, R = B*Ho*Ho
from 16 to 262144, plus ragged row counts (the last row pair of a chunk has one row) and the widest channel counts the kernels
accept (one and two row lanes per block).  Also: bit-identity of the call forms, the forward tile finalizer, tanh with y given,
and the one-pass forward statistics on data whose mean is three standard deviations from zero.
"""
import pytest
import torch

from tests.tc_schedule import assert_within

pytestmark = pytest.mark.gpu

ACT_LRELU, ACT_TANH = 1, 2
EPS = 1e-5
# fp32 per-thread running sums over at most ~1000 rows each (choose_chunks caps a block at 64 chunks), then float64: every add is
# off by at most 2^-24 of the magnitude summed so far, so 2^-14 of the summed magnitude covers the sums and what is built on them
ALPHA = 2.0 ** -14

STEP_SHAPES = [(3, 16, 512), (2, 1, 64), (2, 129, 256), (2, 4097, 128), (4, 1024, 256), (2, 16384, 128), (3, 4096, 512),
               (1, 262144, 64)]


def shapes_for(dt):
    vec = 8 if dt == torch.bfloat16 else 4
    # C = 256 * vec: one row lane per block; C = 128 * vec: two
    return [(dt, *s) for s in STEP_SHAPES + [(2, 300, 256 * vec), (2, 301, 128 * vec)]]


PARAMS = shapes_for(torch.bfloat16) + shapes_for(torch.float32)


@pytest.fixture(scope="module")
def K():
    from p2pvg_b200._lib import CudaKernels
    return CudaKernels("cuda")


def zeros(*n):
    return torch.zeros(*n, device="cuda")


def fwd_stats(K, raw, G, R, C, gamma, beta):
    st = [zeros(G * C) for _ in range(5)]
    K.bn_fwd_stats(raw, G, R, C, gamma, beta, *st)
    return dict(zip(("mean", "invstd", "var", "scale", "shift"), st))


def bn_ref64(raw, gamma, beta, dz_fn, G, R, C):
    """float64 autograd of batch_norm(raw) (training mode, per group, statistics recomputed in float64) followed by the
    activation whose input gradient is dz_fn(pre).  Returns dx, sum dz, sum dz*xhat, dgamma, dbeta and xhat / dz for bounds."""
    x = raw.double().view(G, R, C).clone().requires_grad_()
    g = gamma.double().clone().requires_grad_()
    b = beta.double().clone().requires_grad_()
    m = x.mean(1, keepdim=True)
    v = ((x - m) ** 2).mean(1, keepdim=True)
    xhat = (x - m) / torch.sqrt(v + EPS)
    pre = xhat * g + b
    dz = dz_fn(pre.detach())
    pre.backward(dz)
    xh = xhat.detach()
    return dict(dx=x.grad, sdz=dz.sum(1), sdzx=(dz * xh).sum(1), dgamma=g.grad, dbeta=b.grad, xhat=xh, dz=dz,
                invstd=(1.0 / torch.sqrt(v + EPS)).squeeze(1))


def check_bwd(res, ref, gamma, dt, name):
    """dx, the two sums and the parameter gradients of one bn_bwd call against bn_ref64."""
    dz, xh = ref["dz"], ref["xhat"]
    R = dz.shape[1]
    w = []
    w.append(assert_within(res["sdz"].view_as(ref["sdz"]), ref["sdz"], dz.abs().sum(1), 0, torch.float32, alpha=ALPHA, name=f"{name} sum_dz"))
    w.append(assert_within(res["sdzx"].view_as(ref["sdzx"]), ref["sdzx"], (dz * xh).abs().sum(1), 0, torch.float32, alpha=ALPHA,
                           name=f"{name} sum_dzx"))
    # dx = gamma * invstd * (dz - mean(dz) - xhat * mean(dz * xhat)): bounded by the magnitudes of its three terms
    k0 = (gamma.double() * ref["invstd"]).abs().unsqueeze(1)
    mag = k0 * (dz.abs() + (dz.abs().sum(1, keepdim=True) + xh.abs() * (dz * xh).abs().sum(1, keepdim=True)) / R)
    w.append(assert_within(res["dx"].view_as(ref["dx"]), ref["dx"], mag, 0, dt, alpha=ALPHA, name=f"{name} dx"))
    w.append(assert_within(res["dgamma"], ref["dgamma"], (dz * xh).abs().sum((0, 1)), 0, torch.float32, alpha=ALPHA, name=f"{name} dgamma"))
    w.append(assert_within(res["dbeta"], ref["dbeta"], dz.abs().sum((0, 1)), 0, torch.float32, alpha=ALPHA, name=f"{name} dbeta"))
    return max(w)


@pytest.mark.parametrize("dt,G,R,C", PARAMS)
def test_bn_bwd_against_float64_in_every_call_form(K, dt, G, R, C):
    torch.manual_seed(R + C)
    raw = (torch.randn(G, R, C, device="cuda") * 1.5 + 0.3).to(dt)
    gamma, beta = torch.rand(C, device="cuda") + 0.5, torch.randn(C, device="cuda") * 0.5
    st = fwd_stats(K, raw, G, R, C, gamma, beta)
    # dy correlated with xhat: sum(dz * xhat) is then O(R) and the xhat term of dx carries weight
    r64 = raw.double()
    xh = (r64 - r64.mean(1, keepdim=True)) / torch.sqrt(r64.var(1, unbiased=False, keepdim=True) + EPS)
    dy = (0.5 * xh + torch.randn(G, R, C, device="cuda", dtype=torch.float64)).to(dt)
    # the kernel takes the slope side from sign(fmaf(x, scale, shift)) in fp32; x*scale is exact in float64, so this is that sign.
    # It is the float64 sign of the pre-activation except within rounding of zero: a tie decision, not an error.
    side = (r64 * st["scale"].double().view(G, 1, C) + st["shift"].double().view(G, 1, C)) > 0

    def dz_fn(pre):
        flips = (side != (pre > 0)).sum().item()
        assert flips <= max(4, pre.numel() // 100000), f"{flips} slope sides differ from the float64 pre-activation's sign"
        return dy.double() * torch.where(side, 1.0, 0.2)
    ref = bn_ref64(raw, gamma, beta, dz_fn, G, R, C)
    args = (st["mean"], st["invstd"], gamma, G, R, C, ACT_LRELU)

    def run(y, inplace, **ss):
        d = dy.clone()
        dx = d if inplace else torch.empty_like(d)
        sdz, sdzx = zeros(G * C), zeros(G * C)
        K.bn_bwd(d, raw, y, *args, dx, sdz, sdzx, **ss)
        if not inplace:
            assert torch.equal(d, dy), "out-of-place bn_bwd wrote dy"
        dg, db = zeros(C), zeros(C)
        K.bn_param_grad(sdz, sdzx, G, C, dg, db)
        return dict(dx=dx, sdz=sdz, sdzx=sdzx, dgamma=dg, dbeta=db)
    step = run(None, True, scale=st["scale"], shift=st["shift"])          # TrainEngine.bn_backward
    check_bwd(step, ref, gamma, dt, f"bn_bwd {dt} G={G} R={R} C={C}")
    # the other call forms: bit for bit the same (the y-given slope is the sign of the same fmaf, stored by bn_act)
    y = torch.empty_like(raw)
    K.bn_act(raw, y, st["scale"], st["shift"], G, R, C, ACT_LRELU)
    for form, res in (("y=None out of place", run(None, False, scale=st["scale"], shift=st["shift"])),
                      ("y given in place", run(y, True)), ("y given out of place", run(y, False))):
        for k in ("dx", "sdz", "sdzx"):
            assert torch.equal(res[k], step[k]), f"{form}: {k} differs from the in-place y=None form"


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("G,R", [(30, 256), (30, 16)])
def test_bn_bwd_tanh_encoder_output(K, dt, G, R):
    """The encoders' last layer: BatchNorm + tanh over C = g channels, R = B rows per timestep, with y given (in place, as the
    step calls it).  The kernel's derivative is 1 - y^2 of the STORED y, so the reference takes dz from the stored y too."""
    C = 128
    torch.manual_seed(G + R)
    raw = (torch.randn(G, R, C, device="cuda") * 2 + 0.5).to(dt)
    gamma, beta = torch.rand(C, device="cuda") + 0.5, torch.randn(C, device="cuda") * 0.5
    st = fwd_stats(K, raw, G, R, C, gamma, beta)
    y = torch.empty_like(raw)
    K.bn_act(raw, y, st["scale"], st["shift"], G, R, C, ACT_TANH)
    dy = torch.randn(G, R, C, device="cuda").to(dt)
    ref = bn_ref64(raw, gamma, beta, lambda pre: dy.double() * (1 - y.double() ** 2), G, R, C)
    d = dy.clone()
    sdz, sdzx = zeros(G * C), zeros(G * C)
    K.bn_bwd(d, raw, y, st["mean"], st["invstd"], gamma, G, R, C, ACT_TANH, d, sdz, sdzx)
    dg, db = zeros(C), zeros(C)
    K.bn_param_grad(sdz, sdzx, G, C, dg, db)
    check_bwd(dict(dx=d, sdz=sdz, sdzx=sdzx, dgamma=dg, dbeta=db), ref, gamma, dt, f"bn_bwd tanh {dt} G={G} R={R}")


@pytest.mark.parametrize("C,fold,ppg", [(96, 3, 13), (200, 2, 5), (64, 4, 21)])
def test_fwd_finalize_tiles(K, C, fold, ppg):
    """bn_fwd_finalize_tiles: float64 sums over a group's partial rows and the `fold` column groups of each row
    (parts_per_group not a multiple of the kernel's 8 part lanes, row pitch wider than fold * C)."""
    G, rows = 3, 16
    ldp = fold * C + 8
    torch.manual_seed(C + fold)
    # forward partials from real data, so that every variance is positive: (sum x, sum x^2) over `rows` values per entry
    x = torch.randn(G * ppg, rows, fold * C, device="cuda") * 1.3 + 0.7
    part = torch.zeros(G * ppg, ldp, 2, device="cuda")
    part[:, :fold * C, 0] = x.sum(1)
    part[:, :fold * C, 1] = (x * x).sum(1)
    part[:, fold * C:] = float("nan")     # padding past fold * C is never read
    p64 = part[:, :fold * C].double().view(G, ppg, fold, C, 2)
    a, b = p64[..., 0].sum((1, 2)), p64[..., 1].sum((1, 2))
    gamma, beta = torch.rand(C, device="cuda") + 0.5, torch.randn(C, device="cuda")
    out = [zeros(G * C) for _ in range(5)]
    count = ppg * rows * fold
    K.bn_fwd_finalize_tiles(part, ppg, ldp, fold, G, count, C, gamma, beta, *out)
    m = a / count
    var = b / count - m * m
    inv = 1.0 / torch.sqrt(var + EPS)
    # scale = gamma * float(invstd) and shift = beta - float(mean) * scale are fp32 products / differences of rounded values
    sc = gamma.double() * inv
    want = [(m, m.abs()), (inv, inv), (var * count / (count - 1), var), (sc, sc.abs()),
            (beta.double() - m * sc, beta.double().abs() + (m * sc).abs())]
    for got, (r, mag), nm in zip(out, want, ("mean", "invstd", "var_unbiased", "scale", "shift")):
        assert_within(got.view(G, C), r, mag, 0, torch.float32, alpha=2.0 ** -21, name=f"bn_fwd_finalize_tiles C={C} {nm}")


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("G,R,C", [(2, 4097, 128), (1, 262144, 64), (3, 1024, 512)])
def test_fwd_stats_offset_mean(K, dt, G, R, C):
    """bn_fwd_stats accumulates sum x and sum x^2 per thread in fp32 and forms E[x^2] - m^2 in float64.  With the mean three
    standard deviations from zero, E[x^2] = 10 var: the cancellation costs about three bits, well within what the step tolerates."""
    torch.manual_seed(G * R + C)
    sig = torch.rand(C, device="cuda") + 0.5
    x = (3 * sig + sig * torch.randn(G, R, C, device="cuda")).to(dt)
    gamma, beta = torch.rand(C, device="cuda") + 0.5, torch.randn(C, device="cuda")
    st = fwd_stats(K, x, G, R, C, gamma, beta)
    x64 = x.double()
    m = x64.mean(1)
    ex2 = (x64 * x64).mean(1)
    var = (x64 - m.unsqueeze(1)).pow(2).mean(1)
    name = f"bn_fwd_stats 3-sigma {dt} G={G} R={R} C={C}"
    assert_within(st["mean"].view(G, C), m, x64.abs().mean(1), 0, torch.float32, alpha=ALPHA, name=f"{name} mean")
    # var = E[x^2] - m^2: the error of E[x^2] plus twice that of m, both relative to E[x^2]
    assert_within(st["var"].view(G, C), var * R / max(R - 1, 1), 3 * ex2 * R / max(R - 1, 1), 0, torch.float32, alpha=ALPHA,
                  name=f"{name} var_unbiased")
    inv = 1.0 / torch.sqrt(var + EPS)
    # d invstd / invstd = -1/2 d var / var
    assert_within(st["invstd"].view(G, C), inv, inv * 1.5 * ex2 / (var + EPS), 0, torch.float32, alpha=ALPHA, name=f"{name} invstd")
