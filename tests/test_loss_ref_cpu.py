"""The loss / optimiser checker (tests/loss_ref.py) on the CPU: the torch emulation of the kernel ABI (tests/emu_backend.py,
tests/emu_mlp.py) passes it, and each of a list of small, deliberate corruptions is rejected, so the bounds are sharp enough
to catch them.  Also the launch-shape mirror against bench.CONFIGS and the host-side launch decisions."""
import math

import pytest
import torch

from tests import loss_ref as L
from tests.emu_mlp import EmuKernelsMLP

G, E, T, B = 3, 3 * 8192 + 100, 5, 4


@pytest.fixture(scope="module")
def emu():
    return EmuKernelsMLP("cpu")


def rng(seed):
    return torch.Generator().manual_seed(seed)


def loss_data(seed=0):
    g = rng(seed)
    raw = torch.randn(G * E, generator=g) * 2
    x = torch.rand(T * E, generator=g)
    tgt = torch.tensor([1, 2, 4], dtype=torch.int32)
    coef = torch.tensor([1.0, 1.0, 100.0])
    return raw, x, tgt, coef


def chunked_partials(sq):
    """The kernel's partial layout: [G, 32], each chunk the double sum of its elements, stored as fp32."""
    return torch.stack([L.chunk_sums(s) for s in sq]).float()


def sigmoid_mse_like(raw, x, tgt, coef, corrupt=None):
    r = raw.reshape(G, E)
    s = torch.sigmoid(r)
    d = s - x.reshape(T, E)[tgt.long()]
    q = d * s if corrupt == "sigmoid derivative without (1 - s)" else d * s * (1 - s)
    part = chunked_partials([(dd.double() ** 2) for dd in d])
    if corrupt == "one MSE chunk dropped":
        part[1, 5] = 0
    return (coef.reshape(G, 1) * 2 * q).reshape(-1), part.reshape(-1)


def reparam_data(n, seed=1):
    g = rng(seed)
    return [torch.randn(n, generator=g) * s for s in (1.0, 0.5, 1.0, 0.5, 1.0, 1.0)]


def align_like(H, in_idx, hp, P, Bb, g, coef, dh, dH, corrupt=None):
    Hv = H.reshape(-1, Bb, g)
    h = hp.reshape(-1, Bb, g)[:P]
    row = torch.arange(Bb) if corrupt == "align row 0 replaced by row b" else torch.zeros(Bb, dtype=torch.long)
    h0 = Hv[in_idx[:P].long()][:, row]
    diff = h0 - h
    lp = (diff.double() ** 2).mean((1, 2)).float()
    dh = dh.clone()
    dh.reshape(-1, Bb, g)[:P] += -coef * 2 * diff / (Bb * g)
    dH = dH.clone()
    dH.reshape(-1, Bb, g)[in_idx[:P].long(), 0] += coef * 2 * diff.sum(1) / (Bb * g)
    return lp, dh, dH


def adam_like(p, g, m, v, n, lr, b1, b2, eps, t, corrupt=None):
    m2 = m * b1 + (1 - b1) * g
    v2 = v * b2 + (1 - b2) * g * g
    ss = lr if corrupt == "Adam without bias correction" else L.adam_step_size(lr, b1, b2, t)
    return p - ss * (m2 / (v2.sqrt() + eps)), m2, v2


# ------------------------------------------------------------------ the emulation passes

def test_emulation_passes(emu):
    worst = {}
    raw, x, tgt, coef = loss_data()
    pred, d_raw, part = torch.empty(G * E), torch.empty(G * E), torch.empty(G * 32)
    emu.sigmoid_mse(raw, x, tgt, coef, G, E, pred, d_raw, part)
    L.check_sigmoid_mse(raw, x, tgt, coef, G, E, pred, d_raw, part, per_chunk=False, worst=worst)   # the emulation sums into chunk 0
    d_pred, part2 = torch.empty(G * E), torch.empty(G * 32)
    emu.mse_plain(raw, x, tgt, coef, G, E, d_pred, part2)
    L.check_mse_plain(raw, x, tgt, coef, G, E, d_pred, part2, per_chunk=False, worst=worst)

    # the fused last layer: col2im + sigmoid_mse of the emulation against the tap gather
    Bc, Hi, C = 2, 4, 3
    n_in = Bc * Hi * Hi * 16 * C
    Ec = Bc * 4 * Hi * Hi * C
    g = rng(3)
    col, col2 = torch.randn(G * n_in, generator=g), torch.randn(2 * n_in, generator=g)
    grp = torch.tensor([1, 0, 1], dtype=torch.int32)
    bias = torch.randn(C, generator=g)
    xc = torch.rand(T * Ec, generator=g)
    rawc = torch.empty(G * Ec)
    emu.col2im(col, rawc, G * Bc, Hi, Hi, C, bias=bias, col2=col2, grp_src=grp, imgs_per_group=Bc)
    dc, pc = torch.empty(G * Ec), torch.empty(G * 32)
    emu.sigmoid_mse(rawc, xc, tgt, coef, G, Ec, None, dc, pc)
    L.check_convt_c1_loss(col, col2, grp, bias, xc, tgt, coef, G, Bc, Hi, Hi, C, dc, pc, per_chunk=False, worst=worst)

    out = torch.empty(4)
    kl, al = torch.tensor([12.5]), torch.rand(7, generator=g)
    for has_cpc, n_align in ((True, 2), (False, 0)):
        emu.finalize_losses(part, 2, has_cpc, E, kl, 4.0, al, n_align, 30.0, out)
        L.check_finalize(out, part, 2, has_cpc, E, kl, 4.0, al, n_align, 30.0, worst=worst)

    n = 3 * 8192 + 5
    mu, lv, mu_p, lv_p, eps, eps_p = reparam_data(n)
    z, zp, ks = torch.empty(n), torch.empty(n), torch.empty(1)
    emu.reparam_kl_fwd(mu, lv, mu_p, lv_p, eps, eps_p, z, zp, n, ks)
    L.check_reparam_kl_fwd(mu, lv, mu_p, lv_p, eps, eps_p, z, zp, n, ks, worst=worst)
    dz = torch.randn(n, generator=g)
    outs = [torch.empty(n) for _ in range(4)]
    emu.reparam_kl_bwd(mu, lv, mu_p, lv_p, eps, eps_p, dz, None, 0.25, *outs, n)
    L.check_reparam_kl_bwd(mu, lv, mu_p, lv_p, eps, eps_p, dz, None, 0.25, *outs, n, worst=worst)

    S, Bb, gd, z_ = 4, 5, 6, 3
    H = torch.randn(T * Bb * gd, generator=g)
    Z = torch.randn(S * Bb * z_, generator=g)
    ia, ib = torch.tensor([0, 1, 2, 3], dtype=torch.int32), torch.tensor([3, 1, 0, 2], dtype=torch.int32)
    tuc, dt = torch.rand(S, generator=g), torch.rand(S, generator=g)
    ld = gd + z_ + 2 + 5
    dst = torch.empty(S * Bb * ld)
    emu.build_concat(dst, H, ia, gd, Z, ib, z_, tuc, dt, S, Bb, ld=ld)
    L.assert_bitexact("build_concat", dst, L.build_concat_ref(H, ia, gd, Z, ib, z_, tuc, dt, S, Bb, ld))
    W = 2 * gd + 2
    src = torch.randn(S * Bb * W, generator=g)
    idx = torch.tensor([1, 3, 1, 4], dtype=torch.int32)
    for init in (False, True):
        d0 = torch.randn(T * Bb * gd, generator=g)
        d = d0.clone()
        emu.gather_add_cols(d, src, idx, S, T, Bb, gd, W, gd, init=init)
        L.check_gather_add_cols(d, d0, src, idx, S, T, Bb, gd, W, gd, init, worst=worst)

    hp = torch.randn(S * Bb * gd, generator=g)
    dh0, dH0 = torch.randn(S * Bb * gd, generator=g), torch.randn(T * Bb * gd, generator=g)
    lp, dh, dH = torch.empty(S - 1), dh0.clone(), dH0.clone()
    emu.align(H, ia, hp, S - 1, Bb, gd, 0.5, lp, dh, dH)
    L.check_align(H, ia, hp, S - 1, Bb, gd, 0.5, lp, dh0, dh, dH0, dH, worst=worst)

    for rows, cols, ld_ in ((16384, 1, 1), (300, 7, 9)):
        xs = torch.rand(rows * ld_, generator=g)
        o0 = torch.randn(cols, generator=g)
        o = o0.clone()
        emu.colsum(xs, rows, cols, ld_, o, accumulate=True)
        L.check_colsum(xs, rows, cols, ld_, o0, o, True, 1 << 22, worst=worst)

    xa = torch.randn(5000, generator=g) * 3
    for act in (L.ACT_NONE, L.ACT_LRELU, L.ACT_TANH, L.ACT_RELU):      # the emulation has no sigmoid activation
        y = xa.clone()
        emu.act_fwd(y, y.numel(), act)
        L.assert_bound(f"act_fwd {act}", y, *L.act_fwd_ref(xa, act), None, worst)
        dy, dx = torch.randn(5000, generator=g), torch.empty(5000)
        emu.act_bwd(dy, y, dx, 5000, act)
        L.assert_bound(f"act_bwd {act}", dx, *L.act_bwd_ref(dy, y, act), None, worst)

    rows, C = 700, 96
    xl = torch.randn(rows * C, generator=g) * 2 + 1
    gm, bt = torch.randn(C, generator=g), torch.randn(C, generator=g)
    y, mean, rstd = torch.empty(rows * C), torch.empty(rows), torch.empty(rows)
    emu.layernorm_fwd(xl, gm, bt, y, mean, rstd, rows, C)
    L.check_layernorm_fwd(xl, gm, bt, y, mean, rstd, rows, C, worst=worst)
    dyl = torch.randn(rows * C, generator=g)
    dxl, dgm, dbt = torch.empty(rows * C), torch.empty(C), torch.empty(C)
    emu.layernorm_bwd(dyl, xl, mean, rstd, gm, dxl, dgm, dbt, rows, C)
    L.check_layernorm_bwd(dyl, xl, mean, rstd, gm, dxl, dgm, dbt, rows, C, worst=worst)

    n = 1000
    p0, gr, m0 = (torch.randn(n, generator=g) for _ in range(3))
    v0 = torch.rand(n, generator=g)
    for t in (1, 1000):
        p, m, v = p0.clone(), m0.clone(), v0.clone()
        emu.adam(p, gr, m, v, n, 1e-3, 0.9, 0.999, 1e-8, torch.tensor([t], dtype=torch.int32))
        L.check_adam(p0, gr, m0, v0, p, m, v, n, 1e-3, 0.9, 0.999, 1e-8, t, worst=worst)

    src = torch.randn(3 * 45 * 77, generator=g)
    for dt_ in (torch.float32, torch.bfloat16):
        dst = torch.empty(src.numel(), dtype=dt_)
        emu.transpose_batched(src, dst, 3, 45, 77)
        L.assert_bitexact("transpose", dst, L.transpose_ref(src, 3, 45, 77, dt_))
        bd = torch.empty(4 * 5 * 4 * 7, dtype=dt_)
        emu.blockdiag(src, bd, 5, 7, 4)
        L.assert_bitexact("blockdiag", bd, L.blockdiag_ref(src, 5, 7, 4, dt_))
    L.report(worst, "emulation")
    assert all(v <= 1.0 for v in worst.values())


# ------------------------------------------------------------------ corruptions are rejected

CORRUPT = ["one MSE chunk dropped", "sigmoid derivative without (1 - s)", "KL partials of CTA 7 dropped",
           "align row 0 replaced by row b", "colsum missing its last row", "Adam without bias correction",
           "transpose_batched with P and Q swapped"]


@pytest.mark.parametrize("corrupt", CORRUPT)
def test_corruption_rejected(corrupt):
    with pytest.raises(AssertionError) as ei:
        run_corrupted(corrupt)
    print(corrupt, "->", str(ei.value)[:200])


def test_uncorrupted_versions_pass():
    """The kernel-layout emulations used for the corruptions pass the checker unchanged (so a rejection is the corruption's)."""
    run_corrupted(None)


def run_corrupted(corrupt):
    raw, x, tgt, coef = loss_data()
    d_raw, part = sigmoid_mse_like(raw, x, tgt, coef, corrupt)
    L.check_sigmoid_mse(raw, x, tgt, coef, G, E, None, d_raw, part)

    n = 8 * L.RKL_THREADS * 2 + 300
    mu, lv, mu_p, lv_p, eps, eps_p = reparam_data(n)
    s1, s2 = (0.5 * lv).exp(), (0.5 * lv_p).exp()
    k = torch.log(s2 / s1) + (lv.exp() + (mu - mu_p) ** 2) / (2 * lv_p.exp()) - 0.5
    if corrupt == "KL partials of CTA 7 dropped":
        k = torch.where((torch.arange(n) // L.RKL_THREADS) % L.RKL_CTAS == 7, torch.zeros_like(k), k)
    ks = k.double().sum().float().reshape(1)
    L.check_reparam_kl_fwd(mu, lv, mu_p, lv_p, eps, eps_p, eps * s1 + mu, eps_p * s2 + mu_p, n, ks)

    g = rng(7)
    P, Bb, gd = 3, 9, 130
    H = torch.randn(T * Bb * gd, generator=g)
    in_idx = torch.tensor([2, 0, 4], dtype=torch.int32)
    hp = torch.randn(P * Bb * gd, generator=g)
    dh0, dH0 = torch.randn(P * Bb * gd, generator=g), torch.randn(T * Bb * gd, generator=g)
    lp, dh, dH = align_like(H, in_idx, hp, P, Bb, gd, 0.5, dh0, dH0, corrupt)
    L.check_align(H, in_idx, hp, P, Bb, gd, 0.5, lp, dh0, dh, dH0, dH)

    rows = 16384
    xs = torch.rand(rows * 3, generator=g)
    xm = xs.view(rows, 3)
    out = (xm[:-1] if corrupt == "colsum missing its last row" else xm).double().sum(0).float()
    L.check_colsum(xs, rows, 3, 3, None, out, False, 1 << 22)

    na = 500
    p0, gr, m0 = (torch.randn(na, generator=g) for _ in range(3))
    v0 = torch.rand(na, generator=g)
    p, m, v = adam_like(p0, gr, m0, v0, na, 1e-3, 0.9, 0.999, 1e-8, 3, corrupt)
    L.check_adam(p0, gr, m0, v0, p, m, v, na, 1e-3, 0.9, 0.999, 1e-8, 3)

    A, Pq, Q = 2, 16, 48
    src = torch.randn(A * Pq * Q, generator=g)
    if corrupt == "transpose_batched with P and Q swapped":
        dst = src.reshape(A, Q, Pq).transpose(1, 2).reshape(-1)
    else:
        dst = src.reshape(A, Pq, Q).transpose(1, 2).reshape(-1)
    L.assert_bitexact("transpose_batched", dst, L.transpose_ref(src, A, Pq, Q, torch.float32))


# ------------------------------------------------------------------ the mirror

@pytest.mark.parametrize("cfg", ["C2", "C3", "C4", "C5"])
def test_mirror_matches_bench(cfg):
    import bench
    c = bench.CONFIGS[cfg]
    sh = L.bench_shapes(cfg)
    assert sh["S"] == c["T"] - 1 and sh["G"] == c["T"] and sh["has_cpc"]
    frame = 51 if c["backbone"] == "h36m_mlp" else c["channels"] * c["width"] ** 2
    assert sh["E"] == c["per_gpu"] * frame
    assert sh["reparam_n"] == sh["S"] * c["per_gpu"] * bench.Z_DIM
    assert sh["align"]["P"] == sh["S"] - 1 and sh["finalize"]["n_align"] == sh["S"] - 1
    assert sh["in_idx"] == list(range(sh["S"])) + [sh["S"] - 1]


def test_launch_shape_numbers():
    """The figures the issue of these tests quotes, and both sides of the host-side decisions."""
    c2, c4 = L.bench_shapes("C2"), L.bench_shapes("C4")
    assert (c2["G"], c2["E"], c2["loss"], c2["Hi"], c2["C"]) == (30, 1 << 20, "convt_c1_loss", 32, 1)
    assert (c4["loss"], c4["Hi"], c4["C"]) == ("convt_c1_loss", 64, 3)
    assert L.bench_shapes("C3")["loss"] == "sigmoid_mse" and L.bench_shapes("C2", False)["loss"] == "sigmoid_mse"
    assert L.bench_shapes("C5", False)["loss"] == "mse_plain"
    last = [r for w, r, cols, _ in c2["colsum"] if w == "decoder last bias"][0]
    assert last == 29 * 256 * 64 * 64
    ws = 1 << 22
    plan = L.colsum_plan(last, 1, 1, ws)
    assert [l["fold"] for l in plan] == [True, True] and plan[0]["cols"] == 256 and plan[1]["rows"] == 256
    assert not L.colsum_plan(16383, 1, 1, ws)[0]["fold"] and L.colsum_plan(16384, 1, 1, ws)[0]["fold"]
    assert not L.colsum_plan(16384 + 128, 1, 1, ws)[0]["fold"] and not L.colsum_plan(65536, 5, 5, ws)[0]["fold"]
    assert not L.colsum_plan(65536, 3, 4, ws)[0]["fold"] and not L.colsum_plan(65536, 1, 1, 1025 * 256 - 1)[0]["fold"]
    p = L.colsum_plan(29 * 256, 1024, 1024, ws)[0]
    assert (p["nchunk"], p["rpc"]) == (34, 219)
    assert L.colsum_chain(plan, False) == sum(math.ceil(l["rpc"] / 8) + 8 + l["nchunk"] for l in plan)
    assert L.ln_bwd_chunks(15360) == (60, 256) and L.ln_bwd_chunks(100) == (1, 100)
    per, total = L.arena_numel(__import__("bench").oracle_cfg(__import__("bench").CONFIGS["C2"])[0])
    assert total == 12681280 and per["decoder"] == 6558532
