"""The loss, latent, bias-sum, weight-pack and Adam kernels against float64 (tests/loss_ref.py): at the arguments one step of
the benchmark configurations passes them, on both sides of every host-side launch decision, and at the edges where an index,
chunk count or scale could go wrong.  Stored outputs start as NaN with a NaN tail (every element written, nothing past the
end); accumulated outputs start from nonzero values."""
import pytest
import torch

from tests import loss_ref as L

pytestmark = pytest.mark.gpu

NAN = float("nan")
TAIL = 97
WORST = {}


@pytest.fixture(scope="module")
def K():
    from p2pvg_b200._lib import CudaKernels
    return CudaKernels("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _report():
    torch.cuda.reset_peak_memory_stats()
    yield
    L.report(WORST, "loss/optim")
    print(f"[memory] peak max_memory_allocated {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def canary(n, dtype=torch.float32):
    return torch.full((n + TAIL,), NAN, dtype=dtype, device="cuda")


def assert_tail(name, t, n):
    assert bool(t[n:].isnan().all()), f"{name}: an element past the end ({n}) was written"


def ws_floats(K):
    return K.bn_workspace(1, 1).numel() // 4


def frames(T, E, g):
    return torch.rand(T * E, generator=g, device="cuda")


def loss_inputs(sh):
    S, T = sh["S"], sh["T"]
    tgt = torch.tensor(list(range(1, S + 1)) + [T - 1], dtype=torch.int32, device="cuda")   # tgt_idx of the step's plan
    coef = torch.tensor([1.0] * S + [100.0], device="cuda")                                  # recon calls, weight_cpc
    return tgt, coef


LAUNCH = [("C2", True), ("C2", False), ("C3", True), ("C4", True), ("C4", False), ("C5", False)]


@pytest.mark.parametrize("cfg,bf16", LAUNCH, ids=[f"{c}-{'bf16' if b else 'fp32'}" for c, b in LAUNCH])
def test_loss_at_launch_shape(K, cfg, bf16):
    """The reconstruction loss of one step (convt_c1_loss, sigmoid_mse or mse_plain as the engine picks it) and the loss
    finaliser on its partials."""
    sh = L.bench_shapes(cfg, bf16)
    G, E, T, B = sh["G"], sh["E"], sh["T"], sh["B"]
    g = gen(1)
    tgt, coef = loss_inputs(sh)
    x = frames(T, E, g)
    partial = canary(G * L.MSE_CHUNKS)
    adt = torch.bfloat16 if bf16 else torch.float32
    if sh["loss"] == "convt_c1_loss":
        Hi, C = sh["Hi"], sh["C"]
        n_in = B * Hi * Hi * 16 * C
        col = (torch.randn(G * n_in, generator=g, device="cuda") * 0.6).to(adt)
        col2 = (torch.randn(n_in, generator=g, device="cuda") * 0.6).to(adt)          # one skip source (n_past = 1)
        grp = torch.zeros(G, dtype=torch.int32, device="cuda")
        bias = torch.randn(C, generator=g, device="cuda") * 0.1
        d_raw = canary(G * E, adt)
        K.convt_c1_loss(col, col2, grp, bias, x, tgt, coef, G, B, Hi, Hi, d_raw, partial, C=C)
        torch.cuda.synchronize()
        assert_tail("convt_c1_loss d_raw", d_raw, G * E)
        L.check_convt_c1_loss(col, col2, grp, bias, x, tgt, coef, G, B, Hi, Hi, C, d_raw[:G * E], partial, worst=WORST)
        del col
    elif sh["loss"] == "sigmoid_mse":
        raw = (torch.randn(G * E, generator=g, device="cuda") * 2).to(adt)
        d_raw = canary(G * E, adt)
        K.sigmoid_mse(raw, x, tgt, coef, G, E, None, d_raw, partial)
        torch.cuda.synchronize()
        assert_tail("sigmoid_mse d_raw", d_raw, G * E)
        L.check_sigmoid_mse(raw, x, tgt, coef, G, E, None, d_raw[:G * E], partial, worst=WORST)
    else:
        x = torch.randn(T * E, generator=g, device="cuda") * 3                           # poses, standardised to std 3
        pred = x.reshape(T, E)[tgt.long()].reshape(-1) + torch.randn(G * E, generator=g, device="cuda")
        d_pred = canary(G * E)
        K.mse_plain(pred, x, tgt, coef, G, E, d_pred, partial)
        torch.cuda.synchronize()
        assert_tail("mse_plain d_pred", d_pred, G * E)
        L.check_mse_plain(pred, x, tgt, coef, G, E, d_pred[:G * E], partial, worst=WORST)
    assert_tail("mse partial", partial, G * L.MSE_CHUNKS)
    f = sh["finalize"]
    kl = torch.tensor([1234.5], device="cuda")
    al = torch.rand(f["n_align"] + 1, generator=g, device="cuda") * 1e-3
    out = canary(4)
    K.finalize_losses(partial, f["n_recon"], f["has_cpc"], f["E"], kl, f["batch_size"], al, f["n_align"], f["seq_len"], out)
    torch.cuda.synchronize()
    assert_tail("finalize out", out, 4)
    L.check_finalize(out, partial, f["n_recon"], f["has_cpc"], f["E"], kl, f["batch_size"], al, f["n_align"], f["seq_len"], worst=WORST)


@pytest.mark.parametrize("cfg", ["C2", "C3", "C4", "C5"])
def test_latent_at_launch_shape(K, cfg):
    """reparam_kl forward / backward, build_concat, gather_add_cols and align at the step's shapes and index tables."""
    sh = L.bench_shapes(cfg)
    S, T, B, g, z = sh["S"], sh["T"], sh["B"], sh["g"], sh["z"]
    gg = gen(2)
    n = sh["reparam_n"]
    mu, lv, mu_p, lv_p = (torch.randn(n, generator=gg, device="cuda") * s for s in (1.0, 0.5, 1.0, 0.5))
    eps, eps_p = (torch.randn(n, generator=gg, device="cuda") for _ in range(2))
    zz, zp, kl = canary(n), canary(n), canary(1)
    K.reparam_kl_fwd(mu, lv, mu_p, lv_p, eps, eps_p, zz, zp, n, kl)
    dz = torch.randn(n, generator=gg, device="cuda")
    outs = [canary(n) for _ in range(4)]
    K.reparam_kl_bwd(mu, lv, mu_p, lv_p, eps, eps_p, dz, None, 1e-4 / B, *outs, n)     # backward #1: beta / batch_size
    torch.cuda.synchronize()
    for t in (zz, zp, *outs):
        assert_tail("reparam_kl", t, n)
    assert_tail("kl_sum", kl, 1)
    L.check_reparam_kl_fwd(mu, lv, mu_p, lv_p, eps, eps_p, zz, zp, n, kl, worst=WORST)
    L.check_reparam_kl_bwd(mu, lv, mu_p, lv_p, eps, eps_p, dz, None, 1e-4 / B, *outs, n, worst=WORST)
    dzp = torch.randn(n, generator=gg, device="cuda")
    K.reparam_kl_bwd(mu, lv, mu_p, lv_p, eps, eps_p, None, dzp, 1.0 / B, *outs, n)     # backward #2
    L.check_reparam_kl_bwd(mu, lv, mu_p, lv_p, eps, eps_p, None, dzp, 1.0 / B, *outs, n, worst=WORST)

    H = torch.randn(T * B * g, generator=gg, device="cuda")
    Z = torch.randn((S + 1) * B * z, generator=gg, device="cuda")
    in_idx = torch.tensor(sh["in_idx"], dtype=torch.int32, device="cuda")
    tgt = torch.tensor(list(range(1, S + 1)) + [T - 1], dtype=torch.int32, device="cuda")
    glob = torch.full((S + 1,), T - 1, dtype=torch.int32, device="cuda")
    tuc = torch.rand(S + 1, generator=gg, device="cuda")
    dt = torch.rand(S + 1, generator=gg, device="cuda")
    for (steps, width), (A, ia, ga, Bm, ib, gb) in zip(sh["concat"], [(H, tgt, g, H, glob, g), (H, in_idx, g, Z, torch.arange(S + 1, dtype=torch.int32, device="cuda"), z)]):
        ld = (width + 7) // 8 * 8 + 8                       # a padded pitch, as in_pitch gives the TMA-compatible rows
        dst = canary(steps * B * ld)
        K.build_concat(dst, A, ia, ga, Bm, ib, gb, tuc, dt, steps, B, ld=ld)
        torch.cuda.synchronize()
        assert_tail("build_concat", dst, steps * B * ld)
        L.assert_bitexact("build_concat", dst[:steps * B * ld], L.build_concat_ref(A, ia, ga, Bm, ib, gb, tuc, dt, steps, B, ld))
    for (steps, W, col0), idx in zip(sh["gather"], (tgt, glob, in_idx)):
        src = torch.randn(steps * B * W, generator=gg, device="cuda")
        for init in (False, True):
            d0 = torch.randn(T * B * g, generator=gg, device="cuda")
            dst = torch.cat([d0, torch.full((TAIL,), NAN, device="cuda")])
            K.gather_add_cols(dst, src, idx, steps, T, B, g, W, col0, init=init)
            torch.cuda.synchronize()
            assert_tail("gather_add_cols", dst, T * B * g)
            L.check_gather_add_cols(dst[:T * B * g], d0, src, idx, steps, T, B, g, W, col0, init, worst=WORST)
    run_align(K, H, in_idx, S - 1, T, B, g, sh["align"]["coef"], gg)


def run_align(K, H, in_idx, P, T, B, g, coef, gg):
    N = T * B * g
    hp = torch.randn((P + 1) * B * g, generator=gg, device="cuda")
    dh0 = torch.randn((P + 1) * B * g, generator=gg, device="cuda")
    dH0 = torch.randn(N, generator=gg, device="cuda")
    lp, dh, dH = canary(P), dh0.clone(), dH0.clone()
    K.align(H, in_idx, hp, P, B, g, coef, lp, dh, dH)
    torch.cuda.synchronize()
    assert_tail("align loss_partial", lp, P)
    assert torch.equal(dh[P * B * g:], dh0[P * B * g:]), "align wrote d_hpred past pair P-1"
    L.check_align(H, in_idx, hp, P, B, g, coef, lp[:P], dh0, dh, dH0, dH, worst=WORST)


@pytest.mark.parametrize("g", [128, 100, 200])
@pytest.mark.parametrize("B", [256, 13])
def test_align_widths(K, g, B):
    """Column passes of 128 with a partial one (g = 100, 200), idle row lanes (B = 13), every pair count the step can pass."""
    S, T = 29, 30
    gg = gen(3 + g + B)
    H = torch.randn(T * B * g, generator=gg, device="cuda")
    in_idx = torch.randperm(T, generator=torch.Generator().manual_seed(g * B))[:S].to(torch.int32).cuda()   # distinct frames
    for P in range(1, S):
        run_align(K, H, in_idx, P, T, B, g, 0.5, gg)


# ------------------------------------------------------------------ colsum

COLSUM = [  # rows, cols, ld, bf16, accumulate, fold expected
    (16383, 1, 1, False, False, False),
    (16384, 1, 1, False, False, True),
    (16384 + 128, 1, 1, False, True, False),       # rows % 256 != 0
    (65536, 4, 4, False, True, True),
    (65536, 5, 5, False, False, False),            # cols > 4
    (65536, 3, 8, False, False, False),            # ld > cols
    (65536 * 4, 3, 3, True, True, True),           # bf16 input
    (7, 1024, 1024, False, False, False),          # fewer rows than one 64-row chunk
    (7424, 1024, 1024, False, True, False),        # the LSTM bias shape of C2
]


@pytest.mark.parametrize("rows,cols,ld,bf16,acc,fold", COLSUM)
def test_colsum_paths(K, rows, cols, ld, bf16, acc, fold):
    wsf = ws_floats(K)
    plan = L.colsum_plan(rows, cols, ld, wsf)
    assert plan[0]["fold"] == fold, plan
    run_colsum(K, rows, cols, ld, bf16, acc, gen(rows + cols), f"colsum {rows}x{cols}")


def run_colsum(K, rows, cols, ld, bf16, acc, gg, tag):
    """Positive data with sentinel rows of 2^12 first and last: a dropped row or chunk moves the sum far outside the bound."""
    x = torch.rand(rows * ld, generator=gg, device="cuda") * 0.75 + 0.25
    xm = x.view(rows, ld)
    xm[0, :cols] = 4096.0
    xm[-1, :cols] = 4096.0
    x = x.to(torch.bfloat16) if bf16 else x
    o0 = torch.randn(cols, generator=gg, device="cuda")
    out = torch.cat([o0, torch.full((TAIL,), NAN, device="cuda")]) if acc else canary(cols)
    K.colsum(x, rows, cols, ld, out, accumulate=acc)
    torch.cuda.synchronize()
    assert_tail(tag, out, cols)
    L.check_colsum(x, rows, cols, ld, o0, out[:cols], acc, ws_floats(K), worst=WORST, tag=tag)


@pytest.mark.parametrize("cfg,bf16", [("C2", True), ("C2", False), ("C3", True), ("C4", True), ("C5", False)])
def test_colsum_at_launch_shapes(K, cfg, bf16):
    sh = L.bench_shapes(cfg, bf16)
    for i, (what, rows, cols, xb) in enumerate(sh["colsum"]):
        run_colsum(K, rows, cols, cols, xb, False, gen(10 + i), f"colsum {cfg} {what}")
    last = [c for c in sh["colsum"] if c[0] == "decoder last bias"]
    if last:
        assert L.colsum_plan(last[0][1], last[0][2], last[0][2], ws_floats(K))[0]["fold"], "the last-layer bias sum should fold"


# ------------------------------------------------------------------ reparam_kl edges, finaliser

@pytest.mark.parametrize("n", [74240, 8192 * 3 + 777, 0])
def test_reparam_kl_cluster(K, n):
    """All 8 CTAs of the cluster carry work (the C2 n, a ragged one); n = 0 still writes kl_sum = 0."""
    assert n == 0 or n > 7 * L.RKL_THREADS
    gg = gen(4)
    m = max(n, 1)
    mu, lv, mu_p, lv_p, eps, eps_p = (torch.randn(m, generator=gg, device="cuda") * 0.7 for _ in range(6))
    zz, zp, kl = canary(n), canary(n), canary(1)
    K.reparam_kl_fwd(mu, lv, mu_p, lv_p, eps, eps_p, zz, zp, n, kl)
    torch.cuda.synchronize()
    assert_tail("z", zz, n)
    assert_tail("kl_sum", kl, 1)
    if n == 0:
        assert kl[0].item() == 0.0
        return
    L.check_reparam_kl_fwd(mu, lv, mu_p, lv_p, eps, eps_p, zz, zp, n, kl, worst=WORST)


@pytest.mark.parametrize("has_cpc", [True, False])
@pytest.mark.parametrize("n_recon,n_align", [(29, 28), (59, 58), (5, 0), (1, 0)])
def test_finalize_losses(K, has_cpc, n_recon, n_align):
    gg = gen(5)
    partial = torch.rand((n_recon + 1) * L.MSE_CHUNKS, generator=gg, device="cuda") * 100
    al = torch.rand(max(n_align, 1) + 3, generator=gg, device="cuda")
    kl = torch.tensor([777.25], device="cuda")
    out = canary(4)
    E, bs, T = 256 * 4096, 256.0, 30.0
    K.finalize_losses(partial, n_recon, has_cpc, E, kl, bs, al, n_align, T, out)
    torch.cuda.synchronize()
    assert_tail("finalize", out, 4)
    L.check_finalize(out, partial, n_recon, has_cpc, E, kl, bs, al, n_align, T, worst=WORST)
    if not has_cpc:
        assert out[2].item() == 0.0
    if n_align == 0:
        assert out[3].item() == 0.0


# ------------------------------------------------------------------ activations, LayerNorm

@pytest.mark.parametrize("act", [L.ACT_NONE, L.ACT_LRELU, L.ACT_TANH, L.ACT_SIGMOID, L.ACT_RELU])
def test_activations(K, act):
    """Forward in place and backward, over several grid-stride rounds (the grid is capped at 132*16 blocks)."""
    n = L.GRID_CAP * 256 * 2 + 77
    gg = gen(6 + act)
    x = torch.randn(n, generator=gg, device="cuda") * 3
    y = torch.cat([x.clone(), torch.full((TAIL,), NAN, device="cuda")])
    K.act_fwd(y, n, act)
    torch.cuda.synchronize()
    assert_tail("act_fwd", y, n)
    ref, b = L.act_fwd_ref(x, act)
    L.assert_bound(f"act_fwd {act}", y[:n], ref, b, None, WORST)
    dy = torch.randn(n, generator=gg, device="cuda")
    dx = canary(n)
    K.act_bwd(dy, y, dx, n, act)
    torch.cuda.synchronize()
    assert_tail("act_bwd", dx, n)
    ref, b = L.act_bwd_ref(dy, y[:n], act)
    L.assert_bound(f"act_bwd {act}", dx[:n], ref, b, None, WORST)


def test_layernorm_c5(K):
    """C5's LayerNorm rows and width, forward and backward (dx aliasing dy, as the step calls it), dgamma/dbeta over many
    row chunks."""
    sh = L.bench_shapes("C5", False)
    ln = sh["layernorm"]
    C = ln["C"]
    gg = gen(7)
    gm = torch.randn(C, generator=gg, device="cuda") * 0.5 + 1
    bt = torch.randn(C, generator=gg, device="cuda") * 0.1
    for rows in ln["rows_fwd"]:
        x = torch.randn(rows * C, generator=gg, device="cuda") * 2 + 1.5
        y, mean, rstd = canary(rows * C), canary(rows), canary(rows)
        K.layernorm_fwd(x, gm, bt, y, mean, rstd, rows, C)
        torch.cuda.synchronize()
        for nm, t, k in (("y", y, rows * C), ("mean", mean, rows), ("rstd", rstd, rows)):
            assert_tail(f"layernorm_fwd {nm}", t, k)
        L.check_layernorm_fwd(x, gm, bt, y, mean, rstd, rows, C, worst=WORST)
    for rows in ln["rows_bwd"]:
        nchunk, _ = L.ln_bwd_chunks(rows)
        assert rows <= L.LN_ROW_CHUNK or nchunk > 1
        x = torch.randn(rows * C, generator=gg, device="cuda") * 2
        mean = x.view(rows, C).mean(1)
        rstd = torch.rsqrt(x.view(rows, C).var(1, unbiased=False) + 1e-5)
        dy = torch.randn(rows * C, generator=gg, device="cuda")
        buf = torch.cat([dy, torch.full((TAIL,), NAN, device="cuda")])
        dgm, dbt = canary(C), canary(C)
        K.layernorm_bwd(buf, x, mean, rstd, gm, buf, dgm, dbt, rows, C)       # dx aliases dy
        torch.cuda.synchronize()
        assert_tail("layernorm_bwd dx", buf, rows * C)
        assert_tail("layernorm_bwd dgamma", dgm, C)
        L.check_layernorm_bwd(dy, x, mean, rstd, gm, buf[:rows * C], dgm, dbt, rows, C, worst=WORST)


# ------------------------------------------------------------------ Adam

@pytest.mark.parametrize("which", ["1", "255", "C2 arena + tail"])
def test_adam(K, which):
    if which == "C2 arena + tail":
        n = L.bench_shapes("C2", with_arena=True)["arena_numel"] + 37
        assert L.grid_for(n) == L.GRID_CAP and n > 2 * L.GRID_CAP * 256
    else:
        n = int(which)
    gg = gen(8)
    p0 = torch.randn(n, generator=gg, device="cuda")
    gr = torch.randn(n, generator=gg, device="cuda") * 1e-2
    m0 = torch.randn(n, generator=gg, device="cuda") * 1e-3
    v0 = torch.rand(n, generator=gg, device="cuda") * 1e-4
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    for t in (1, 2, 1000, 10 ** 6):
        p, m, v = (torch.cat([a, torch.full((TAIL,), NAN, device="cuda")]) for a in (p0, m0, v0))
        step.fill_(t)
        K.adam(p, gr, m, v, n, 1e-3, 0.9, 0.999, 1e-8, step)
        torch.cuda.synchronize()
        for nm, a in (("p", p), ("m", m), ("v", v)):
            assert_tail(f"adam {nm}", a, n)
        L.check_adam(p0, gr, m0, v0, p, m, v, n, 1e-3, 0.9, 0.999, 1e-8, t, worst=WORST)


def test_adam_graph_reads_live_step(K):
    """A captured graph replayed after the step counter changed in device memory uses the new bias correction."""
    n = 4099
    gg = gen(9)
    p0, gr, m0 = (torch.randn(n, generator=gg, device="cuda") for _ in range(3))
    v0 = torch.rand(n, generator=gg, device="cuda")
    p, m, v = p0.clone(), m0.clone(), v0.clone()
    step = torch.ones(1, dtype=torch.int32, device="cuda")
    K.adam(p, gr, m, v, n, 1e-3, 0.9, 0.999, 1e-8, step)        # load the module outside the capture
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            K.adam(p, gr, m, v, n, 1e-3, 0.9, 0.999, 1e-8, step)
    torch.cuda.current_stream().wait_stream(s)
    for t in (1, 7):
        p.copy_(p0), m.copy_(m0), v.copy_(v0)
        step.fill_(t)
        graph.replay()
        torch.cuda.synchronize()
        L.check_adam(p0, gr, m0, v0, p, m, v, n, 1e-3, 0.9, 0.999, 1e-8, t, worst=WORST)
    assert L.adam_step_size(1e-3, 0.9, 0.999, 1) != L.adam_step_size(1e-3, 0.9, 0.999, 7)


# ------------------------------------------------------------------ weight packing

def _transpose_cases():
    cases = set()
    for cfg in ("C2", "C3", "C4", "C5"):
        for bf16 in (True, False):
            cases.update(L.bench_shapes(cfg, bf16)["transpose"])
    cases.update({(3, 45, 77, False, True), (2, 33, 1, False, False), (5, 1, 31, True, True), (1, 100, 65, False, False)})
    return sorted(cases)


def test_transpose_batched(K):
    """Every (A, P, Q) and dtype pair the engine passes, and P, Q off the 32-tile: bit-exact against permute + RNE cast."""
    gg = gen(10)
    cases = _transpose_cases()
    assert any(p % 32 and q % 32 for _, p, q, _, _ in cases)
    for A, P, Q, sb, db in cases:
        src = torch.randn(A * P * Q, generator=gg, device="cuda")
        src = src.to(torch.bfloat16) if sb else src
        dt = torch.bfloat16 if db else torch.float32
        dst = canary(A * P * Q, dt)
        K.transpose_batched(src, dst, A, P, Q)
        torch.cuda.synchronize()
        assert_tail(f"transpose {A}x{P}x{Q}", dst, A * P * Q)
        L.assert_bitexact(f"transpose_batched {A}x{P}x{Q} {src.dtype}->{dt}", dst[:A * P * Q], L.transpose_ref(src, A, P, Q, dt))
    from p2pvg_b200._lib import KernelError
    with pytest.raises(KernelError, match="transpose_batched"):
        K.transpose_batched(torch.zeros(8, device="cuda"), torch.zeros(8, device="cuda"), 65536, 1, 1)


def test_blockdiag(K):
    gg = gen(11)
    cases = {c + (True, True) for cfg in ("C2", "C4") for c in L.bench_shapes(cfg)["blockdiag"]}
    assert cases, "the 1/3-channel ends should use the block-diagonal weights"
    cases.update({(5, 7, 3, False, False), (64, 48, 4, False, True), (33, 16, 4, True, True)})
    for R, C, g, sb, db in sorted(cases):
        src = torch.randn(R * C, generator=gg, device="cuda")
        src = src.to(torch.bfloat16) if sb else src
        dt = torch.bfloat16 if db else torch.float32
        n = g * R * g * C
        dst = canary(n, dt)
        K.blockdiag(src, dst, R, C, g)
        torch.cuda.synchronize()
        assert_tail("blockdiag", dst, n)
        L.assert_bitexact(f"blockdiag {R}x{C} x{g}", dst[:n], L.blockdiag_ref(src, R, C, g, dt))


# ------------------------------------------------------------------ publish_scalars, convt_c1_loss limit

def test_publish_scalars(K):
    from p2pvg_b200._lib import KernelError
    for n in (4, 64):
        src = torch.randn(n, generator=gen(12), device="cuda")
        seq = torch.tensor([1000 + n], dtype=torch.int32, device="cuda")
        host = torch.full((n + 8,), NAN, dtype=torch.float32).pin_memory()
        K.publish_scalars(src, n, host, seq)
        torch.cuda.current_stream().synchronize()
        assert torch.equal(host[:n], src.cpu()), "published values differ"
        assert int(host[n:n + 1].view(torch.int32)[0]) == 1000 + n, "sequence number"
        assert bool(host[n + 1:].isnan().all()), "publish_scalars wrote past the sequence number"
    host = torch.zeros(80, dtype=torch.float32).pin_memory()
    for n in (0, 65):
        with pytest.raises(KernelError, match="publish_scalars"):
            K.publish_scalars(torch.zeros(80, device="cuda"), n, host, torch.zeros(1, dtype=torch.int32, device="cuda"))


def test_convt_c1_loss_index_limit(K):
    """B Hi Wi 16 C = 2^31 cannot be indexed in 32 bits: rejected before launch (tiny tensors suffice)."""
    from p2pvg_b200._lib import KernelError
    t = torch.zeros(64, dtype=torch.bfloat16, device="cuda")
    f = torch.zeros(64, device="cuda")
    i = torch.zeros(4, dtype=torch.int32, device="cuda")
    for B, Hi, C in ((32768, 64, 1), (2 ** 31 // (16 * 3 * 64 * 64) + 1, 64, 3)):
        assert B * Hi * Hi * 16 * C >= 2 ** 31
        with pytest.raises(KernelError, match="error -2.*32-bit"):
            K.convt_c1_loss(t, t, i, f, f, i, f, 1, B, Hi, Hi, t, f, C=C)
