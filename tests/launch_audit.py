"""What the launch tests of every backbone share (tests/test_dcgan_launches_gpu.py, test_vgg_launches_gpu.py,
test_vgg128_launches_gpu.py, test_mlp_launches_gpu.py): fixtures, seeded operands, one training step from the seeded initial
state, a view of CudaKernels that records what the step launches, and a view that checks each launch against float64 on its
own operands as it runs.

A test module imports the fixtures it uses by name (K, sms and the autouse memory_per_test).  A backbone declares what its
recording logs per entry point (RecordingKernels.RECORD), and subclasses AuditKernels with its own audits and with the class
attributes that set how the shared GEMM audit bounds and probes its launches.

The kernel an fp32 GEMM runs on (wgmma .tf32 or gemm_simt with its split-K schedule) and the bound of gemm_simt's fp32 sum
live here too: the h36m_mlp tests and the fp32 dcgan / vgg tests all launch it.
"""
import gc
import inspect
import time

import numpy as np
import pytest
import torch

from oracle import p2p_oracle as O
from p2pvg_b200._lib import CudaKernels
from p2pvg_b200.engine import StepPlan
from tests.lstm_schedule import gamma
from tests.ref64 import EPS, assert_exact, bn_group_ref64, bound_check, finalize_ref, gemm_ref64
from tests.tc_schedule import BETA, alpha_for, assert_within, cdiv, image_slices, sm_count

BENCH_OPT = dict(skip_prob=0.0, n_past=1, last_frame_skip=False)
SKIP_OPT = dict(skip_prob=0.5, n_past=2, last_frame_skip=True)
NAN = float("nan")
# BatchNorm sums: fp32 per-thread running sums, combined in float64 (test_bn_backward_gpu.py ALPHA)
ALPHA_BN = 2.0 ** -14


@pytest.fixture(scope="module")
def K():
    return CudaKernels("cuda")


@pytest.fixture(scope="module")
def sms():
    return sm_count()


@pytest.fixture(autouse=True)
def memory_per_test(request):
    if torch.cuda.is_available():
        torch.cuda.reset_peak_memory_stats()
        t0 = time.time()
    yield
    if torch.cuda.is_available():
        release()
        print(f"\n[memory] {request.node.name}: {time.time() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


def release():
    """Hand freed device memory back: an engine whose backbone methods are wrapped (watch_backbone) refers to itself, so it
    goes with the garbage collector, not with its last name."""
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def randn(*shape, scale=1.0, dtype=torch.bfloat16):
    return (torch.randn(*shape, device="cuda") * scale).to(dtype)


def slices_with_boundary(N, HW, s, sms, B):
    """Tile-aligned image ranges of the first, middle and last round, each a launch of <= SMs tiles; the middle one straddles
    the boundary between two groups of B images."""
    unit = max(1, s.BM // HW)
    first, _, last = image_slices(N, HW, unit, s, sms)
    ni = first[1]
    if ni < 2:
        return [first, last]
    b = (N // 2) // B * B
    i0 = max(unit, (b - ni // 2) // unit * unit)
    return [first, (i0, min(N, i0 + ni)), last]


def addend_index(srcl, ipg, N, device="cuda"):
    """The addend image each of N output images reads: image n of group n // ipg reads image n % ipg of source srcl[n // ipg]."""
    return torch.tensor([srcl[n // ipg] * ipg + n % ipg for n in range(N)], device=device)


def skip_seed(T):
    """The first probability seed whose SKIP_OPT plan reads at least three skip sources."""
    opt = O.default_opt(**SKIP_OPT)
    for seed in range(100):
        p = StepPlan(T, np.random.RandomState(seed).uniform(0, 1, T - 1), opt)
        if len(set(p.skip_src)) >= 3:
            return seed
    raise AssertionError("no seed gives three skip sources")


def bn_inputs(G, R, C, seed, dt=torch.bfloat16):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    raw = (torch.randn(G * R * C, device="cuda", generator=gen) * 1.5 + 0.3).to(dt)
    gamma = torch.rand(C, device="cuda", generator=gen) + 0.5
    beta = torch.randn(C, device="cuda", generator=gen) * 0.5
    return raw, gamma, beta, gen


def bn_stats(K, raw, G, R, C, gamma_, beta):
    st = {k: torch.full((G * C,), NAN, device="cuda") for k in ("mean", "invstd", "varu", "scale", "shift", "sdz", "sdzx")}
    K.bn_fwd_stats(raw, G, R, C, gamma_, beta, st["mean"], st["invstd"], st["varu"], st["scale"], st["shift"])
    return st


def check_bn_stats(st, raw, G, R, C, gamma_, beta, name):
    """bn_fwd_stats against float64 group by group (finalize_ref's bounds with sums known within ALPHA_BN)."""
    x = raw.reshape(-1)[:G * R * C].view(G, R, C)
    s1 = torch.stack([x[g].double().sum(0) for g in range(G)])
    s2 = torch.stack([(x[g].double() ** 2).sum(0) for g in range(G)])
    m1 = torch.stack([x[g].double().abs().sum(0) for g in range(G)])
    w = 0.0
    for got, (ref, bnd), nm in zip((st["mean"], st["invstd"], st["varu"], st["scale"], st["shift"]),
                                   finalize_ref(s1, s2, m1, R, gamma_, beta, EPS, ALPHA_BN), ("mean", "invstd", "varu", "scale", "shift")):
        w = max(w, bound_check(got.reshape(-1)[:G * C].view(G, C), ref, bnd, f"{name} {nm}"))
    return w


def bn_side(raw, scale, shift, G, R, C):
    """The LeakyReLU slope side bn_bwd takes without y: the sign of its fp32 raw * scale + shift."""
    return raw.reshape(-1)[:G * R * C].view(G, R, C).double() * scale.reshape(-1)[:G * C].view(G, 1, C).double() \
        + shift.reshape(-1)[:G * C].view(G, 1, C).double() > 0


def bn_bwd_refs(raw, dy, st, gamma_, beta, G, R, C, act, y=None):
    """Per-group float64 references of bn_bwd (ref64.bn_group_ref64): LeakyReLU on the slope side of st's scale / shift,
    tanh from the stored y."""
    x, d = raw.reshape(-1)[:G * R * C].view(G, R, C), dy.reshape(-1)[:G * R * C].view(G, R, C)
    side = bn_side(raw, st["scale"], st["shift"], G, R, C) if act == 1 else None
    refs = []
    for g in range(G):
        r = bn_group_ref64(x[g], d[g], gamma_, beta, act, side=side[g] if side is not None else None,
                           y=y.reshape(-1)[:G * R * C].view(G, R, C)[g] if y is not None else None)
        refs.append({k: r[k] for k in ("dx", "dx_mag", "sdz", "sdz_mag", "sdzx", "sdzx_mag")})
    return refs


def check_bn_bwd(res, refs, G, C, name, dx_dtype=torch.bfloat16):
    """dx (stored in dx_dtype), sum dz, sum dz*xhat per group, and dgamma / dbeta, against the per-group float64 references:
    the BatchNorm sums within ALPHA_BN of their magnitudes, dx within that plus one rounding to dx_dtype."""
    w = 0.0
    for g, r in enumerate(refs):
        w = max(w, assert_within(res["dx"][g], r["dx"], r["dx_mag"], 0, dx_dtype, alpha=ALPHA_BN, quiet=True, name=f"{name} dx group {g}"))
        w = max(w, assert_within(res["sdz"].reshape(-1)[:G * C].view(G, C)[g], r["sdz"], r["sdz_mag"], 0, torch.float32, alpha=ALPHA_BN,
                                 quiet=True, name=f"{name} sum_dz group {g}"))
        w = max(w, assert_within(res["sdzx"].reshape(-1)[:G * C].view(G, C)[g], r["sdzx"], r["sdzx_mag"], 0, torch.float32,
                                 alpha=ALPHA_BN, quiet=True, name=f"{name} sum_dzx group {g}"))
    if "dgamma" in res:
        dg, db = sum(r["sdzx"] for r in refs), sum(r["sdz"] for r in refs)
        w = max(w, assert_within(res["dgamma"], dg, sum(r["sdzx_mag"] for r in refs), 0, torch.float32, alpha=ALPHA_BN, name=f"{name} dgamma"))
        w = max(w, assert_within(res["dbeta"], db, sum(r["sdz_mag"] for r in refs), 0, torch.float32, alpha=ALPHA_BN, name=f"{name} dbeta"))
    return w


def check_bn_param_grad(sdz, sdzx, G, C, dgamma, dbeta, name):
    """bn_param_grad: dgamma / dbeta = the per-group sums of sum_dzx / sum_dz over G groups, within G fp32 roundings."""
    w = 0.0
    for got, part in ((dgamma, sdzx), (dbeta, sdz)):
        p = part.reshape(-1)[:G * C].view(G, C).double()
        w = max(w, bound_check(got.reshape(-1)[:C], p.sum(0), G * 2.0 ** -24 * p.abs().sum(0) + 1e-30, name))
    return w


# ------------------------------------------------------------------ the kernel an fp32 GEMM runs on, and its bound

TF32_FLAG, TF32_REQUIRE = 1, 2   # include/p2pvg_b200.h P2PVG_GEMM_TF32 / P2PVG_GEMM_TF32_REQUIRE
GEMM_WS_BYTES = 256 << 20        # CudaKernels.gemm_workspace()
SIMT_BM = SIMT_BN = 64           # gemm_simt.cu:12
SIMT_BK = 16


def gemm_ws_bytes(kernels):
    """The split-K workspace a GEMM launch of this backend gets (the lane's CudaKernels.gemm_workspace())."""
    return kernels.gemm_workspace().numel()


def _tma_ok(off_elems, ld):
    """gemm_tc.cu:180-182 tc_operand_ok for fp32: a 16-byte aligned base (every engine buffer and every arena view starts
    16-byte aligned, engine.py:108) and a 16-byte multiple pitch."""
    return (off_elems * 4) % 16 == 0 and (ld * 4) % 16 == 0


def simt_split(M, N, K, ws_bytes=GEMM_WS_BYTES):
    """gemm_simt.cu:101-113: (splits, k_per_split)."""
    splits, kps = 1, (K if K > 0 else 1)
    tiles = cdiv(M, SIMT_BM) * cdiv(N, SIMT_BN)
    if tiles < 74 and K >= 2048 and ws_bytes > 0:
        want = (296 + tiles - 1) // tiles
        maxs = K // 256
        splits = min(want, maxs)
        while splits > 1 and splits * M * N * 4 > ws_bytes:
            splits //= 2
        splits = max(1, splits)
        kps = cdiv(cdiv(K, splits), SIMT_BK) * SIMT_BK
        splits = cdiv(K, kps)
    return splits, kps


def kernel_for(M, N, K, a_mn, b_mn, lda, ldb, a_off, b_off, tf32, ws_bytes=GEMM_WS_BYTES):
    """api.cu:51-64 with gemm_tc.cu:183-189: an fp32 GEMM of a view with P2PVG_GEMM_TF32 (tf32=True) runs on wgmma .tf32 if
    both operands are K-major, K >= 32 and both are TMA-compatible; everything else runs on gemm_simt, split over K by
    simt_split.  Returns "tf32", "simt" or ("simt-splitK", splits, k_per_split)."""
    if tf32 and not a_mn and not b_mn and K >= 32 and _tma_ok(a_off, lda) and _tma_ok(b_off, ldb):
        return "tf32"
    s, kps = simt_split(M, N, K, ws_bytes)
    return "simt" if s == 1 else ("simt-splitK", s, kps)


def entry_kernel(e, tf32, ws_bytes=GEMM_WS_BYTES):
    """kernel_for of a derived launch-list entry (operands given as (buffer, element offset))."""
    return kernel_for(e["M"], e["N"], e["K"], e["a_mn"], e["b_mn"], e["lda"], e["ldb"], e["A"][1], e["B"][1], tf32, ws_bytes)


def simt_alpha(K, kern, extra):
    """Relative bound (to sum_k |a_k b_k| + |bias| + |addend| + |C0|) of gemm_simt's fp32 result.  Each output element is one
    thread's fmaf chain over its k range (gemm_simt.cu:62-71): acc = fmaf(a_k, b_k, acc) rounds once per term, so a chain of n
    terms is within gamma(n) of its exact sum relative to the sum of the magnitudes (Higham, Thm 3.1; the zero-filled loads past
    K add nothing).  Without split-K n = K, and the epilogue adds bias, addend and C0 with one rounding each (:87-90).  With
    split-K every z slice is a chain over k_per_split terms, stored as it is (fp32), and splitk_reduce_kernel
    (gemm_tc.cu:144-149) sums the `splits` partials in ascending z from 0 (one rounding per add) before bias / addend / C0.
    Every partial sum along the way is bounded by the total magnitude, so the whole is gamma(k_per_split + splits + extra);
    `extra` counts the epilogue adds."""
    if kern == "simt":
        return gamma(K + extra)
    _, splits, kps = kern
    return gamma(kps + splits + extra)


def simt_bound(kernels, M, N, K, a_mn=False, b_mn=False, extra=0):
    """(alpha, kernel) of an fp32 GEMM on gemm_simt with the split-K schedule this backend's workspace allows."""
    kern = kernel_for(M, N, K, a_mn, b_mn, 1, 1, 0, 0, False, gemm_ws_bytes(kernels))
    return simt_alpha(K, kern, extra), kern


# ------------------------------------------------------------------ fp32 launch lists (tests/dcgan_ref.py, tests/vgg_ref.py)

# the entry points an fp32 dcgan / vgg step's backbone methods launch that the fp32 launch lists name
FP32_OPS = ("gemm", "im2col", "col2im", "im2col3", "col2im3", "gather_add", "group_sum", "add_indexed", "bn_fwd_stats", "bn_act",
            "bn_bwd", "bn_param_grad", "sigmoid_mse", "colsum")


def gemm32(name, M, N, K, a_mn=False, b_mn=False, lda=None, ldb=None, ldc=None, accumulate=False, bias=False):
    """An fp32 GEMM of a launch list, CudaKernels.gemm's defaults (_lib.py:198-203) filled in."""
    lda = lda if lda is not None else (M if a_mn else K)
    ldb = ldb if ldb is not None else (N if b_mn else K)
    ldc = ldc if ldc is not None else N
    return dict(op="gemm", name=name, M=M, N=N, K=K, a_mn=a_mn, b_mn=b_mn, lda=lda, ldb=ldb, ldc=ldc, accumulate=accumulate,
                bias=bias, key=("gemm", M, N, K, a_mn, b_mn, lda, ldb, ldc, accumulate, bias))


def op32(op, name, *args):
    """Any other entry of an fp32 launch list: what fp32_call_key logs for the call."""
    return dict(op=op, name=name, args=args, key=(op,) + args)


def fp32_call_key(op, x):
    """What a recording of an fp32 step logs for one call of entry point `op` with arguments x (by name; CudaKernels and
    tests/emu_backend.EmuKernels alike)."""
    nn = lambda v: v is not None   # noqa: E731
    if op == "gemm":
        lda = x["lda"] if x["lda"] is not None else (x["M"] if x["a_mn"] else x["K"])
        ldb = x["ldb"] if x["ldb"] is not None else (x["N"] if x["b_mn"] else x["K"])
        ldc = x["ldc"] if x["ldc"] is not None else x["N"]
        assert x["addend"] is None
        return ("gemm", x["M"], x["N"], x["K"], bool(x["a_mn"]), bool(x["b_mn"]), lda, ldb, ldc, bool(x["accumulate"]), nn(x["bias"]))
    if op == "im2col":
        assert x["H"] == x["W"]
        return ("im2col", x["N"], x["H"], x["C"])
    if op == "col2im":
        assert x["Hi"] == x["Wi"] and not x["accumulate"]
        return ("col2im", x["N"], x["Hi"], x["C"], nn(x["bias"]), nn(x["col2"]), x["imgs_per_group"])
    if op == "im2col3":
        return ("im2col3", x["N"], x["H"], x["C"], x["ld"], x["sgn"])
    if op == "col2im3":
        return ("col2im3", x["N"], x["H"], x["C"], x["ld"], nn(x["bias"]))
    if op == "gather_add":
        return ("gather_add", x["G"], x["n"])
    if op == "group_sum":
        return ("group_sum", x["G"], x.get("F", x.get("F_")), x["n"])
    if op == "add_indexed":
        return ("add_indexed", x.get("F", x.get("F_")), x["n"])
    if op in ("bn_fwd_stats",):
        return (op, x["G"], x["R"], x["C"])
    if op in ("bn_act", "bn_bwd"):
        return (op, x["G"], x["R"], x["C"], x["act"])
    if op == "bn_param_grad":
        return (op, x["G"], x["C"])
    if op == "sigmoid_mse":
        return (op, x["G"], x["E"])
    if op == "colsum":
        assert not x["accumulate"]
        return (op, x["rows"], x["cols"], x["ld"])
    raise KeyError(op)


def gemm_alpha(K, kern, extra):
    """alpha for assert_within of one fp32-operand GEMM on the kernel that ran it: alpha_for(K, tf32=True) for wgmma .tf32 (its
    16 spare steps cover the epilogue adds), simt_alpha otherwise."""
    return alpha_for(K, tf32=True) if kern == "tf32" else simt_alpha(K, kern, extra)


# ------------------------------------------------------------------ float64 checkers of the skip sums and fp32 GEMMs

def check_group_sum(inp, out, srcl, G, F_, n, name, chunk=1 << 24):
    """out[f] = the sum of the groups g of inp with srcl[g] == f (group_sum / the skip sums: fp32 in group order from zero, one
    output rounding), in chunks of the n elements per group; zeros for a source no group reads.  Returns the worst ratio."""
    iv = inp.reshape(-1)[:G * n].view(G, n)
    ov = out.reshape(-1)[:F_ * n].view(F_, n)
    w = 0.0
    for f in range(F_):
        gs = [g for g in range(G) if srcl[g] == f]
        for j0 in range(0, n, chunk):
            j1 = min(n, j0 + chunk)
            ref = torch.zeros(j1 - j0, dtype=torch.float64, device=inp.device)
            mag = torch.zeros_like(ref)
            for g in gs:
                x = iv[g, j0:j1].double()
                ref += x
                mag += x.abs()
            w = max(w, bound_check(ov[f, j0:j1], ref, len(gs) * 2.0 ** -24 * mag + BETA[out.dtype] * ref.abs(),
                                   f"{name} source {f} elements [{j0}, {j1})"))
    return w


def check_simt_gemm(C, A, B, M, N, K, a_mn, b_mn, lda, ldb, ldc, kern, bias=None, c0=None, rows=None, name=""):
    """An fp32 GEMM on gemm_simt against float64 on strided operands, within simt_alpha of the split schedule `kern` that ran
    it (c0: C before an accumulating launch).  rows = (m0, m1): those rows of C only.  Returns the worst ratio."""
    m0, m1 = rows if rows is not None else (0, M)
    ref, absref = gemm_ref64(A, B, M, N, K, a_mn, b_mn, lda, ldb, bias=bias, rows=(m0, m1),
                             c0=c0[m0:m1] if c0 is not None else None)
    got = C.as_strided((M, N), (ldc, 1))[m0:m1]
    extra = int(bias is not None) + int(c0 is not None)
    return assert_within(got, ref, absref, K, torch.float32, alpha=simt_alpha(K, kern, extra), quiet=True,
                         name=f"{name} {M}x{N}x{K} on {kern} rows [{m0}, {m1})")


# ------------------------------------------------------------------ one training step

def snapshot(eng):
    return {m: (eng.arena[m].flat.clone(), {k: v.clone() for k, v in eng.buffers[m].items()}) for m in O.MODULES}


def restore(eng, snap):
    """Back to the initial state IN PLACE (captured graphs keep pointing at the same arenas)."""
    for m in O.MODULES:
        A = eng.arena[m]
        A.flat.copy_(snap[m][0])
        A.grad.zero_()
        A.m.zero_()
        A.v.zero_()
        A.step_t.zero_()
        for k, v in snap[m][1].items():
            eng.buffers[m][k].copy_(v)


def step_inputs(cfg, optkw, T, B, np_seed):
    """(opt, probs, plan, x, eps) of one step, on the host: frames uniform in [0, 1) (for the mlp backbone poses of std 3, as
    bench.py synth_batch draws them) and skip probabilities drawn from np_seed."""
    opt = O.default_opt(**optkw)
    opt["batch_size"] = B
    probs = np.random.RandomState(np_seed).uniform(0, 1, T - 1)
    plan = StepPlan(T, probs, opt)
    gen = torch.Generator().manual_seed(5)
    if cfg.get("backbone") == "mlp":
        x = 3 * torch.randn(T, B, 17, 3, generator=gen)
    else:
        x = torch.rand(T, B, cfg["channels"], cfg["image_width"], cfg["image_width"], generator=gen)
    eps = O.draw_eps(plan.S, B, cfg["z_dim"], seed=11)
    return opt, probs, plan, x, eps


def assert_concurrent(eng, x):
    assert eng.concurrent, "the step does not run its concurrent lanes"


def assert_serial(eng, x):
    """The fp32 step runs on the caller's stream alone: no side lanes (TrainEngine.fork is then a no-op)."""
    assert not eng.concurrent and not eng.streams, "the fp32 step runs side lanes"


def run_step(engine_cls, cfg, optkw, kernels, T, B, np_seed, use_graph=False, act_dtype=torch.bfloat16, prepare=None):
    """One step of engine_cls on `kernels` from the seeded initial state: (plan, (losses, gradients, parameters)).
    prepare(eng, x) runs before the step.  use_graph: the step replayed from a captured CUDA graph, the engine restored in
    place to its initial state before the replay."""
    opt, probs, plan, x, eps = step_inputs(cfg, optkw, T, B, np_seed)
    eng = engine_cls(O.build_state(cfg, seed=1), cfg, opt, kernels, act_dtype=act_dtype)
    x, eps = x.cuda(), eps.cuda()
    if prepare is not None:
        prepare(eng, x)
    if use_graph:
        snap = snapshot(eng)
        for _ in range(2):   # eager warm-up, then capture
            eng.step(x, probs=probs, eps=eps, use_graph=True)
        restore(eng, snap)
        del snap
        losses = eng.step(x, probs=probs, eps=eps, use_graph=True)
        assert any(v != "warm" for v in eng._graphs.values()), "the step was not graph-replayed"
    else:
        losses = eng.step(x, probs=probs, eps=eps)
    torch.cuda.synchronize()
    out = (np.asarray(losses), {m: {k: v.detach().clone() for k, v in eng.arena[m].g.items()} for m in eng.arena},
           {m: {k: v.detach().clone() for k, v in eng.arena[m].p.items()} for m in eng.arena})
    del eng
    release()
    return plan, out


def assert_equal_steps(a, b, what):
    """(losses, gradients, parameters) of two steps are equal bit for bit."""
    assert np.array_equal(a[0], b[0]), f"{what}: losses {a[0]} vs {b[0]}"
    for i, kind in ((1, "grad"), (2, "param")):
        for m in a[i]:
            for k in a[i][m]:
                assert torch.equal(a[i][m][k], b[i][m][k]), f"{what}: {kind} {m}.{k} differs"


def audit_step(engine_cls, cfg, optkw, T, B, audit, expect, label, prepare=None, act_dtype=torch.bfloat16):
    """One eager step in act_dtype on plain CudaKernels (bf16: with its concurrent lanes; fp32: serial, no lanes), then the
    same step on `audit` (an AuditKernels), every audited launch checked as it runs.  expect(plan) -> (variants, skip reads):
    every variant must occur in the audited step, and the skip sources it read must be exactly those.  The audited step must
    equal the plain one bit for bit.  A skip plan draws its probabilities from skip_seed.  Returns (plan, the plain step's
    results)."""
    np_seed = skip_seed(T) if optkw.get("skip_prob") else 0
    lanes = assert_concurrent if act_dtype == torch.bfloat16 else assert_serial
    plan, plain = run_step(engine_cls, cfg, optkw, CudaKernels("cuda"), T, B, np_seed, act_dtype=act_dtype, prepare=lanes)
    if optkw.get("skip_prob"):
        assert len(set(plan.skip_src)) >= 3
    _, audited = run_step(engine_cls, cfg, optkw, audit, T, B, np_seed, act_dtype=act_dtype, prepare=prepare)
    want, reads = expect(plan)
    missing = want - audit.seen
    assert not missing, f"launch variants that did not occur in the step: {sorted(missing, key=str)}"
    assert sorted(audit.skip_reads) == sorted(reads), f"skip sources read: {audit.skip_reads}, the schedule says {reads}"
    gemms = "GEMM " if audit.REPORT_GEMMS_ONLY else ""
    worst = max((w for _, v, w in audit.log if not gemms or v[0].startswith("gemm")), default=0.0)
    print(f"[audit] {label}: {len(audit.log)} launches checked, worst {gemms}error/bound {worst:.3g}")
    assert_equal_steps(plain, audited, f"{label}: the audited step")
    return plan, plain


# ------------------------------------------------------------------ recording and audited views of CudaKernels

def _recorded(op):
    sig = inspect.signature(getattr(CudaKernels, op))

    def method(self, *a, **kw):
        x = sig.bind(self, *a, **kw)
        x.apply_defaults()
        t = self.RECORD[op](self, x.arguments)
        if t is not None:
            self.calls.append(t)
        return self.launch(op, x.arguments)
    return method


class RecordingKernels(CudaKernels):
    """CudaKernels that logs one tuple per call of each entry point named in RECORD, then calls through.  RECORD maps an entry
    point to f(kernels, arguments by name) -> the tuple to log, or None to log nothing."""
    RECORD = {}

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.calls = []

    def __init_subclass__(cls, **kw):
        super().__init_subclass__(**kw)
        for op in cls.RECORD:
            setattr(cls, op, _recorded(op))

    def launch(self, op, args):
        return getattr(CudaKernels, op)(**args)


class AuditKernels(CudaKernels):
    """CudaKernels whose audited launches are each checked against float64 on their own operands right after they run (device
    synchronised around each call; inputs a call overwrites are cloned first; nothing the step reads is changed).  Each check
    appends (what, variant, worst error/bound) to `log` and the variant to `seen`; launches with a skip addend append the
    sources they read to `skip_reads`.  Here: GEMMs, group_sum and add_indexed; a backbone adds its own entry points."""
    PRINT_RECORDS = False           # print an [audit] line per checked launch
    REPORT_GEMMS_ONLY = False       # audit_step reports the worst ratio of the GEMMs alone
    GEMM_FP32 = True                # check GEMMs with fp32 operands (else they run unchecked)
    GEMM_ACCUMULATE = True          # a GEMM may accumulate or take an addend (else either is an error)
    GEMM_PROBE_K = 1 << 16          # fp32-output GEMMs from this K on are rerun on the 0 / 1 pattern of their operands
    GEMM_PROBE_ACCUMULATING = True  # ... also those that accumulate

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.log, self.seen, self.skip_reads = [], set(), []
        self._sms = sm_count()

    def _rec(self, what, v, worst):
        self.log.append((what, v, worst))
        self.seen.add(v)
        if self.PRINT_RECORDS:
            print(f"[audit] {what} {v}: worst error/bound {worst:.3g}")

    def _sync(self, op, *a):
        """CudaKernels' entry point op, the device synchronised before and after."""
        torch.cuda.synchronize()
        getattr(CudaKernels, op)(self, *a)
        torch.cuda.synchronize()

    def _addend(self, addend, grp_src, imgs_per_group, N, Ho, Cn):
        """(the addend images a launch over N images reads, as [images, Ho, Ho, Cn], the index of the one each image reads);
        grp_src[:groups] goes to skip_reads."""
        ipg = max(1, imgs_per_group)
        srcl = grp_src.tolist()[:cdiv(N, ipg)]
        self.skip_reads.append(srcl)
        nimg = (max(srcl) + 1) * ipg
        return addend.view(-1)[:nimg * Ho * Ho * Cn].view(nimg, Ho, Ho, Cn), addend_index(srcl, ipg, N, addend.device)

    def gemm(self, A, B, C, M, N, K, a_mn=False, b_mn=False, lda=None, ldb=None, ldc=None, accumulate=False, bias=None,
             addend=None, ldd=None):
        args = (A, B, C, M, N, K, a_mn, b_mn, lda, ldb, ldc, accumulate, bias, addend, ldd)
        if A.dtype != torch.bfloat16 and not self.GEMM_FP32:
            return super().gemm(*args)
        assert self.GEMM_ACCUMULATE or (not accumulate and addend is None)
        lda_ = lda if lda is not None else (M if a_mn else K)
        ldb_ = ldb if ldb is not None else (N if b_mn else K)
        ldc_ = ldc if ldc is not None else N
        cv = C.as_strided((M, N), (ldc_, 1))
        torch.cuda.synchronize()
        c0 = cv.clone() if accumulate else None
        self._sync("gemm", *args)
        alpha, kern = self.gemm_bound(A, B, M, N, K, a_mn, b_mn, lda_, ldb_, int(bias is not None) + int(addend is not None) + int(accumulate))
        add = addend.as_strided((M, N), (ldd if ldd is not None else N, 1)) if addend is not None else None
        # the full K bounds every split-K schedule the launcher may pick
        w, step = 0.0, max(1, (1 << 22) // N)
        for m0 in range(0, M, step):
            m1 = min(M, m0 + step)
            ref, absref = gemm_ref64(A, B, M, N, K, a_mn, b_mn, lda_, ldb_, bias=bias, rows=(m0, m1),
                                     addend=add[m0:m1] if add is not None else None, c0=c0[m0:m1] if c0 is not None else None)
            w = max(w, assert_within(cv[m0:m1], ref, absref, K, C.dtype, alpha=alpha, quiet=True,
                                     name=f"audit gemm {M}x{N}x{K} {A.dtype}->{C.dtype} a_mn={a_mn} b_mn={b_mn} on {kern} rows {m0}"))
        if K >= self.GEMM_PROBE_K and C.dtype == torch.float32 and (self.GEMM_PROBE_ACCUMULATING or not accumulate):
            # long reductions (weight gradients) cancel and the bound above is loose: the same launch on the 0 / 1 pattern of
            # the operands must be exact
            A01, B01 = (A > 0).to(A.dtype), (B > 0).to(B.dtype)
            probe = torch.full((M, N), NAN, device=C.device)
            super().gemm(A01, B01, probe, M, N, K, a_mn, b_mn, lda, ldb)
            assert_exact(probe, gemm_ref64(A01, B01, M, N, K, a_mn, b_mn, lda_, ldb_)[0], K, f"audit gemm {M}x{N}x{K} 0/1 probe")
        self._rec(f"gemm {M}x{N}x{K}", self.gemm_variant(A, kern, a_mn, b_mn, accumulate, bias, ldc_ != N), w)

    def gemm_bound(self, A, B, M, N, K, a_mn, b_mn, lda, ldb, extra):
        """(alpha of the launch's accumulation bound, the kernel it runs on); extra: bias, addend and accumulate terms."""
        tf32 = A.dtype == torch.float32 and self.gemm_flags == 1
        return alpha_for(K, tf32=tf32), "tf32" if tf32 else "-"

    def gemm_variant(self, A, kern, a_mn, b_mn, accumulate, bias, strided):
        return ("gemm", str(A.dtype)[6:], kern)

    def _skip_sums(self, inp, out, srcl, G, F_, n, what):
        return check_group_sum(inp, out, srcl, G, F_, n, f"audit {what}")

    def group_sum(self, inp, out, grp_src, G, F_, n):
        self._sync("group_sum", inp, out, grp_src, G, F_, n)
        self._rec(f"group_sum G={G} F={F_}", ("group_sum",), self._skip_sums(inp, out, grp_src.tolist()[:G], G, F_, n, "group_sum"))

    def add_indexed(self, dst, src, dst_idx, F_, n):
        torch.cuda.synchronize()
        di = dst_idx.tolist()[:F_]
        d0 = [dst.view(-1)[d * n:(d + 1) * n].clone() for d in di]
        self._sync("add_indexed", dst, src, dst_idx, F_, n)
        w = 0.0
        for f, d in enumerate(di):
            ref = d0[f].double() + src.view(-1)[f * n:(f + 1) * n].double()
            w = max(w, bound_check(dst.view(-1)[d * n:(d + 1) * n], ref, BETA[dst.dtype] * ref.abs(), "audit add_indexed"))
        self._rec(f"add_indexed F={F_}", ("add_indexed",), w)


# ------------------------------------------------------------------ fp32 dcgan / vgg steps: recording, audit, GEMMs at shape

BACKBONE = ("encode", "decode", "losses_fwd", "decoder_backward", "encoder_backward")


def watch_backbone(eng):
    """Sets eng.K.on while the engine runs a backbone method (everything outside the recurrent phase)."""
    for nm in BACKBONE:
        f = getattr(eng, nm)

        def w(*a, _f=f, **kw):
            eng.K.on = True
            try:
                return _f(*a, **kw)
            finally:
                eng.K.on = False
        setattr(eng, nm, w)


class Fp32Recording(RecordingKernels):
    """Logs fp32_call_key of every FP32_OPS launch of the backbone methods (while `on`)."""
    on = False
    RECORD = {op: (lambda op: lambda k, x: fp32_call_key(op, x) if k.on else None)(op) for op in FP32_OPS}


def recorded_fp32_step(engine_cls, cfg, optkw, T, B):
    """One eager fp32 step on Fp32Recording from the seeded initial state: (plan, recorded keys, peak device memory in GiB of
    the step, engine construction included)."""
    release()
    torch.cuda.reset_peak_memory_stats()
    rec = Fp32Recording("cuda")
    np_seed = skip_seed(T) if optkw.get("skip_prob") else 0
    plan, (losses, _, _) = run_step(engine_cls, cfg, optkw, rec, T, B, np_seed, act_dtype=torch.float32,
                                    prepare=lambda eng, x: (assert_serial(eng, x), watch_backbone(eng)))
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    assert np.all(np.isfinite(losses))
    return plan, rec.calls, peak


class SimtAudit(AuditKernels):
    """AuditKernels whose fp32 GEMMs are bounded by simt_alpha of the split-K schedule gemm_simt takes with this backend's
    workspace (the fp32 step never sets P2PVG_GEMM_TF32), with the unfused BatchNorm entry points of the fp32 step
    (bn_fwd_stats, bn_act, bn_bwd, bn_param_grad) checked against float64 too."""
    GEMM_PROBE_K = 1 << 12

    def gemm_bound(self, A, B, M, N, K, a_mn, b_mn, lda, ldb, extra):
        assert A.dtype == torch.float32 and not self.gemm_flags & TF32_FLAG
        kern = kernel_for(M, N, K, a_mn, b_mn, lda, ldb, 0, 0, False, gemm_ws_bytes(self))
        return simt_alpha(K, kern, extra), kern

    def gemm_variant(self, A, kern, a_mn, b_mn, accumulate, bias, strided):
        return ("gemm", kern if isinstance(kern, str) else kern[0], a_mn, b_mn, bias is not None)

    def bn_fwd_stats(self, x, G, R, C, gamma_, beta, mean, invstd, var_unb, scale, shift, eps=1e-5):
        self._sync("bn_fwd_stats", x, G, R, C, gamma_, beta, mean, invstd, var_unb, scale, shift, eps)
        xv = x.reshape(-1)[:G * R * C].view(G, R, C)
        s1 = torch.stack([xv[g].double().sum(0) for g in range(G)])
        s2 = torch.stack([(xv[g].double() ** 2).sum(0) for g in range(G)])
        m1 = torch.stack([xv[g].double().abs().sum(0) for g in range(G)])
        w = 0.0
        for got, (ref, bnd), nm in zip((mean, invstd, var_unb, scale, shift), finalize_ref(s1, s2, m1, R, gamma_, beta, eps, ALPHA_BN),
                                       ("mean", "invstd", "varu", "scale", "shift")):
            w = max(w, bound_check(got.view(-1)[:G * C].view(G, C), ref, bnd, f"audit bn_fwd_stats G={G} R={R} C={C} {nm}"))
        self._rec(f"bn_fwd_stats G={G} R={R} C={C}", ("bn_fwd_stats",), w)

    def bn_bwd(self, dy, x, y, mean, invstd, gamma_, G, R, C, act, dx, sum_dz, sum_dzx, scale=None, shift=None):
        torch.cuda.synchronize()
        d0 = dy.reshape(-1)[:G * R * C].clone()
        self._sync("bn_bwd", dy, x, y, mean, invstd, gamma_, G, R, C, act, dx, sum_dz, sum_dzx, scale, shift)
        st = dict(scale=scale, shift=shift)
        refs = bn_bwd_refs(x, d0, st, gamma_, torch.zeros_like(gamma_), G, R, C, act, y=y if act != 1 else None)
        w = check_bn_bwd(dict(dx=dx.reshape(-1)[:G * R * C].view(G, R, C), sdz=sum_dz, sdzx=sum_dzx), refs, G, C,
                         f"audit bn_bwd G={G} R={R} C={C}", dx_dtype=dx.dtype)
        self._rec(f"bn_bwd G={G} R={R} C={C}", ("bn_bwd", act), w)

    def bn_param_grad(self, sum_dz, sum_dzx, G, C, dgamma, dbeta):
        self._sync("bn_param_grad", sum_dz, sum_dzx, G, C, dgamma, dbeta)
        self._rec(f"bn_param_grad G={G} C={C}", ("bn_param_grad",),
                  check_bn_param_grad(sum_dz, sum_dzx, G, C, dgamma, dbeta, f"audit bn_param_grad G={G} C={C}"))

    def bn_act(self, x, y, scale, shift, G, R, C, act):
        self._sync("bn_act", x, y, scale, shift, G, R, C, act)
        xv, yv = x.reshape(-1)[:G * R * C].view(G, R, C), y.reshape(-1)[:G * R * C].view(G, R, C)
        sc, sh = scale.view(-1)[:G * C].view(G, 1, C).double(), shift.view(-1)[:G * C].view(G, 1, C).double()
        w = 0.0
        for g in range(G):
            pre = xv[g].double() * sc[g] + sh[g]
            mag = (xv[g].double() * sc[g]).abs() + sh[g].abs()
            # fmaf(x, scale, shift) rounds once, the activation once more (tanh: within a few ulp)
            ref = torch.where(pre > 0, pre, 0.2 * pre) if act == 1 else torch.tanh(pre)
            bnd = 2.0 ** -23 * mag + (2.0 ** -23 * ref.abs() if act == 1 else 2.0 ** -21)
            w = max(w, bound_check(yv[g], ref, bnd, f"audit bn_act G={G} R={R} C={C} group {g}"))
        self._rec(f"bn_act G={G} R={R} C={C}", ("bn_act", act), w)


def _fill_rows(v, values, gen):
    """Fill the 2-D (possibly pitched) view v in row chunks: randn, binary (0 / 1, 1 with probability 1/4), positive (uniform
    [0, 1)) or half (normal of mean 1/2 and std 1/2)."""
    step = max(1, (1 << 26) // v.shape[1])
    for r0 in range(0, v.shape[0], step):
        c = v[r0:r0 + step]
        if values == "randn":
            c.copy_(torch.randn(c.shape, device="cuda", generator=gen))
        elif values == "binary":
            c.copy_((torch.rand(c.shape, device="cuda", generator=gen) < 0.25).float())
        elif values == "positive":
            c.copy_(torch.rand(c.shape, device="cuda", generator=gen))
        else:
            c.copy_(torch.randn(c.shape, device="cuda", generator=gen) * 0.5 + 0.5)


SENTINEL = -777.0


def gemm32_at_shape(K, e, seed, label):
    """One fp32 GEMM of a launch list (gemm32 entry) at its shape and pitches, on gemm_simt: operands in buffers whose
    elements outside the operands are NaN, the output's tail a sentinel.  Every output element must be written and nothing
    past it; rows of the first, middle and last part of the output against float64 within simt_alpha of the split schedule
    this backend takes.  A weight gradient (both operands MN-major) must be exact on 0 / 1 operands (K < 2^24) and within the
    bound on operands that do not cancel.  Returns (kernel, worst ratio)."""
    M, N, Kd, a_mn, b_mn, lda, ldb, ldc = e["M"], e["N"], e["K"], e["a_mn"], e["b_mn"], e["lda"], e["ldb"], e["ldc"]
    assert not e["accumulate"]
    kern = kernel_for(M, N, Kd, a_mn, b_mn, lda, ldb, 0, 0, False, gemm_ws_bytes(K))
    name = f"{label} {e['name']} {M}x{N}x{Kd} lda={lda} ldb={ldb} on {kern}"
    gen = torch.Generator(device="cuda").manual_seed(seed)
    ar, ac = (Kd, M) if a_mn else (M, Kd)
    br, bc = (Kd, N) if b_mn else (N, Kd)
    Abuf = torch.full((ar * lda + 64,), NAN, device="cuda")
    Bbuf = torch.full((br * ldb + 64,), NAN, device="cuda")
    Av, Bv = Abuf[:ar * lda].view(ar, lda)[:, :ac], Bbuf[:br * ldb].view(br, ldb)[:, :bc]
    Cbuf = torch.full((M * ldc + 64,), SENTINEL, device="cuda")
    Cv = Cbuf[:M * ldc].view(M, ldc)[:, :N]
    bias = torch.randn(N, device="cuda", generator=gen) if e["bias"] else None
    wgrad = a_mn and b_mn
    r = min(M, 4) if wgrad else min(M, max(1, (1 << 22) // N))
    rows = sorted({(0, r), (max(0, M // 2 - r // 2), max(0, M // 2 - r // 2) + r), (M - r, M)})

    def launch(values):
        _fill_rows(Av, values, gen)
        _fill_rows(Bv, "half" if values == "positive" else values, gen)
        Cv.fill_(NAN)
        K.gemm(Abuf, Bbuf, Cbuf, M, N, Kd, a_mn, b_mn, lda, ldb, ldc, bias=bias if values == "randn" else None)
        torch.cuda.synchronize()
        assert (Cbuf[M * ldc:] == SENTINEL).all(), f"{name}: elements past the output were written"
        for r0 in range(0, M, max(1, (1 << 26) // N)):
            assert not torch.isnan(Cv[r0:r0 + (1 << 26) // N]).any(), f"{name}: unwritten output elements from row {r0}"

    launch("randn")
    w = max(check_simt_gemm(Cbuf, Abuf, Bbuf, M, N, Kd, a_mn, b_mn, lda, ldb, ldc, kern, bias=bias, rows=rr, name=name)
            for rr in rows)
    if wgrad:
        assert Kd < 1 << 24
        launch("binary")
        for rr in rows:
            ref = gemm_ref64(Abuf, Bbuf, M, N, Kd, True, True, lda, ldb, rows=rr)[0]
            assert_exact(Cv[rr[0]:rr[1]], ref, Kd, f"{name} 0/1 operands rows [{rr[0]}, {rr[1]})")
        launch("positive")
        for rr in rows:
            ref, absref = gemm_ref64(Abuf, Bbuf, M, N, Kd, True, True, lda, ldb, rows=rr)
            assert (ref.abs() >= 0.25 * absref).all()
            w = max(w, check_simt_gemm(Cbuf, Abuf, Bbuf, M, N, Kd, True, True, lda, ldb, ldc, kern, rows=rr,
                                       name=name + " non-cancelling operands"))
    print(f"[bound] {name}: worst error/bound {w:.3g}")
    del Abuf, Bbuf, Cbuf
    release()
    return kern, w
