"""What the launch tests of every backbone share (tests/test_dcgan_launches_gpu.py, test_vgg_launches_gpu.py,
test_vgg128_launches_gpu.py, test_mlp_launches_gpu.py): fixtures, seeded operands, one training step from the seeded initial
state, a view of CudaKernels that records what the step launches, and a view that checks each launch against float64 on its
own operands as it runs.

A test module imports the fixtures it uses by name (K, sms and the autouse memory_per_test).  A backbone declares what its
recording logs per entry point (RecordingKernels.RECORD), and subclasses AuditKernels with its own audits and with the class
attributes that set how the shared GEMM audit bounds and probes its launches.
"""
import inspect
import time

import numpy as np
import pytest
import torch

from oracle import p2p_oracle as O
from p2pvg_b200._lib import CudaKernels
from p2pvg_b200.engine import StepPlan
from tests.ref64 import assert_exact, bound_check, gemm_ref64
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


def bn_stats(K, raw, G, R, C, gamma, beta):
    st = {k: torch.full((G * C,), NAN, device="cuda") for k in ("mean", "invstd", "varu", "scale", "shift", "sdz", "sdzx")}
    K.bn_fwd_stats(raw, G, R, C, gamma, beta, st["mean"], st["invstd"], st["varu"], st["scale"], st["shift"])
    return st


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


def audit_step(engine_cls, cfg, optkw, T, B, audit, expect, label, prepare=None):
    """One eager bf16 step on plain CudaKernels, then the same step on `audit` (an AuditKernels), every audited launch checked
    as it runs.  expect(plan) -> (variants, skip reads): every variant must occur in the audited step, and the skip sources it
    read must be exactly those.  The audited step must equal the plain one bit for bit.  A skip plan draws its probabilities
    from skip_seed.  Returns (plan, the plain step's results)."""
    np_seed = skip_seed(T) if optkw.get("skip_prob") else 0
    plan, plain = run_step(engine_cls, cfg, optkw, CudaKernels("cuda"), T, B, np_seed, prepare=assert_concurrent)
    if optkw.get("skip_prob"):
        assert len(set(plan.skip_src)) >= 3
    _, audited = run_step(engine_cls, cfg, optkw, audit, T, B, np_seed, prepare=prepare)
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
        """out[f] = the sum of the groups g of inp with srcl[g] == f (fp32 in group order, one output rounding)."""
        iv = inp.view(-1)[:G * n].view(G, n)
        w = 0.0
        for f in range(F_):
            gs = [g for g in range(G) if srcl[g] == f]
            ref = iv[gs].double().sum(0) if gs else torch.zeros(n, dtype=torch.float64, device=inp.device)
            mag = iv[gs].double().abs().sum(0) if gs else torch.zeros_like(ref)
            w = max(w, bound_check(out.view(-1)[f * n:(f + 1) * n], ref, len(gs) * 2.0 ** -24 * mag + BETA[out.dtype] * ref.abs(),
                                    f"audit {what} source {f}"))
        return w

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
