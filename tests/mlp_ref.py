"""The h36m_mlp backbone's launches, mirrored on the host from p2pvg_b200/engine_mlp.py: the list of kernel calls one training
step makes outside the recurrent phase (tests/test_mlp_launches_gpu.py).  The kernel each fp32 GEMM of it runs on and the bound
of that kernel's fp32 sum are tests/launch_audit.py's kernel_for / entry_kernel / simt_alpha.

Operands are named by where they live: ("x", off) the input frames, ("p:<module>.<key>", off) / ("g:<module>.<key>", off) a
parameter / its gradient in the arena, ("<name>", off) the engine scratch buffer fbuf(<name>), off in elements from its start.
Line references are to engine_mlp.py unless stated; when the engine changes, they say what to re-read.
"""

POSE = 51               # 17 joints x 3 (engine.py:167)
ACT_TANH, ACT_RELU = 2, 4


def at(op, d):
    return (op[0], op[1] + d)


class _List:
    def __init__(self):
        self.L = []

    def gemm(self, name, A, B, C, M, N, K, a_mn=False, b_mn=False, lda=None, ldb=None, ldc=None, accumulate=False, bias=False):
        """CudaKernels.gemm's defaults (_lib.py:195-197) filled in."""
        self.L.append(dict(op="gemm", name=name, M=M, N=N, K=K, a_mn=a_mn, b_mn=b_mn,
                           lda=lda if lda is not None else (M if a_mn else K), ldb=ldb if ldb is not None else (N if b_mn else K),
                           ldc=ldc if ldc is not None else N, accumulate=bool(accumulate), bias=bool(bias), A=A, B=B, C=C))

    def op(self, op, name, *args):
        self.L.append(dict(op=op, name=name, args=tuple(args)))


def key(e):
    """What the recording kernels log for one call (tests/test_mlp_launches_gpu.py RecordingKernels)."""
    if e["op"] == "gemm":
        return ("gemm", e["M"], e["N"], e["K"], e["a_mn"], e["b_mn"], e["lda"], e["ldb"], e["ldc"], e["accumulate"], e["bias"],
                e["A"], e["B"], e["C"])
    return (e["op"],) + e["args"]


class _Lin:
    """Linear (:18-52): weight [Nout, Kt] of `mod`, column segments at koff."""

    def __init__(self, mod, name, Nout, Kt):
        self.mod, self.name, self.Nout, self.Kt = mod, name, Nout, Kt
        self.W, self.gW = (f"p:{mod}.{name}.weight", 0), (f"g:{mod}.{name}.weight", 0)

    def fwd(self, L, tag, segs, out, rows):   # :28-36
        koff = 0
        for i, (X, ks, ldx) in enumerate(segs):
            L.gemm(f"{tag}.{self.name} fwd seg{i}", X, at(self.W, koff), out, rows, self.Nout, ks, lda=ldx, ldb=self.Kt,
                   accumulate=i > 0, bias=i == 0)
            koff += ks

    def bwd(self, L, tag, segs, dY, rows, dsegs, want_wgrad=True):   # :38-52
        koff = 0
        for (X, ks, ldx), d in zip(segs, dsegs):
            if d is not None:
                L.gemm(f"{tag}.{self.name} dgrad seg", dY, at(self.W, koff), d[0], rows, ks, self.Nout, b_mn=True, ldb=self.Kt,
                       accumulate=d[1])
            if want_wgrad:
                L.gemm(f"{tag}.{self.name} wgrad seg", dY, X, at(self.gW, koff), self.Nout, ks, rows, a_mn=True, b_mn=True,
                       lda=self.Nout, ldb=ldx, ldc=self.Kt)
            koff += ks
        if want_wgrad:
            L.op("colsum", f"{tag}.{self.name} bias grad", dY, rows, self.Nout, self.Nout, (f"g:{self.mod}.{self.name}.bias", 0))


class _Res:
    """ResidualLinear (:55-122) of `mod`.`pre`, tag = its scratch-buffer prefix."""

    def __init__(self, mod, pre, tag, nin, nout):
        self.mod, self.pre, self.tag, self.nin, self.nout, self.mid = mod, pre, tag, nin, nout, nin // 2
        mid = self.mid
        self.sc = _Lin(mod, pre + ".shortcut.0", nout, nin)
        self.l1 = _Lin(mod, pre + ".long_path.0", mid, nin)
        self.l2 = _Lin(mod, pre + ".long_path.2", mid, mid)
        self.l3 = _Lin(mod, pre + ".long_path.4", nout, mid)

    def b(self, nm):
        return (f"{self.tag}_{nm}", 0)

    def fwd(self, L, segs, rows):   # :65-85
        nout, mid, b, t = self.nout, self.mid, self.b, self.tag
        self.sc.fwd(L, t, segs, b("sc"), rows)
        L.op("act_fwd", f"{t} relu sc", b("sc"), rows * nout, ACT_RELU)
        self.l1.fwd(L, t, segs, b("a1"), rows)
        L.op("act_fwd", f"{t} relu a1", b("a1"), rows * mid, ACT_RELU)
        self.l2.fwd(L, t, [(b("a1"), mid, mid)], b("a2"), rows)
        L.op("act_fwd", f"{t} relu a2", b("a2"), rows * mid, ACT_RELU)
        self.l3.fwd(L, t, [(b("a2"), mid, mid)], b("a3"), rows)
        L.op("act_fwd", f"{t} relu a3", b("a3"), rows * nout, ACT_RELU)
        L.op("permute4", f"{t} residual copy", b("sc"), b("s"), (rows * nout, 1, 1, 1), (1, 0, 0, 0), False)
        L.op("permute4", f"{t} residual sum", b("a3"), b("s"), (rows * nout, 1, 1, 1), (1, 0, 0, 0), True)
        L.op("layernorm_fwd", f"{t} layernorm", b("s"), b("y"), rows, nout)
        return b("y")

    def bwd_head(self, L, dY, r0, rows, want_wgrad):
        """LayerNorm and the long path down to g1 (:87-108 and :228-248 alike)."""
        nout, mid, b, t = self.nout, self.mid, self.b, self.tag
        L.op("layernorm_bwd", f"{t} layernorm bwd", dY, at(b("s"), r0 * nout), b("ds"), want_wgrad, rows, nout)
        L.op("act_bwd", f"{t} relu' sc", b("ds"), at(b("sc"), r0 * nout), b("gsc"), rows * nout, ACT_RELU)
        L.op("act_bwd", f"{t} relu' a3", b("ds"), at(b("a3"), r0 * nout), b("g3"), rows * nout, ACT_RELU)
        self.l3.bwd(L, t, [(at(b("a2"), r0 * mid), mid, mid)], b("g3"), rows, [(b("g2"), False)], want_wgrad)
        L.op("act_bwd", f"{t} relu' a2", b("g2"), at(b("a2"), r0 * mid), b("g2"), rows * mid, ACT_RELU)
        self.l2.bwd(L, t, [(at(b("a1"), r0 * mid), mid, mid)], b("g2"), rows, [(b("g1"), False)], want_wgrad)
        L.op("act_bwd", f"{t} relu' a1", b("g1"), at(b("a1"), r0 * mid), b("g1"), rows * mid, ACT_RELU)

    def bwd(self, L, in_segs, dY, r0, r1, dsegs, want_wgrad=True):   # :87-112
        rows, b = r1 - r0, self.b
        self.bwd_head(L, dY, r0, rows, want_wgrad)
        segs = [(at(X, r0 * ldx), ks, ldx) for (X, ks, ldx) in in_segs]
        self.sc.bwd(L, self.tag, segs, b("gsc"), rows, [d for d in dsegs], want_wgrad)
        self.l1.bwd(L, self.tag, segs, b("g1"), rows, [(d[0], True) if d is not None else None for d in dsegs], want_wgrad)


def backbone_launches(plan, B, g=128, h=128):
    """Every launch of encode (:142-155), decode (:158-175), losses_fwd (:180-189), decoder_backward (:192-260) for the
    S recon calls (backward_decoder, engine.py:1236) and for the CPC call (S, S+1) without weight or skip gradients
    (backward_prior, engine.py:1355), and encoder_backward (:262-283), in the order one step enqueues them."""
    T, S = plan.T, plan.S
    G = S + 1
    ld = 2 * h + 2
    sk_src = ("plan_int", plan.int_layout["skip_src"][0])
    tgt_idx = ("plan_int", plan.int_layout["tgt_idx"][0])
    L = _List()
    e1, e2 = _Res("encoder", "fc1", "e1", POSE, h), _Res("encoder", "fc2", "e2", h, h)
    e3 = _Lin("encoder", "fc3", g, h)
    d1, d2 = _Res("decoder", "fc1", "d1", g, h), _Res("decoder", "fc2", "d2", 2 * h, h)
    d3 = _Lin("decoder", "fc3", POSE, 2 * h)
    # encode
    N = T * B
    x = ("x", 0)
    h1 = e1.fwd(L, [(x, POSE, POSE)], N)
    h2 = e2.fwd(L, [(h1, h, h)], N)
    e3.fwd(L, "e3", [(h2, h, h)], ("Hlat", 0), N)
    L.op("act_fwd", "latent tanh", ("Hlat", 0), N * g, ACT_TANH)
    # decode
    Nd = G * B
    y1 = d1.fwd(L, [(("h_pred", 0), g, g)], Nd)
    skipsel = ("skipsel", 0)
    L.op("build_concat", "skipsel", skipsel, h1, sk_src, h, h2, sk_src, h, G, B, ld)
    sk0, sk1 = skipsel, at(skipsel, h)
    y2 = d2.fwd(L, [(y1, h, h), (sk1, h, ld)], Nd)
    d3.fwd(L, "d3", [(y2, h, h), (sk0, h, ld)], ("pred", 0), Nd)
    L.op("mse_plain", "pose mse", ("pred", 0), x, tgt_idx, G, B * POSE)

    def decoder_backward(g0, g1, want_wgrad, want_skip):
        r0, r1 = g0 * B, g1 * B
        rows = r1 - r0
        dy = ("d_pred", r0 * POSE)
        dd2, dd1 = ("dd2", 0), ("dd1", 0)
        dsk = ("dskipsel", r0 * ld)
        # d3 over [d2 | skip0] (:213-226)
        L.gemm("d3 dgrad d2", dy, d3.W, dd2, rows, h, POSE, b_mn=True, ldb=2 * h)
        if want_skip:
            L.gemm("d3 dgrad skip0", dy, at(d3.W, h), dsk, rows, h, POSE, b_mn=True, ldb=2 * h, ldc=ld, accumulate=True)
        if want_wgrad:
            L.gemm("d3 wgrad d2", dy, at(y2, r0 * h), d3.gW, POSE, h, rows, a_mn=True, b_mn=True, lda=POSE, ldb=h, ldc=2 * h)
            L.gemm("d3 wgrad skip0", dy, at(skipsel, r0 * ld), at(d3.gW, h), POSE, h, rows, a_mn=True, b_mn=True, lda=POSE, ldb=ld,
                   ldc=2 * h)
            L.op("colsum", "d3 bias grad", dy, rows, POSE, POSE, ("g:decoder.fc3.bias", 0))
        # d2 over [d1 | skip1(pitched)] (:228-260)
        d2.bwd_head(L, dd2, r0, rows, want_wgrad)
        segs = [(at(y1, r0 * h), h, h), (at(skipsel, h + r0 * ld), h, ld)]
        for lin, gg, first in ((d2.sc, d2.b("gsc"), True), (d2.l1, d2.b("g1"), False)):
            L.gemm(f"d2.{lin.name} dgrad d1", gg, lin.W, dd1, rows, h, lin.Nout, b_mn=True, ldb=lin.Kt, accumulate=not first)
            if want_skip:
                L.gemm(f"d2.{lin.name} dgrad skip1", gg, at(lin.W, h), at(dsk, h), rows, h, lin.Nout, b_mn=True, ldb=lin.Kt, ldc=ld,
                       accumulate=True)
            if want_wgrad:
                L.gemm(f"d2.{lin.name} wgrad d1", gg, segs[0][0], lin.gW, lin.Nout, h, rows, a_mn=True, b_mn=True, lda=lin.Nout,
                       ldb=h, ldc=lin.Kt)
                L.gemm(f"d2.{lin.name} wgrad skip1", gg, segs[1][0], at(lin.gW, h), lin.Nout, h, rows, a_mn=True, b_mn=True,
                       lda=lin.Nout, ldb=ld, ldc=lin.Kt)
                L.op("colsum", f"d2.{lin.name} bias grad", gg, rows, lin.Nout, lin.Nout, (f"g:decoder.{lin.name}.bias", 0))
        d1.bwd(L, [(("h_pred", 0), g, g)], ("dd1", 0), r0, r1, [(("d_hpred", r0 * g), False)], want_wgrad)

    decoder_backward(0, S, True, True)
    if plan.has_cpc:
        decoder_backward(S, S + 1, False, False)
    # encoder_backward
    L.op("act_bwd", "latent tanh'", ("dH", 0), ("Hlat", 0), ("enc_dpre", 0), N * g, ACT_TANH)
    e3.bwd(L, "e3", [(h2, h, h)], ("enc_dpre", 0), N, [(("enc_dh2", 0), False)], True)
    L.op("gather_add_cols", "skip1 grads", ("enc_dh1", 0), ("dskipsel", 0), sk_src, S, T, B, h, ld, 0)
    L.op("gather_add_cols", "skip2 grads", ("enc_dh2", 0), ("dskipsel", 0), sk_src, S, T, B, h, ld, h)
    e2.bwd(L, [(h1, h, h)], ("enc_dh2", 0), 0, N, [(("enc_dx1", 0), False)], True)
    L.op("permute4", "dx1 fold", ("enc_dx1", 0), ("enc_dh1", 0), (N * h, 1, 1, 1), (1, 0, 0, 0), True)
    e1.bwd(L, [(x, POSE, POSE)], ("enc_dh1", 0), 0, N, [None], True)
    return L.L


# ------------------------------------------------------------------ launch variants

def gemm_variant(e, kern):
    """What part E counts as one launch variant: the kernel and the operand roles of the call."""
    k = kern if isinstance(kern, str) else kern[0]
    return ("gemm", k, e["a_mn"], e["b_mn"], e["accumulate"], e["bias"], e["ldc"] != e["N"])

