"""Train-step schedule for the human3.6m pose backbone (reference models/h36m_mlp.py): residual-MLP encoder /
decoder around the same recurrent phase, losses, two-phase update and optimiser as p2pvg_b200/engine.py.

There is no BatchNorm, so every encoder / decoder call is row-wise independent: all T frames (and all S+1 decoder
calls) are plain row batches.  ``torch.cat([d, skip], 1)`` before a Linear is never materialised: the Linear is
evaluated as two GEMMs over the two column blocks of its weight.  All tensors are fp32; in the tensor-core mode the
K-major GEMMs with TMA-compatible operands run as wgmma .tf32 (p2pvg_gemm), the rest on the CUDA cores.
"""
from __future__ import annotations

import torch

from .engine import ACT_TANH, TrainEngine

ACT_RELU = 4


class Linear:
    """y = [x_0 | x_1 | ...] . W^T + b over column segments of W (no concat buffer)."""

    def __init__(self, eng, module, name):
        self.eng, self.m, self.name = eng, module, name

    @property
    def W(self):
        return self.eng.arena[self.m].p[self.name + ".weight"]

    def fwd(self, segs, out, rows):
        K, W = self.eng.K, self.W
        N, Kt = W.shape
        b = self.eng.arena[self.m].p[self.name + ".bias"]
        koff = 0
        for i, (X, ks, ldx) in enumerate(segs):
            K.gemm(X, W.view(-1)[koff:], out, rows, N, ks, lda=ldx, ldb=Kt, accumulate=(i > 0), bias=b if i == 0 else None)
            koff += ks
        self.segs = segs

    def bwd(self, dY, rows, dsegs, want_wgrad=True):
        """dsegs[i] = (tensor or None, accumulate): gradient w.r.t. input segment i."""
        K, W = self.eng.K, self.W
        A = self.eng.arena[self.m]
        N, Kt = W.shape
        koff = 0
        for (X, ks, ldx), d in zip(self.segs, dsegs):
            if d is not None:
                dX, acc = d
                K.gemm(dY, W.view(-1)[koff:], dX, rows, ks, N, b_mn=True, ldb=Kt, accumulate=acc)
            if want_wgrad:
                K.gemm(dY, X, A.g[self.name + ".weight"].view(-1)[koff:], N, ks, rows, a_mn=True, b_mn=True, lda=N, ldb=ldx, ldc=Kt)
            koff += ks
        if want_wgrad:
            K.colsum(dY, rows, N, N, A.g[self.name + ".bias"])


class ResidualLinear:
    """models/h36m_mlp.py:28-46: LayerNorm(relu(L_s x) + relu(L_3 relu(L_2 relu(L_1 x))))."""

    def __init__(self, eng, module, prefix, tag):
        self.eng, self.m, self.pre, self.tag = eng, module, prefix, tag
        self.sc = Linear(eng, module, prefix + ".shortcut.0")
        self.l1 = Linear(eng, module, prefix + ".long_path.0")
        self.l2 = Linear(eng, module, prefix + ".long_path.2")
        self.l3 = Linear(eng, module, prefix + ".long_path.4")

    def fwd(self, segs, rows):
        e, K = self.eng, self.eng.K
        nout, mid = self.sc.W.shape[0], self.l1.W.shape[0]
        b = lambda nm, n: e.fbuf(f"{self.tag}_{nm}", rows * n)
        self.a_sc, self.a1, self.a2, self.a3 = b("sc", nout), b("a1", mid), b("a2", mid), b("a3", nout)
        self.s, self.y = b("s", nout), b("y", nout)
        self.mean, self.rstd = b("mean", 1), b("rstd", 1)
        self.sc.fwd(segs, self.a_sc, rows)
        K.act_fwd(self.a_sc, rows * nout, ACT_RELU)
        self.l1.fwd(segs, self.a1, rows)
        K.act_fwd(self.a1, rows * mid, ACT_RELU)
        self.l2.fwd([(self.a1, mid, mid)], self.a2, rows)
        K.act_fwd(self.a2, rows * mid, ACT_RELU)
        self.l3.fwd([(self.a2, mid, mid)], self.a3, rows)
        K.act_fwd(self.a3, rows * nout, ACT_RELU)
        K.permute4(self.a_sc, self.s, (rows * nout, 1, 1, 1), (1, 0, 0, 0))
        K.permute4(self.a3, self.s, (rows * nout, 1, 1, 1), (1, 0, 0, 0), accumulate=True)
        P = e.arena[self.m].p
        K.layernorm_fwd(self.s, P[self.pre + ".norm.weight"], P[self.pre + ".norm.bias"], self.y, self.mean, self.rstd, rows, nout)
        self.rows, self.nout, self.mid = rows, nout, mid
        return self.y

    def bwd(self, dY, r0, r1, dsegs, want_wgrad=True):
        """Backward for rows [r0, r1) of the forward batch.  dY: [r1-r0, nout] (overwritten)."""
        e, K = self.eng, self.eng.K
        A = e.arena[self.m]
        rows, nout, mid = r1 - r0, self.nout, self.mid
        sl = lambda t, n: t[r0 * n:r1 * n]
        ds = e.fbuf(f"{self.tag}_ds", self.rows * nout)[:rows * nout]
        K.layernorm_bwd(dY, sl(self.s, nout), self.mean[r0:r1], self.rstd[r0:r1], A.p[self.pre + ".norm.weight"], ds,
                        A.g[self.pre + ".norm.weight"] if want_wgrad else None, A.g[self.pre + ".norm.bias"] if want_wgrad else None,
                        rows, nout)
        g_sc = e.fbuf(f"{self.tag}_gsc", self.rows * nout)[:rows * nout]
        g3 = e.fbuf(f"{self.tag}_g3", self.rows * nout)[:rows * nout]
        K.act_bwd(ds, sl(self.a_sc, nout), g_sc, rows * nout, ACT_RELU)
        K.act_bwd(ds, sl(self.a3, nout), g3, rows * nout, ACT_RELU)
        g2 = e.fbuf(f"{self.tag}_g2", self.rows * mid)[:rows * mid]
        g1 = e.fbuf(f"{self.tag}_g1", self.rows * mid)[:rows * mid]
        self._slice_segs(self.l3, [(self.a2, mid, mid)], r0)
        self.l3.bwd(g3, rows, [(g2, False)], want_wgrad)
        K.act_bwd(g2, sl(self.a2, mid), g2, rows * mid, ACT_RELU)
        self._slice_segs(self.l2, [(self.a1, mid, mid)], r0)
        self.l2.bwd(g2, rows, [(g1, False)], want_wgrad)
        K.act_bwd(g1, sl(self.a1, mid), g1, rows * mid, ACT_RELU)
        # the shortcut and the first long-path Linear read the same input segments
        self.sc.segs = self.l1.segs = self.in_segs_for(r0)
        self.sc.bwd(g_sc, rows, [(d[0], d[1]) if d is not None else None for d in dsegs], want_wgrad)
        self.l1.bwd(g1, rows, [(d[0], True) if d is not None else None for d in dsegs], want_wgrad)

    def set_inputs(self, segs):
        self._in = segs

    def in_segs_for(self, r0):
        return [(X[r0 * ldx:], ks, ldx) for (X, ks, ldx) in self._in]

    @staticmethod
    def _slice_segs(lin, segs, r0):
        lin.segs = [(X[r0 * ldx:], ks, ldx) for (X, ks, ldx) in segs]


class TrainEngineMLP(TrainEngine):
    def __init__(self, state, cfg, opt, kernels, act_dtype=torch.float32, mode="A"):
        cfg = dict(cfg, backbone="mlp")
        super().__init__(state, cfg, opt, kernels, act_dtype=act_dtype, mode=mode)
        self.implicit = False
        self.h = self.arena["encoder"].p["fc3.weight"].shape[1]  # h_dim
        self.e1 = ResidualLinear(self, "encoder", "fc1", "e1")
        self.e2 = ResidualLinear(self, "encoder", "fc2", "e2")
        self.e3 = Linear(self, "encoder", "fc3")
        self.d1 = ResidualLinear(self, "decoder", "fc1", "d1")
        self.d2 = ResidualLinear(self, "decoder", "fc2", "d2")
        self.d3 = Linear(self, "decoder", "fc3")

    def pack_weights(self, which=("encoder", "decoder"), backward=True):
        pass  # fp32 master weights are used directly

    # -- Phase E ----------------------------------------------------------------------------
    def encode(self, x, plan):
        K, T, B, g, h = self.K, self.T, self.B, self.g, self.h
        N = T * B
        self.x_nhwc = x.contiguous().view(-1)  # [T*B, 51] fp32: also the MSE target
        segs = [(self.x_nhwc, 51, 51)]
        self.e1.set_inputs(segs)
        h1 = self.e1.fwd(segs, N)
        segs2 = [(h1, h, h)]
        self.e2.set_inputs(segs2)
        h2 = self.e2.fwd(segs2, N)
        self.Hlat = self.fbuf("Hlat", N * g)
        self.e3.fwd([(h2, h, h)], self.Hlat, N)
        K.act_fwd(self.Hlat, N * g, ACT_TANH)
        self.h1, self.h2 = h1, h2

    # -- Phase D ----------------------------------------------------------------------------
    def decode(self, plan):
        K, B, S, g, h = self.K, self.B, self.S, self.g, self.h
        G = S + 1
        N = G * B
        segs = [(self.h_pred, g, g)]
        self.d1.set_inputs(segs)
        d1 = self.d1.fwd(segs, N)
        # skip tensors of the source frame of every call (models/p2p_model.py:235-238): gathered rows, pitch h+2
        ix = self.ix
        ld = h + h + 2
        self.skipsel = self.fbuf("skipsel", N * ld)
        K.build_concat(self.skipsel, self.h1, ix["skip_src"], h, self.h2, ix["skip_src"], h, self.tuc, self.dt, G, B, ld=ld)
        sk0, sk1 = self.skipsel, self.skipsel[h:]          # columns [0,h) = h1 (skip[0]), [h,2h) = h2 (skip[1])
        segs2 = [(d1, h, h), (sk1, h, ld)]
        self.d2.set_inputs(segs2)
        d2 = self.d2.fwd(segs2, N)
        self.pred = self.fbuf("pred", N * 51)
        self.d3.fwd([(d2, h, h), (sk0, h, ld)], self.pred, N)

    def decoded(self):
        return self.pred, False   # fc3 output: the pose itself (no output nonlinearity)

    def losses_fwd(self, plan):
        K, B, S = self.K, self.B, self.S
        G = S + 1
        E = B * 51
        self.d_pred = self.fbuf("d_pred", G * E)
        self.mse_partial = self.fbuf("mse_partial", G * K.mse_chunks())
        K.mse_plain(self.pred, self.x_nhwc, self.ix["tgt_idx"], self.coef, G, E, self.d_pred, self.mse_partial)
        self.align_partial = self.fbuf("align_partial", max(S, 1))
        self.d_hpred = self.fbuf("d_hpred", G * B * self.g)
        self.dH = self.fbuf("dH", self.T * B * self.g)

    # -- backward ---------------------------------------------------------------------------
    def decoder_backward(self, g0, g1, want_wgrad, want_skip):
        K, B, g, h = self.K, self.B, self.g, self.h
        r0, r1 = g0 * B, g1 * B
        rows = r1 - r0
        ld = 2 * h + 2
        dy = self.d_pred[r0 * 51:r1 * 51]
        dd2 = self.fbuf("dd2", (self.S + 1) * B * h)[:rows * h]
        dskip = self.fbuf("dskipsel", (self.S + 1) * B * ld)
        dsk = dskip[r0 * ld:]
        if want_skip:
            dskip[r0 * ld:r1 * ld].zero_()
        self.d3.segs = [(self.d2.y[r0 * h:], h, h), (self.skipsel[r0 * ld:], h, ld)]
        self._lin_bwd_pitched(self.d3, dy, rows, dd2, dsk if want_skip else None, 0, ld, want_wgrad)
        dd1 = self.fbuf("dd1", (self.S + 1) * B * h)[:rows * h]
        self.d2._in = [(self.d1.y, h, h), (self.skipsel[h:], h, ld)]
        self._rl_bwd_pitched(self.d2, dd2, r0, r1, dd1, dsk[h:] if want_skip else None, ld, want_wgrad)
        dhp = self.d_hpred[r0 * g:r1 * g]
        self.d1._in = [(self.h_pred, g, g)]
        self.d1.bwd(dd1, r0, r1, [(dhp, False)], want_wgrad)
        self.dskipsel = dskip

    def _lin_bwd_pitched(self, lin, dY, rows, d0, dsk, col0, ld, want_wgrad):
        """Linear over [x0 | skip]: d x0 dense, d skip written into the pitched skip-gradient matrix."""
        K, W = self.K, lin.W
        A = self.arena[lin.m]
        N, Kt = W.shape
        h = self.h
        K.gemm(dY, W, d0, rows, h, N, b_mn=True, ldb=Kt)
        if dsk is not None:
            K.gemm(dY, W.view(-1)[h:], dsk[col0:], rows, h, N, b_mn=True, ldb=Kt, ldc=ld, accumulate=True)
        if want_wgrad:
            (X0, k0, l0), (X1, k1, l1) = lin.segs
            K.gemm(dY, X0, A.g[lin.name + ".weight"], N, h, rows, a_mn=True, b_mn=True, lda=N, ldb=l0, ldc=Kt)
            K.gemm(dY, X1, A.g[lin.name + ".weight"].view(-1)[h:], N, h, rows, a_mn=True, b_mn=True, lda=N, ldb=l1, ldc=Kt)
            K.colsum(dY, rows, N, N, A.g[lin.name + ".bias"])

    def _rl_bwd_pitched(self, rl, dY, r0, r1, d0, dsk, ld, want_wgrad):
        """ResidualLinear whose input is [x0 | skip(pitched)]."""
        K = self.K
        A = self.arena[rl.m]
        rows, nout, mid, h = r1 - r0, rl.nout, rl.mid, self.h
        sl = lambda t, n: t[r0 * n:r1 * n]
        ds = self.fbuf(f"{rl.tag}_ds", rl.rows * nout)[:rows * nout]
        K.layernorm_bwd(dY, sl(rl.s, nout), rl.mean[r0:r1], rl.rstd[r0:r1], A.p[rl.pre + ".norm.weight"], ds,
                        A.g[rl.pre + ".norm.weight"] if want_wgrad else None, A.g[rl.pre + ".norm.bias"] if want_wgrad else None, rows, nout)
        g_sc = self.fbuf(f"{rl.tag}_gsc", rl.rows * nout)[:rows * nout]
        g3 = self.fbuf(f"{rl.tag}_g3", rl.rows * nout)[:rows * nout]
        K.act_bwd(ds, sl(rl.a_sc, nout), g_sc, rows * nout, ACT_RELU)
        K.act_bwd(ds, sl(rl.a3, nout), g3, rows * nout, ACT_RELU)
        g2 = self.fbuf(f"{rl.tag}_g2", rl.rows * mid)[:rows * mid]
        g1 = self.fbuf(f"{rl.tag}_g1", rl.rows * mid)[:rows * mid]
        rl.l3.segs = [(rl.a2[r0 * mid:], mid, mid)]
        rl.l3.bwd(g3, rows, [(g2, False)], want_wgrad)
        K.act_bwd(g2, sl(rl.a2, mid), g2, rows * mid, ACT_RELU)
        rl.l2.segs = [(rl.a1[r0 * mid:], mid, mid)]
        rl.l2.bwd(g2, rows, [(g1, False)], want_wgrad)
        K.act_bwd(g1, sl(rl.a1, mid), g1, rows * mid, ACT_RELU)
        segs = [(rl._in[0][0][r0 * rl._in[0][2]:], h, rl._in[0][2]), (rl._in[1][0][r0 * ld:], h, ld)]
        for lin, gg, first in ((rl.sc, g_sc, True), (rl.l1, g1, False)):
            lin.segs = segs
            W = lin.W
            N, Kt = W.shape
            K.gemm(gg, W, d0, rows, h, N, b_mn=True, ldb=Kt, accumulate=not first)
            if dsk is not None:
                K.gemm(gg, W.view(-1)[h:], dsk, rows, h, N, b_mn=True, ldb=Kt, ldc=ld, accumulate=True)
            if want_wgrad:
                K.gemm(gg, segs[0][0], A.g[lin.name + ".weight"], N, h, rows, a_mn=True, b_mn=True, lda=N, ldb=segs[0][2], ldc=Kt)
                K.gemm(gg, segs[1][0], A.g[lin.name + ".weight"].view(-1)[h:], N, h, rows, a_mn=True, b_mn=True, lda=N, ldb=ld, ldc=Kt)
                K.colsum(gg, rows, N, N, A.g[lin.name + ".bias"])

    def encoder_backward(self, plan):
        K, T, B, g, h = self.K, self.T, self.B, self.g, self.h
        N = T * B
        S = self.S
        ld = 2 * h + 2
        # latent path: tanh + fc3
        dpre = self.fbuf("enc_dpre", N * g)
        K.act_bwd(self.dH, self.Hlat, dpre, N * g, ACT_TANH)
        dh2 = self.fbuf("enc_dh2", N * h)
        dh1 = self.fbuf("enc_dh1", N * h)
        self.e3.segs = [(self.h2, h, h)]
        self.e3.bwd(dpre, N, [(dh2, False)], True)
        dh1[:N * h].zero_()
        # skip gradients of the S recon calls, gathered per source frame (deterministic)
        K.gather_add_cols(dh1, self.dskipsel, self.ix["skip_src"], S, T, B, h, ld, 0)
        K.gather_add_cols(dh2, self.dskipsel, self.ix["skip_src"], S, T, B, h, ld, h)
        dx1 = self.fbuf("enc_dx1", N * h)
        self.e2._in = [(self.h1, h, h)]
        self.e2.bwd(dh2, 0, N, [(dx1, False)], True)
        K.permute4(dx1, dh1, (N * h, 1, 1, 1), (1, 0, 0, 0), accumulate=True)
        self.e1._in = [(self.x_nhwc, 51, 51)]
        self.e1.bwd(dh1, 0, N, [None], True)
