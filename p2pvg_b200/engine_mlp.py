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

    def bwd(self, dY, r0, r1, dsegs, want_wgrad=True):
        """Backward for rows [r0, r1) of the forward batch.  dsegs[i] = None or (tensor, accumulate, ld): the gradient
        w.r.t. input segment i, written (accumulate: added) with row pitch ld."""
        K, W = self.eng.K, self.W
        A = self.eng.arena[self.m]
        N, Kt = W.shape
        rows = r1 - r0
        koff = 0
        for (X, ks, ldx), d in zip(self.segs, dsegs):
            if d is not None:
                dX, acc, ld = d
                K.gemm(dY, W.view(-1)[koff:], dX, rows, ks, N, b_mn=True, ldb=Kt, ldc=ld, accumulate=acc)
            koff += ks
        if not want_wgrad:
            return
        koff = 0
        for X, ks, ldx in self.segs:
            K.gemm(dY, X[r0 * ldx:], A.g[self.name + ".weight"].view(-1)[koff:], N, ks, rows, a_mn=True, b_mn=True, lda=N, ldb=ldx, ldc=Kt)
            koff += ks
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
        """Backward for rows [r0, r1) of the forward batch.  dY: [r1-r0, nout] (overwritten).  dsegs: as for Linear.bwd."""
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
        self.l3.bwd(g3, r0, r1, [(g2, False, mid)], want_wgrad)
        K.act_bwd(g2, sl(self.a2, mid), g2, rows * mid, ACT_RELU)
        self.l2.bwd(g2, r0, r1, [(g1, False, mid)], want_wgrad)
        K.act_bwd(g1, sl(self.a1, mid), g1, rows * mid, ACT_RELU)
        # the shortcut and the first long-path Linear read the same input segments: the second adds to the first's gradient
        self.sc.bwd(g_sc, r0, r1, dsegs, want_wgrad)
        self.l1.bwd(g1, r0, r1, [None if d is None else (d[0], True, d[2]) for d in dsegs], want_wgrad)


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
        h1 = self.e1.fwd([(self.x_nhwc, 51, 51)], N)
        h2 = self.e2.fwd([(h1, h, h)], N)
        self.Hlat = self.fbuf("Hlat", N * g)
        self.e3.fwd([(h2, h, h)], self.Hlat, N)
        K.act_fwd(self.Hlat, N * g, ACT_TANH)
        self.h1, self.h2 = h1, h2

    # -- Phase D ----------------------------------------------------------------------------
    def decode(self, plan):
        K, B, S, g, h = self.K, self.B, self.S, self.g, self.h
        G = S + 1
        N = G * B
        d1 = self.d1.fwd([(self.h_pred, g, g)], N)
        # skip tensors of the source frame of every call (models/p2p_model.py:235-238): gathered rows, pitch h+2
        ix = self.ix
        ld = h + h + 2
        self.skipsel = self.fbuf("skipsel", N * ld)
        K.build_concat(self.skipsel, self.h1, ix["skip_src"], h, self.h2, ix["skip_src"], h, self.tuc, self.dt, G, B, ld=ld)
        sk0, sk1 = self.skipsel, self.skipsel[h:]          # columns [0,h) = h1 (skip[0]), [h,2h) = h2 (skip[1])
        d2 = self.d2.fwd([(d1, h, h), (sk1, h, ld)], N)
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
        self.d3.bwd(dy, r0, r1, [(dd2, False, h), (dsk, True, ld) if want_skip else None], want_wgrad)
        dd1 = self.fbuf("dd1", (self.S + 1) * B * h)[:rows * h]
        self.d2.bwd(dd2, r0, r1, [(dd1, False, h), (dsk[h:], True, ld) if want_skip else None], want_wgrad)
        self.d1.bwd(dd1, r0, r1, [(self.d_hpred[r0 * g:r1 * g], False, g)], want_wgrad)
        self.dskipsel = dskip

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
        self.e3.bwd(dpre, 0, N, [(dh2, False, h)], True)
        dh1[:N * h].zero_()
        # skip gradients of the S recon calls, gathered per source frame (deterministic)
        K.gather_add_cols(dh1, self.dskipsel, self.ix["skip_src"], S, T, B, h, ld, 0)
        K.gather_add_cols(dh2, self.dskipsel, self.ix["skip_src"], S, T, B, h, ld, h)
        dx1 = self.fbuf("enc_dx1", N * h)
        self.e2.bwd(dh2, 0, N, [(dx1, False, h)], True)
        K.permute4(dx1, dh1, (N * h, 1, 1, 1), (1, 0, 0, 0), accumulate=True)
        self.e1.bwd(dh1, 0, N, [None], True)
