"""Train-step schedule for the vgg_64 backbone (reference models/vgg_64.py) around the recurrent phase, losses,
two-phase update and optimiser of p2pvg_b200/engine.py.

Layer = Conv2d(3,1,1) + BatchNorm2d + LeakyReLU(0.2) (models/vgg_64.py:8-13); encoder stages are separated by
MaxPool2d(2,2) and end in a 4x4 valid conv + BatchNorm + Tanh (models/vgg_64.py:16-56); the decoder starts with the
1x1 -> 4x4 ConvTranspose of the dcgan decoder, then alternates nearest x2 upsampling, torch.cat([up, skip], 1) and vgg
layers, and ends in ConvTranspose2d(64, nc, 3, 1, 1) + Sigmoid (models/vgg_64.py:59-105).

As in the dcgan schedule the encoder runs once over all T frames and the decoder once over all S+1 calls with
BatchNorm statistics grouped per reference call; torch.cat is never materialised: the first layer of every decoder
stage is evaluated as two convolutions over the two halves of its weight, the skip half once per distinct source frame
(fp32 addend), the upsampled half with the addend folded into the GEMM epilogue.  In bf16 mode every layer with >= 64
channels on both sides is an implicit GEMM (p2pvg_conv_gemm kinds 3-5: 4-D TMA pixel boxes -> wgmma); the 3-channel
ends and the fp32 mode use the explicit im2col3 lowering.
"""
from __future__ import annotations

import torch

from .engine import ACT_LRELU, TrainEngine
from .layouts import implicit_shape, pack_conv3, pack_conv3_t, unpack_conv3, up8

VGG_ENC = [[(None, 64), (64, 64)], [(64, 128), (128, 128)], [(128, 256), (256, 256), (256, 256)], [(256, 512), (512, 512), (512, 512)]]
VGG_DEC = [[(1024, 512), (512, 512), (512, 256)], [(512, 256), (256, 256), (256, 128)], [(256, 128), (128, 64)], [(128, 64)]]
# models/vgg_128.py:16-105: one more 512-channel stage on both sides
VGG_ENC_128 = VGG_ENC + [[(512, 512), (512, 512), (512, 512)]]
VGG_DEC_128 = [[(1024, 512), (512, 512), (512, 512)]] + VGG_DEC


def vgg_tables(width):
    """(encoder, decoder) stage tables of the vgg backbone for width x width frames (vgg_64 or vgg_128)."""
    if width not in (64, 128):
        raise ValueError("vgg backbones exist for 64x64 (vgg_64) and 128x128 (vgg_128) frames")
    return (VGG_ENC_128, VGG_DEC_128) if width == 128 else (VGG_ENC, VGG_DEC)


def vgg_layers(width, nc):
    """The 3x3 layers of the vgg backbone as two lists of (stage, index, cin, cout, state-dict prefix of the vgg_layer's
    ``main``): the encoder's, then the decoder's (cin of a decoder stage's first layer counts both torch.cat halves)."""
    ENC, DEC = vgg_tables(width)
    enc = [(i, j, nc if cin is None else cin, cout, f"c{i + 1}.{j}.main")
           for i, stage in enumerate(ENC) for j, (cin, cout) in enumerate(stage)]
    dec = [(k, j, cin, cout, f"upc{k + 2}.{j}.main") for k, stage in enumerate(DEC) for j, (cin, cout) in enumerate(stage)]
    return enc, dec


class TrainEngineVGG(TrainEngine):
    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.ENC, self.DEC = vgg_tables(self.W0)
        self.enc_layers, self.dec_layers = vgg_layers(self.W0, self.nc)
        self.nst = len(self.ENC)                 # stages; the final 4x4 conv is c{nst+1}, the last decoder block upc{nst+1}
        self.top, self.last = f"c{self.nst + 1}", f"upc{self.nst + 1}"
        self.ldl = up8(9 * self.nc)  # row pitch of the last layer's [pix, 9*nc] matrix

    # ------------------------------------------------------------------ weights
    def _pack_conv3(self, key, w, c0, cin, want_t=True):
        """pack_conv3 and (want_t) pack_conv3_t of input channels [c0, c0+cin); thin inputs are packed via the wp_ scratch."""
        K = self.K
        cout = w.shape[0]
        ld = up8(9 * cin)
        wp = self.buf(f"wp_{key}", cout * 9 * cin + 8)
        out = self.buf(f"wq_{key}", cout * ld) if ld != 9 * cin else wp
        pack_conv3(K, w, out, c0, cin, scratch=wp)
        self._packed[key + ".wp"] = out
        if want_t:
            wt = self.buf(f"wt_{key}", cin * 9 * cout)
            pack_conv3_t(K, w, wt, c0, cin)
            self._packed[key + ".wt"] = wt

    def pack_weights(self, which=("encoder", "decoder"), backward=True):
        """backward=False: without the transposed copies (pack_conv3_t) that only the data gradients read."""
        K = self.K
        if "encoder" in which:
            P = self.arena["encoder"].p
            for i, j, cin, cout, pre in self.enc_layers:
                self._pack_conv3(f"enc.{i}.{j}", P[pre + ".0.weight"], 0, cin, want_t=backward and not (i == 0 and j == 0))
            self.pack_enc_top()
        if "decoder" in which:
            self.pack_dec_head()
            P = self.arena["decoder"].p
            for k, j, cin, cout, pre in self.dec_layers:
                w = P[pre + ".0.weight"]
                if j == 0:
                    C = cin // 2
                    self._pack_conv3(f"dec.{k}.{j}.D", w, 0, C, want_t=backward)
                    self._pack_conv3(f"dec.{k}.{j}.S", w, C, C, want_t=backward)
                else:
                    self._pack_conv3(f"dec.{k}.{j}", w, 0, cin, want_t=backward)
            # ConvTranspose2d(64, nc, 3, 1, 1): Wl[64, (kh,kw,co)] with the row pitch padded to ldl
            wl = self.buf("wp_dec_last", 64 * self.ldl)
            pack_conv3(K, P[self.last + ".1.weight"], wl, scratch=self.buf("wp_dec_last27", 64 * 9 * self.nc + 8))
            self._packed["dec.last"] = wl

    # ------------------------------------------------------------------ 3x3 layer primitives
    def conv3_fwd(self, a, wp, out, N, H, cin, cout, bias=None, addend=None, grp_src=None, ipg=0, stat=None):
        """stat: stat_buf() workspace -> the BatchNorm statistics of `out` come from the GEMM epilogue (implicit path only)."""
        K = self.K
        if self.implicit and implicit_shape(cin, cout):
            K.conv_gemm(3, a, wp, out, N, H, H, cin, cout, bias=bias, addend=addend, grp_src=grp_src, imgs_per_group=ipg,
                        stat_partial=stat["buf"] if stat else None)
            return
        assert stat is None
        ld = up8(9 * cin)
        col = self.buf("vgg_col", N * H * H * ld)
        K.im2col3(a, col, N, H, H, cin, ld, 1)
        K.gemm(col, wp, out, N * H * H, cout, ld, bias=bias)
        if addend is not None:
            K.gather_add(out, addend, grp_src, N // ipg, ipg * H * H * cout)

    def conv3_dgrad(self, dy, wt, out, N, H, cout, cin):
        K = self.K
        if self.implicit and implicit_shape(cout, cin):
            K.conv_gemm(5, dy, wt, out, N, H, H, cout, cin)
            return
        col = self.buf("vgg_dcol", N * H * H * 9 * cout)
        K.im2col3(dy, col, N, H, H, cout, 9 * cout, -1)
        K.gemm(col, wt, out, N * H * H, cin, 9 * cout)

    def conv3_wgrad(self, dy, inp, gw, N, H, cout, cin):
        """gw[cout, (tap, cin)] (row pitch up8(9 cin), fp32)."""
        K = self.K
        if self.implicit and implicit_shape(cin, cout):
            K.conv_gemm(4, dy, inp, gw, N, H, H, 0, cin, Cm=cout)
            return
        ld = up8(9 * cin)
        col = self.buf("vgg_col", N * H * H * ld)
        K.im2col3(inp, col, N, H, H, cin, ld, 1)
        K.gemm(dy, col, gw, cout, ld, N * H * H, a_mn=True, b_mn=True, lda=cout, ldb=ld)

    # ------------------------------------------------------------------ Phase E
    def encode(self, x, plan):
        K, T, B, nc = self.K, self.T, self.B, self.nc
        P = self.arena["encoder"].p
        N = T * B
        a = self.frames_nhwc(x)
        self.venc = [[] for _ in self.ENC]
        H, C = self.W0, nc
        for i, j, cin, cout, pre in self.enc_layers:
            if j == 0 and i > 0:
                pooled = self.buf(f"venc_pool{i}", N * (H // 2) * (H // 2) * C)
                K.maxpool2_fwd(a, pooled, N, H, H, C)
                a, H = pooled, H // 2
            M = N * H * H
            raw = self.buf(f"venc_raw{i}_{j}", M * cout)
            y = self.buf(f"venc_y{i}_{j}", M * cout)
            sp = self.stat_buf(f"venc{i}_{j}", M, 1, cout, B * H * H, kred=9 * cin) if self.implicit and implicit_shape(cin, cout) else None
            self.conv3_fwd(a, self._packed[f"enc.{i}.{j}.wp"], raw, N, H, cin, cout, bias=P[pre + ".0.bias"], stat=sp)
            st = self.bn_forward("venc", f"{i}_{j}", raw, y, T, B * H * H, cout, P[pre + ".1.weight"], P[pre + ".1.bias"], ACT_LRELU, tiles=sp)
            self.venc[i].append(dict(inp=a, raw=raw, y=y, st=st, cin=cin, cout=cout, H=H, pre=pre))
            a, C = y, cout
        pooled = self.buf("venc_pool_top", N * 16 * 512)
        K.maxpool2_fwd(a, pooled, N, 8, 8, 512)
        self.encode_top(pooled)
        self.update_running_stats("encoder", "enc_order", [(rec["pre"] + ".1", rec["st"]) for recs in self.venc for rec in recs]
                                  + [(self.top + ".1", self.enc_final["st"])])

    # ------------------------------------------------------------------ Phase D
    def decode(self, plan):
        K, B, S, nc = self.K, self.B, self.S, self.nc
        G = S + 1
        P = self.arena["decoder"].p
        N = G * B
        d = self.decode_head()
        nskip = plan.nskip
        self.vdec = [[] for _ in self.DEC]
        H, C = 4, 512
        a = d
        for k, j, cin, cout, pre in self.dec_layers:
            M = N * (2 * H if j == 0 else H) ** 2
            if j == 0:
                H *= 2
                u = self.buf(f"vdec_up{k}", N * H * H * C)
                K.upsample2_fwd(a, u, N, H // 2, H // 2, C)
                a = u
            raw = self.buf(f"vdec_raw{k}_{j}", M * cout)
            y = self.buf(f"vdec_y{k}_{j}", M * cout)
            rec = dict(inp=a, raw=raw, y=y, cout=cout, H=H, pre=pre, cat=(j == 0), k=k, j=j)
            if j == 0:
                skip = self.venc[self.nst - 1 - k][-1]["y"]  # frames are a prefix -> the first nskip frames
                imp = self.implicit and implicit_shape(C, cout)
                addS = self.buf(f"vdec_addS{k}", nskip * B * H * H * cout, self.adt if imp else torch.float32)
                self.conv3_fwd(skip, self._packed[f"dec.{k}.0.S.wp"], addS, nskip * B, H, C, cout, bias=P[pre + ".0.bias"])
                sp = self.stat_buf(f"vdec{k}_{j}", M, 1, cout, B * H * H, kred=9 * C) if imp else None
                self.conv3_fwd(a, self._packed[f"dec.{k}.0.D.wp"], raw, N, H, C, cout, addend=addS, grp_src=self.ix["skip_src"], ipg=B, stat=sp)
                rec.update(cin=C, skip=skip)
            else:
                sp = self.stat_buf(f"vdec{k}_{j}", M, 1, cout, B * H * H, kred=9 * cin) if self.implicit and implicit_shape(cin, cout) else None
                self.conv3_fwd(a, self._packed[f"dec.{k}.{j}.wp"], raw, N, H, cin, cout, bias=P[pre + ".0.bias"], stat=sp)
                rec.update(cin=cin)
            rec["st"] = self.bn_forward("vdec", f"{k}_{j}", raw, y, G, B * H * H, cout, P[pre + ".1.weight"], P[pre + ".1.bias"], ACT_LRELU, tiles=sp)
            self.vdec[k].append(rec)
            a, C = y, cout
        # ConvTranspose2d(64, nc, 3, 1, 1): [pix,64] x [64, 9*nc] GEMM, then the 9-tap gather; the Sigmoid lives in the loss kernel
        W0 = self.W0
        M, ldl = N * W0 * W0, self.ldl
        colT = self.buf("vdec_colT", M * ldl)
        K.gemm(a, self._packed["dec.last"], colT, M, ldl, 64, b_mn=True)
        raw_out = self.buf("vdec_rawout", M * nc)
        K.col2im3(colT, raw_out, N, W0, W0, nc, ldl, bias=P[self.last + ".1.bias"])
        self.vlast = dict(inp=a)
        self.dec = [dict(raw=raw_out)]
        self.update_running_stats("decoder", "dec_order", [("upc1.1", self.dec_first["st"])]
                                  + [(rec["pre"] + ".1", rec["st"]) for recs in self.vdec for rec in recs])

    # ------------------------------------------------------------------ backward
    def decoder_backward(self, g0, g1, want_wgrad, want_skip):
        K, B, nc = self.K, self.B, self.nc
        Gn = g1 - g0
        N = Gn * B
        A = self.arena["decoder"]
        nskip = self.last_plan.nskip
        W0 = self.W0
        E = nc * W0 * W0
        dy = self.d_rawout[g0 * B * E:g1 * B * E]
        # last layer
        M, ldl = N * W0 * W0, self.ldl
        wl = self._packed["dec.last"]
        dcolT = self.buf("vgg_col", M * ldl)
        K.im2col3(dy, dcolT, N, W0, W0, nc, ldl, 1)
        x_in = self.vlast["inp"][g0 * B * W0 * W0 * 64:g1 * B * W0 * W0 * 64]
        dd = self.buf("vdec_gd_last", M * 64)
        K.gemm(dcolT, wl, dd, M, 64, ldl)
        if want_wgrad:
            K.colsum(dy, M, nc, nc, A.g[self.last + ".1.bias"])
            gwl = self.fbuf("gwp_dec_last", 64 * ldl)
            K.gemm(x_in, dcolT, gwl, 64, ldl, M, a_mn=True, b_mn=True, lda=64, ldb=ldl)
            unpack_conv3(K, gwl, A.g[self.last + ".1.weight"])
        dy = dd
        for k in range(self.nst - 1, -1, -1):
            for rec in reversed(self.vdec[k]):
                cout, cin, H, pre, j = rec["cout"], rec["cin"], rec["H"], rec["pre"], rec["j"]
                st = rec["st"]
                per = B * H * H
                sl = slice(g0 * per * cout, g1 * per * cout)
                c0, c1 = g0 * cout, g1 * cout
                self.bn_backward(dy, rec["raw"][sl], rec["y"][sl], st, c0, c1, Gn, per, cout, ACT_LRELU)
                if want_wgrad:
                    K.bn_param_grad(st["sdz"][c0:c1], st["sdzx"][c0:c1], Gn, cout, A.g[pre + ".1.weight"], A.g[pre + ".1.bias"])
                    A.g[pre + ".0.bias"].zero_()  # bias feeding a training-mode BatchNorm: gradient is exactly zero
                x_in = rec["inp"][g0 * per * cin:g1 * per * cin]
                if rec["cat"]:
                    C = cin
                    dprev = self.buf(f"vdec_gu{k}", N * H * H * C)
                    self.conv3_dgrad(dy, self._packed[f"dec.{k}.0.D.wt"], dprev, N, H, cout, C)
                    if want_wgrad:
                        gw = self.fbuf(f"gwp_vdec{k}_0", 2 * cout * 9 * C)
                        self.conv3_wgrad(dy, x_in, gw[:cout * 9 * C], N, H, cout, C)
                    if want_skip:
                        dyS = self.buf("scratch_dyS", nskip * per * cout)
                        K.group_sum(dy, dyS, self.ix["skip_src"][g0:g1], Gn, nskip, per * cout)
                        dsk = self.buf(f"vdskip{k}", nskip * per * C)
                        self.conv3_dgrad(dyS, self._packed[f"dec.{k}.0.S.wt"], dsk, nskip * B, H, cout, C)
                        rec["dskip"] = dsk
                        if want_wgrad:
                            self.conv3_wgrad(dyS, rec["skip"], gw[cout * 9 * C:], nskip * B, H, cout, C)
                    elif want_wgrad:
                        gw[cout * 9 * C:].zero_()
                    if want_wgrad:
                        unpack_conv3(K, gw, A.g[pre + ".0.weight"], halves=2)
                    dd = self.buf(f"vdec_gd{k}", N * (H // 2) * (H // 2) * C)
                    K.upsample2_bwd(dprev, dd, N, H // 2, H // 2, C)
                    dy = dd
                else:
                    dprev = self.buf(f"vdec_g{k}_{j}", N * H * H * cin)
                    self.conv3_dgrad(dy, self._packed[f"dec.{k}.{j}.wt"], dprev, N, H, cout, cin)
                    if want_wgrad:
                        gw = self.fbuf(f"gwp_vdec{k}_{j}", cout * 9 * cin)
                        self.conv3_wgrad(dy, x_in, gw, N, H, cout, cin)
                        unpack_conv3(K, gw, A.g[pre + ".0.weight"])
                    dy = dprev
        self.decode_head_backward(dy, g0, g1, want_wgrad)

    def encoder_backward(self, plan):
        K, T, B = self.K, self.T, self.B
        A = self.arena["encoder"]
        N = T * B
        nskip = plan.nskip
        gy = self.buf("venc_gpool4", N * 16 * 512)
        self.encode_top_backward(gy)
        for i in range(self.nst - 1, -1, -1):
            recs = self.venc[i]
            top = recs[-1]
            H, C = top["H"], top["cout"]
            # MaxPool backward into this stage's output, plus the skip gradient from the decoder stage that consumed it
            gyo = self.buf(f"venc_gy{i}", N * H * H * C)
            K.maxpool2_bwd(top["y"], gy, gyo, N, H, H, C)
            dsk = self.vdec[self.nst - 1 - i][0].get("dskip")
            if dsk is not None:
                K.add_indexed(gyo, dsk, self.ix["skip_dst"], nskip, B * H * H * C)
            gy = gyo
            for j in range(len(recs) - 1, -1, -1):
                rec = recs[j]
                cin, cout, pre = rec["cin"], rec["cout"], rec["pre"]
                st = rec["st"]
                self.bn_backward(gy, rec["raw"], rec["y"], st, 0, T * cout, T, B * H * H, cout, ACT_LRELU)
                K.bn_param_grad(st["sdz"], st["sdzx"], T, cout, A.g[pre + ".1.weight"], A.g[pre + ".1.bias"])
                A.g[pre + ".0.bias"].zero_()
                gw = self.fbuf(f"gwp_venc{i}_{j}", cout * up8(9 * cin))
                self.conv3_wgrad(gy, rec["inp"], gw, N, H, cout, cin)
                unpack_conv3(K, gw, A.g[pre + ".0.weight"])
                if i > 0 or j > 0:
                    gprev = self.buf(f"venc_g{i}_{j}", N * H * H * cin)
                    self.conv3_dgrad(gy, self._packed[f"enc.{i}.{j}.wt"], gprev, N, H, cout, cin)
                    gy = gprev
