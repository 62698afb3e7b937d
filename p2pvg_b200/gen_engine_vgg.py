"""Graph-captured point-to-point generation for the vgg_64 / vgg_128 backbones (reference models/vgg_64.py,
models/vgg_128.py): the backbone hooks of gen_engine.GenerateEngine, whose planner, tables, eps, LSTM state handling,
captured sequence and output assembly are used unchanged (as engine_vgg.py sits beside engine.py for training).

Layer dispatch (bf16 mode), every launch inside the graph:
  * weights: pack_conv3 of every 3x3 layer with >= 64 input channels (the first layer of each decoder stage as its two
    input-channel halves, c0 = 0 for up(d) and c0 = cin for the skip), pack_conv4 of the final 4x4-valid encoder conv,
    pack_convt4 + tile_bias of upc1 and bn_eval_coeffs of every BatchNorm, recomputed from the live parameters on every
    replay (9 * cin is a multiple of 8 for all of them, so no re-pitching scratch is needed);
  * encoder: the first layer is ONE p2pvg_vgg_first_eval launch from the fp32 NCHW frames; every other 3x3 layer ONE
    p2pvg_conv_gemm kind-3 launch with the eval-BatchNorm + LeakyReLU epilogue; maxpool2_fwd between stages; the final
    4x4-valid GEMM, bn_act(tanh) and a cast to the fp32 latent;
  * skip halves: per decoder stage one bias-free kind-3 launch on the skip source's nsrc images (bf16 output), once per
    call, or once per decode with last_frame_skip;
  * decoder: upc1 GEMM + bn_act; per stage upsample2_fwd, the first layer as kind 3 + eval epilogue with the skip half read
    as a grp_src addend (image n adds skip image n % nsrc), the other layers as kind 3 + eval epilogue; then ONE
    p2pvg_vgg_last_eval launch (ConvTranspose2d(64, nc, 3, 1, 1) + Sigmoid) straight into the graph's output slot.
fp32 mode (P2PVG_PRECISION=fp32) lowers the >= 64-channel layers explicitly, as infer_vgg.py does: im2col3 + exact GEMM
+ bn_act, with gather_add for the skip half; the thin ends use the same two kernels in both modes.

Memory: only the skip maps of an encode persist (the decoder reads them); the other layer outputs, the pooled maps, the
decoder's maps, the skip halves and the fp32 mode's column buffers live in a few scratch buffers that grow to their
largest use during the uncaptured warm-up run of a signature.
"""
from __future__ import annotations

import torch

from ._lib import ACT_LRELU
from .engine_vgg import vgg_layers, vgg_tables
from .gen_engine import GenerateEngine, _check_eval
from .layouts import pack_conv3


class VggGenerateEngine(GenerateEngine):
    """p2p_generate_graphed for the vgg_64 / vgg_128 backbones in eval mode."""

    # ------------------------------------------------------------------ checks (before any device work)
    def _check_model(self):
        from .models.vgg import VggDecoder, VggEncoder
        model = self.model
        if getattr(model, "is_pose", False) or not isinstance(model.encoder, VggEncoder) or not isinstance(model.decoder, VggDecoder):
            raise ValueError("p2p_generate_graphed: VggGenerateEngine runs the vgg_64 / vgg_128 backbones only; use p2p_generate")
        _check_eval(model)
        R = int(model.rnn_size)
        if not (64 <= R <= 512 and R % 8 == 0):
            raise ValueError(f"p2p_generate_graphed runs rnn_size 64..512 in multiples of 8 (got {R}); use p2p_generate")
        nc = int(model.encoder.nc)
        if not 1 <= nc <= 4:
            raise ValueError(f"p2p_generate_graphed runs the vgg backbones on 1..4 image channels (got {nc}); use p2p_generate")
        dev = next(model.parameters()).device
        if dev.type != "cuda":
            raise ValueError(f"p2p_generate_graphed needs the model on a CUDA device (its parameters are on {dev}); move the model "
                             "with model.cuda(), or use p2p_generate")

    def _frame_shape(self, f):
        enc = self.model.encoder
        W, nc = enc.image_width, enc.nc
        if f.dim() != 4 or tuple(f.shape[1:]) != (nc, W, W):
            raise ValueError(f"p2p_generate_graphed: frames of shape {tuple(f.shape)} do not fit the {W}-pixel, {nc}-channel vgg "
                             "backbone (expected [B, nc, W, W])")
        return (nc, W, W)

    # ------------------------------------------------------------------ buffers
    def _scratch(self, name, numel):
        """The first numel elements of scratch buffer `name` (activation dtype).  A buffer grows to the largest request of
        the signature's uncaptured warm-up run, so the captured run never allocates."""
        G = self.G
        key = f"scratch_{name}"
        t = G.bufs.get(key)
        if t is None or t.numel() < numel:
            assert not torch.cuda.is_current_stream_capturing(), f"scratch {name} grew during capture"
            t = G.bufs[key] = torch.empty(int(numel), dtype=G.cfg["adt"], device=G.cfg["dev"])
        return t[:numel]

    def _conv3(self, a, wp, y, N, H, cin, cout, bias, bn, addend=None, nsrc=0):
        """y = LeakyReLU(eval-BatchNorm(conv3x3(a) + bias [+ addend image n % nsrc])) for a >= 64-channel layer."""
        K, G = self.K, self.G
        sc, sh = bn
        gz = G.bufs["grp_zero"] if addend is not None else None
        if G.cfg["adt"] == torch.bfloat16:
            K.conv_gemm(3, a, wp, y, N, H, H, cin, cout, bias=bias, addend=addend, grp_src=gz, imgs_per_group=nsrc, eval_scale=sc,
                        eval_shift=sh, act=ACT_LRELU)
            return
        M = N * H * H
        col, raw = self._scratch("col", M * 9 * cin), self._scratch("raw", M * cout)
        K.im2col3(a, col, N, H, H, cin, 9 * cin, 1)
        K.gemm(col, wp, raw, M, cout, 9 * cin, bias=bias)
        if addend is not None:
            K.gather_add(raw, addend, gz, N // nsrc, nsrc * H * H * cout)
        K.bn_act(raw, y, sc, sh, 1, M, cout, ACT_LRELU)

    # ------------------------------------------------------------------ weights
    def _prepare_weights(self):
        K, G, model = self.K, self.G, self.model
        adt = G.cfg["adt"]
        enc, dec = model.encoder, model.decoder
        self.ENC, self.DEC = vgg_tables(enc.image_width)
        enc_layers, dec_layers = vgg_layers(enc.image_width, enc.nc)
        # (stage, index, cin, cout, vgg_layer.main) of every 3x3 layer; cin of a decoder stage's first layer counts both cat halves
        self.enc_layers = [(i, j, cin, cout, enc.get_submodule(pre)) for i, j, cin, cout, pre in enc_layers]
        self.dec_layers = [(k, j, cin, cout, dec.get_submodule(pre)) for k, j, cin, cout, pre in dec_layers]
        self.wp, self.bn = {}, {}

        def pack3(tag, conv, c0, cin, cout):
            wp = self._buf(G, f"wp_{tag}", cout * 9 * cin, adt)
            pack_conv3(K, conv.weight.data, wp, c0, cin)
            self.wp[tag] = wp

        for i, j, cin, cout, m in self.enc_layers:
            if i or j:   # the first layer reads its fp32 weight in place (p2pvg_vgg_first_eval)
                pack3(f"enc{i}_{j}", m[0], 0, cin, cout)
            self._bn_coeffs(f"enc{i}_{j}", m[1])
        self._prepare_latent(getattr(enc, f"c{len(self.ENC) + 1}"), dec.upc1)
        for k, j, cin, cout, m in self.dec_layers:
            if j == 0:   # torch.cat([up(d), skip], 1): the two input-channel halves of the weight
                pack3(f"dec{k}_0D", m[0], 0, cin // 2, cout)
                pack3(f"dec{k}_0S", m[0], cin // 2, cin // 2, cout)
            else:
                pack3(f"dec{k}_{j}", m[0], 0, cin, cout)
            self._bn_coeffs(f"dec{k}_{j}", m[1])

    # ------------------------------------------------------------------ encoder / decoder
    def _encode(self, tag, frames, N, h_out):
        """frames: fp32 NCHW [N, nc, W, W] -> h_out fp32 [N, g]; returns the skip maps (NHWC, one per stage)."""
        K, G, model = self.K, self.G, self.model
        adt = G.cfg["adt"]
        enc = model.encoder
        H = G.cfg["W"]
        skips, a, slot = [], None, None   # slot: the scratch buffer (0 / 1) holding `a`, None for a skip map
        for i, j, cin, cout, m in self.enc_layers:
            if i and not j:
                a, slot = self._pool(a, N, H, cin), 0
                H //= 2
            if j == len(self.ENC[i]) - 1:
                y = self._buf(G, f"{tag}_skip{i}", N * H * H * cout, adt)
            else:
                slot = 0 if slot is None else 1 - slot
                y = self._scratch(slot, N * H * H * cout)
            if i or j:
                self._conv3(a, self.wp[f"enc{i}_{j}"], y, N, H, cin, cout, m[0].bias.data, self.bn[f"enc{i}_{j}"])
            else:
                sc, sh = self.bn["enc0_0"]
                K.vgg_first_eval(frames, enc.nc, m[0].weight.data, m[0].bias.data, sc, sh, y, N, H, H)
            if j == len(self.ENC[i]) - 1:
                skips.append(y)
                slot = None
            a = y
        p = self._pool(a, N, H, 512)
        self._encode_top(tag, p, N, h_out, getattr(enc, f"c{len(self.ENC) + 1}")[0].bias)
        return skips

    def _pool(self, a, N, H, C):
        p = self._scratch(0, N * (H // 2) * (H // 2) * C)
        self.K.maxpool2_fwd(a, p, N, H, H, C)
        return p

    def _skip_halves(self, tag, skips, nsrc):
        """The skip half of the first layer of every decoder stage (bias-free 3x3 convolution of the nsrc skip images with
        the c0 = cin half of its weight).  Returns per stage (tensor, nsrc) for the decodes."""
        K, G = self.K, self.G
        n, out = len(self.DEC), []
        for k, j, cin, cout, _ in self.dec_layers:
            if j:
                continue
            C, H = cin // 2, 8 << k
            sk, wS = skips[n - 1 - k], self.wp[f"dec{k}_0S"]
            addS = self._scratch(f"{tag}_addS{k}", nsrc * H * H * cout)
            if G.cfg["adt"] == torch.bfloat16:
                K.conv_gemm(3, sk, wS, addS, nsrc, H, H, C, cout)
            else:
                col = self._scratch("col", nsrc * H * H * 9 * C)
                K.im2col3(sk, col, nsrc, H, H, C, 9 * C, 1)
                K.gemm(col, wS, addS, nsrc * H * H, cout, 9 * C)
            out.append((addS, nsrc))
        return out

    def _decode(self, h_pred, halves, frame_out, rows):
        """h_pred fp32 [rows, g] -> frame_out fp32 NCHW [rows, nc, W, W] (sigmoid applied), on the first rows rows."""
        K, dec = self.K, self.model.decoder
        d = self._scratch(0, rows * 16 * 512)
        self._decode_head(h_pred, rows, self._scratch("raw", rows * 16 * 512), d)
        slot, H = 0, 4
        for k, j, cin, cout, m in self.dec_layers:
            if j == 0:
                C = cin // 2
                slot = 1 - slot
                u = self._scratch(slot, rows * 4 * H * H * C)
                K.upsample2_fwd(d, u, rows, H, H, C)
                H *= 2
                d, cin, wp = u, C, self.wp[f"dec{k}_0D"]
                addS, nsrc = halves[k]
            else:
                wp, addS, nsrc = self.wp[f"dec{k}_{j}"], None, 0
            slot = 1 - slot
            y = self._scratch(slot, rows * H * H * cout)
            self._conv3(d, wp, y, rows, H, cin, cout, m[0].bias.data, self.bn[f"dec{k}_{j}"], addend=addS, nsrc=nsrc)
            d = y
        last = getattr(dec, f"upc{len(self.DEC) + 1}")[1]
        K.vgg_last_eval(d, last.weight.data, last.bias.data, frame_out, dec.nc, rows, H, H)
