"""Torch emulation of the held-out scoring kernels (p2pvg_bn_eval_coeffs, p2pvg_seq_losses) as a mixin over the emulated
backends of tests/emu_backend.py, tests/emu_vgg.py and tests/emu_mlp.py.  TEST INFRASTRUCTURE ONLY."""
import torch

from tests.emu_backend import EmuKernels, _flat
from tests.emu_mlp import EmuKernelsMLP
from tests.emu_vgg import EmuKernelsVGG
from tests.loss_eval_ref import seq_losses_ref


class SeqLossesEmu:
    def bn_eval_coeffs(self, gamma, beta, rmean, rvar, C, scale, shift, eps=1e-5):
        sc = gamma[:C].float() / torch.sqrt(rvar[:C].float() + eps)
        scale[:C].copy_(sc)
        shift[:C].copy_(beta[:C].float() - rmean[:C].float() * sc)

    def seq_losses(self, rec, sigmoid, x, tgt, S, B, E, mu, lv, mu_p, lv_p, z, H, in_idx, h_pred, g, has_cpc, batch_size, seq_len,
                   partial, counter, per_seq, out):
        per, o = seq_losses_ref(rec, sigmoid, x, tgt, S, B, E, mu, lv, mu_p, lv_p, z, H, in_idx, h_pred, g, has_cpc, batch_size, seq_len)
        _flat(per_seq, 4 * B).copy_(per.reshape(-1))
        _flat(out, 4).copy_(o)


class EmuKernelsEval(SeqLossesEmu, EmuKernels):
    pass


class EmuKernelsVGGEval(SeqLossesEmu, EmuKernelsVGG):
    pass


class EmuKernelsMLPEval(SeqLossesEmu, EmuKernelsMLP):
    pass
