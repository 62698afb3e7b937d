"""``KLCriterion`` — same constructor / call signature as the reference's misc/criterion.py:5-15, computed by
the fused sm_90a reparameterise+KL kernel (p2pvg_reparam_kl_fwd)."""
import torch
import torch.nn as nn


class KLCriterion(nn.Module):
    def __init__(self, opt=None):
        super().__init__()
        self.opt = opt

    def forward(self, mu1, logvar1, mu2, logvar2):
        """KL(N(mu1, e^logvar1) || N(mu2, e^logvar2)) summed, divided by the *configured* opt.batch_size."""
        from .._lib import kernels_for
        if not mu1.is_cuda:
            raise RuntimeError("p2pvg_b200 has no CPU path: KLCriterion needs CUDA tensors")
        K = kernels_for(mu1.device)   # the device's one backend (no per-call workspace allocation)
        n = mu1.numel()
        args = [t.detach().contiguous().float() for t in (mu1, logvar1, mu2, logvar2)]
        zeros = torch.zeros(n, device=mu1.device)
        scratch = torch.empty(2 * n, device=mu1.device)
        out = torch.zeros(4, device=mu1.device)
        K.reparam_kl_fwd(args[0], args[1], args[2], args[3], zeros, zeros, scratch[:n], scratch[n:], n, out)
        return out[0] / self.opt.batch_size
