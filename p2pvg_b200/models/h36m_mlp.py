"""``models.h36m_mlp`` drop-in (reference models/h36m_mlp.py:28-95): residual-MLP pose encoder / decoder with the
reference's constructor keywords and ``state_dict`` keys.  The nn layers hold parameters only; arithmetic runs in the
sm_90a kernels (p2pvg_b200/engine_mlp.py for training, p2pvg_b200/infer.py for stand-alone calls)."""
import torch.nn as nn


class residual_linear(nn.Module):
    def __init__(self, nin, nout):
        super().__init__()
        self.shortcut = nn.Sequential(nn.Linear(nin, nout), nn.ReLU(inplace=True))
        half = nin // 2
        self.long_path = nn.Sequential(nn.Linear(nin, half), nn.ReLU(inplace=True), nn.Linear(half, half), nn.ReLU(inplace=True),
                                       nn.Linear(half, nout), nn.ReLU(inplace=True))
        self.norm = nn.LayerNorm(nout)


class encoder(nn.Module):
    def __init__(self, in_dim=17 * 3, out_dim=128, h_dim=128):
        super().__init__()
        self.in_dim, self.out_dim, self.h_dim = in_dim, out_dim, h_dim
        self.fc1 = residual_linear(in_dim, h_dim)
        self.fc2 = residual_linear(h_dim, h_dim)
        self.fc3 = nn.Linear(h_dim, out_dim)
        self.tanh = nn.Tanh()

    def forward(self, input):
        from ..infer import mlp_encoder_forward
        return mlp_encoder_forward(self, input)


class decoder(nn.Module):
    def __init__(self, in_dim=128, out_dim=17 * 3, h_dim=128):
        super().__init__()
        self.in_dim, self.h_dim, self.out_dim = in_dim, h_dim, out_dim
        self.fc1 = residual_linear(in_dim, h_dim)
        self.fc2 = residual_linear(h_dim * 2, h_dim)
        self.fc3 = nn.Linear(h_dim * 2, out_dim)

    def forward(self, input):
        from ..infer import mlp_decoder_forward
        vec, skip = input
        return mlp_decoder_forward(self, vec, skip)
