"""Parameter containers for the DCGAN encoder / decoder with the reference's ``state_dict`` layout
(SURVEY.md A.1; reference models/dcgan_64.py:28-88, models/dcgan_128.py:28-94).

The torch.nn layers below are *holders* of parameters and BatchNorm buffers only: they are created in the
reference's order so that the torch RNG is consumed identically, but their ``forward`` is never used — all
arithmetic goes through the sm_90a kernels (p2pvg_b200/engine.py for the train step, p2pvg_b200/infer.py for
stand-alone calls).
"""
import torch.nn as nn

STAGE_CHANNELS = {64: [64, 128, 256, 512], 128: [64, 128, 256, 512, 512]}


class _Stage(nn.Module):
    """One stride-2 block; exposes ``.main`` = [conv, batchnorm, activation] like the reference blocks."""

    def __init__(self, conv, cout):
        super().__init__()
        self.main = nn.Sequential(conv, nn.BatchNorm2d(cout), nn.LeakyReLU(0.2, inplace=True))


class DcganEncoder(nn.Module):
    image_width = 64

    def __init__(self, dim, nc=1):
        super().__init__()
        self.dim, self.nc = dim, nc
        chans = STAGE_CHANNELS[self.image_width]
        cin = nc
        for i, cout in enumerate(chans, 1):
            setattr(self, f"c{i}", _Stage(nn.Conv2d(cin, cout, 4, 2, 1), cout))
            cin = cout
        setattr(self, f"c{len(chans) + 1}", nn.Sequential(nn.Conv2d(cin, dim, 4, 1, 0), nn.BatchNorm2d(dim), nn.Tanh()))

    def forward(self, input):
        from ..infer import encoder_forward
        return encoder_forward(self, input)


class DcganDecoder(nn.Module):
    image_width = 64

    def __init__(self, dim, nc=1):
        super().__init__()
        self.dim, self.nc = dim, nc
        chans = STAGE_CHANNELS[self.image_width]
        top = chans[-1]
        self.upc1 = nn.Sequential(nn.ConvTranspose2d(dim, top, 4, 1, 0), nn.BatchNorm2d(top), nn.LeakyReLU(0.2, inplace=True))
        cin = top
        outs = chans[-2::-1]
        for k, cout in enumerate(outs, 2):
            setattr(self, f"upc{k}", _Stage(nn.ConvTranspose2d(cin * 2, cout, 4, 2, 1), cout))
            cin = cout
        setattr(self, f"upc{len(outs) + 2}", nn.Sequential(nn.ConvTranspose2d(cin * 2, nc, 4, 2, 1), nn.Sigmoid()))

    def forward(self, input):
        from ..infer import decoder_forward
        vec, skip = input
        return decoder_forward(self, vec, skip)
