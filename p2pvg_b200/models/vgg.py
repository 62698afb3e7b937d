"""Parameter containers for the VGG-style encoder / decoder pairs (reference models/vgg_64.py:5-105,
models/vgg_128.py:4-120) with the reference's ``state_dict`` layout: ``c<stage>.<idx>.main.<0|1>.*``, a final
``c<n+1>.{0,1}.*`` (4x4 valid conv + BatchNorm), ``upc1.{0,1}.*``, ``upc<stage>.<idx>.main.<0|1>.*`` and the closing
``upc<n+1>.1.*`` ConvTranspose2d(64, nc, 3, 1, 1).

The stages are generated from the channel tables of p2pvg_b200/engine_vgg.py in the reference's construction order, so
the torch RNG stream (and with it ``init_weights``) is consumed identically.  The layers only *hold* parameters and
BatchNorm buffers: arithmetic runs in the sm_90a kernels (engine_vgg.py for training, infer_vgg.py for stand-alone calls).
"""
import torch.nn as nn

from ..engine_vgg import vgg_tables


class vgg_layer(nn.Module):
    def __init__(self, nin, nout):
        super().__init__()
        self.main = nn.Sequential(nn.Conv2d(nin, nout, 3, 1, 1), nn.BatchNorm2d(nout), nn.LeakyReLU(0.2, inplace=True))


def _stage(pairs, nc):
    return nn.Sequential(*[vgg_layer(nc if a is None else a, b) for a, b in pairs])


class VggEncoder(nn.Module):
    backbone = "vgg"
    image_width = 64

    def __init__(self, dim, nc=1):
        super().__init__()
        self.dim, self.nc = dim, nc
        table = vgg_tables(self.image_width)[0]
        self.nstage = len(table)
        for i, pairs in enumerate(table, 1):
            setattr(self, f"c{i}", _stage(pairs, nc))
        setattr(self, f"c{self.nstage + 1}", nn.Sequential(nn.Conv2d(512, dim, 4, 1, 0), nn.BatchNorm2d(dim), nn.Tanh()))
        self.mp = nn.MaxPool2d(kernel_size=2, stride=2, padding=0)

    def forward(self, input):
        from ..infer_vgg import vgg_encoder_forward
        return vgg_encoder_forward(self, input)


class VggDecoder(nn.Module):
    backbone = "vgg"
    image_width = 64

    def __init__(self, dim, nc=1):
        super().__init__()
        self.dim, self.nc = dim, nc
        table = vgg_tables(self.image_width)[1]
        self.nstage = len(table)
        self.upc1 = nn.Sequential(nn.ConvTranspose2d(dim, 512, 4, 1, 0), nn.BatchNorm2d(512), nn.LeakyReLU(0.2, inplace=True))
        for i, pairs in enumerate(table[:-1], 2):
            setattr(self, f"upc{i}", _stage(pairs, nc))
        cin, cout = table[-1][0]
        setattr(self, f"upc{self.nstage + 1}", nn.Sequential(vgg_layer(cin, cout), nn.ConvTranspose2d(cout, nc, 3, 1, 1), nn.Sigmoid()))
        self.up = nn.UpsamplingNearest2d(scale_factor=2)

    def forward(self, input):
        from ..infer_vgg import vgg_decoder_forward
        vec, skip = input
        return vgg_decoder_forward(self, vec, skip)
