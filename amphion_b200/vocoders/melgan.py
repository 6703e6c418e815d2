"""MelGAN generator — drop-in for the reference class
``models/vocoders/gan/generator/melgan.py:50`` (``_vocoders["melgan"]``,
models/vocoders/vocoder_inference.py:39-49): same constructor (``cfg``), the same
``nn.Sequential`` of parameters (``model.1.weight_g``, ``model.4.block.2.bias``, ...),
``hop_length``, ``forward(mel[B,n_mel,T]) -> wav[B,1,T*hop]`` on the native pipeline.
"""
from __future__ import annotations

import numpy as np
from torch import nn
from torch.nn.utils import weight_norm

from .. import _capi
from .generator import NativeGenerator


def weights_init(m):
    # melgan.py:17-23.  With weight norm the drawn `weight` is recomputed from weight_g / weight_v on the next call, so
    # this only advances the RNG; it is kept so that a seeded model matches the reference's parameters exactly.
    classname = m.__class__.__name__
    if classname.find("Conv") != -1:
        m.weight.data.normal_(0.0, 0.02)
    elif classname.find("BatchNorm2d") != -1:
        m.weight.data.normal_(1.0, 0.02)
        m.bias.data.fill_(0)


def WNConv1d(*args, **kwargs):
    return weight_norm(nn.Conv1d(*args, **kwargs))


def WNConvTranspose1d(*args, **kwargs):
    return weight_norm(nn.ConvTranspose1d(*args, **kwargs))


class ResnetBlock(nn.Module):
    """Parameter holder for melgan.py:34-47: ``shortcut(x) + block(x)``; runs inside the generator's pipeline."""

    def __init__(self, dim, dilation=1):
        super().__init__()
        self.block = nn.Sequential(
            nn.LeakyReLU(0.2),
            nn.ReflectionPad1d(dilation),
            WNConv1d(dim, dim, kernel_size=3, dilation=dilation),
            nn.LeakyReLU(0.2),
            WNConv1d(dim, dim, kernel_size=1),
        )
        self.shortcut = WNConv1d(dim, dim, kernel_size=1)

    def forward(self, x):
        raise RuntimeError("amphion_b200: MelGAN's residual blocks execute inside the generator's CUDA pipeline; "
                           "call the generator's forward()")


class _NativeOnly(nn.Sequential):
    def forward(self, x):
        raise RuntimeError("amphion_b200: MelGAN's layers execute inside the generator's CUDA pipeline; "
                           "call the generator's forward()")


class MelGAN(NativeGenerator):
    kind = "melgan"
    hp_key = "melgan"

    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        hp = cfg.model.melgan
        ratios = [int(r) for r in hp.ratios]
        self.hop_length = np.prod(ratios)
        mult = int(2 ** len(ratios))
        ngf = int(hp.ngf)
        model = [
            nn.ReflectionPad1d(3),
            WNConv1d(cfg.preprocess.n_mel, mult * ngf, kernel_size=7, padding=0),
        ]
        for r in ratios:
            model += [
                nn.LeakyReLU(0.2),
                WNConvTranspose1d(mult * ngf, mult * ngf // 2, kernel_size=r * 2, stride=r,
                                  padding=r // 2 + r % 2, output_padding=r % 2),
            ]
            for j in range(int(hp.n_residual_layers)):
                model += [ResnetBlock(mult * ngf // 2, dilation=3 ** j)]
            mult //= 2
        model += [
            nn.LeakyReLU(0.2),
            nn.ReflectionPad1d(3),
            WNConv1d(ngf, 1, kernel_size=7, padding=0),
            nn.Tanh(),
        ]
        self.model = _NativeOnly(*model)
        self.apply(weights_init)

    def _upsample_rates(self):
        return [int(r) for r in self.cfg.model.melgan.ratios]

    def _c_config(self):
        hp = self.cfg.model.melgan
        rates = self._upsample_rates()
        R = int(hp.n_residual_layers)
        if len(rates) > _capi.AB_MAX_STAGES or R > _capi.AB_MAX_DILATIONS or R < 1:
            raise ValueError("amphion_b200: MelGAN needs 1..%d ratios and 1..%d residual layers for the native generator"
                             % (_capi.AB_MAX_STAGES, _capi.AB_MAX_DILATIONS))
        c = _capi.GeneratorConfig()
        c.kind = _capi.GEN_MELGAN
        c.n_mel = int(self.cfg.preprocess.n_mel)
        c.upsample_initial_channel = int(hp.ngf) * 2 ** len(rates)
        c.num_upsamples = len(rates)
        for i, r in enumerate(rates):
            c.upsample_rates[i], c.upsample_kernel_sizes[i] = r, 2 * r
        c.resblock = 1
        c.num_kernels = 1
        c.resblock_kernel_sizes[0] = 3
        c.num_dilations[0] = R
        for j in range(R):
            c.resblock_dilation_sizes[0][j] = 3 ** j
        c.activation = _capi.ACT_LRELU
        return c
