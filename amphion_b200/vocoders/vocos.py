"""Vocos — drop-in for the reference class ``models/codec/amphion_codec/vocos.py:824`` (Vevo's vocoder,
models/vc/vevo/vevo_utils.py:117-121, and the codec decoders, models/codec/amphion_codec/codec.py:373): same
constructor (keyword defaults, ``cfg`` fields override them), the same parameter tree (``backbone.embed``,
``backbone.convnext.{i}.{dwconv,norm,pwconv1,pwconv2,gamma}``, ``backbone.final_layer_norm``, ``head.out``,
``head.istft.window``) drawn in the same order, ``hop_length``, and ``forward(x [B, input_channels, L]) -> [B, 1, L*hop]``
on the native pipeline (``AB_GEN_VOCOS``): the ConvNeXt pointwise layers and the head run on the pointwise wgmma GEMM,
the iSTFT on cuFFT C2R + overlap-add.  The non-conditional backbone with "same" padding is served; AdaLayerNorm
(``adanorm_num_embeddings``) and ``padding="center"`` are refused at construction."""
from __future__ import annotations

import torch
from torch import nn

from .. import _capi
from .generator import NativeGenerator


def _native_only(name):
    raise RuntimeError(f"amphion_b200: Vocos' {name} executes inside the generator's CUDA pipeline; "
                       "call Vocos.forward()")


class ConvNeXtBlock(nn.Module):
    """Parameter holder for vocos.py:469-527 (non-conditional LayerNorm)."""

    def __init__(self, dim: int, intermediate_dim: int, layer_scale_init_value: float):
        super().__init__()
        self.dwconv = nn.Conv1d(dim, dim, kernel_size=7, padding=3, groups=dim)
        self.norm = nn.LayerNorm(dim, eps=1e-6)
        self.pwconv1 = nn.Linear(dim, intermediate_dim)
        self.act = nn.GELU()
        self.pwconv2 = nn.Linear(intermediate_dim, dim)
        self.gamma = (nn.Parameter(layer_scale_init_value * torch.ones(dim), requires_grad=True)
                      if layer_scale_init_value > 0 else None)

    def forward(self, *args, **kwargs):
        _native_only("ConvNeXt blocks")


class VocosBackbone(nn.Module):
    """Parameter holder for vocos.py:720-783; ``_init_weights`` redraws every Conv1d / Linear as the reference does."""

    def __init__(self, input_channels: int, dim: int, intermediate_dim: int, num_layers: int,
                 layer_scale_init_value=None):
        super().__init__()
        self.input_channels = input_channels
        self.embed = nn.Conv1d(input_channels, dim, kernel_size=7, padding=3)
        self.norm = nn.LayerNorm(dim, eps=1e-6)
        layer_scale_init_value = layer_scale_init_value or 1 / num_layers
        self.convnext = nn.ModuleList([ConvNeXtBlock(dim, intermediate_dim, layer_scale_init_value)
                                       for _ in range(num_layers)])
        self.final_layer_norm = nn.LayerNorm(dim, eps=1e-6)
        self.apply(self._init_weights)

    def _init_weights(self, m):
        if isinstance(m, (nn.Conv1d, nn.Linear)):
            nn.init.trunc_normal_(m.weight, std=0.02)
            nn.init.constant_(m.bias, 0)

    def forward(self, *args, **kwargs):
        _native_only("backbone")


class _ISTFTWindow(nn.Module):
    """The reference ISTFT's state (vocos.py:99-112): its Hann window is a persistent buffer, ``head.istft.window``."""

    def __init__(self, n_fft: int, hop_length: int, win_length: int, padding: str):
        super().__init__()
        self.padding, self.n_fft, self.hop_length, self.win_length = padding, n_fft, hop_length, win_length
        self.register_buffer("window", torch.hann_window(win_length))

    def forward(self, *args, **kwargs):
        _native_only("ISTFT")


class ISTFTHead(nn.Module):
    """Parameter holder for vocos.py:314-361: ``out = Linear(dim, n_fft + 2)`` and the ISTFT."""

    def __init__(self, dim: int, n_fft: int, hop_length: int, padding: str = "same"):
        super().__init__()
        self.out = nn.Linear(dim, n_fft + 2)
        self.istft = _ISTFTWindow(n_fft, hop_length, n_fft, padding)

    def forward(self, *args, **kwargs):
        _native_only("ISTFT head")


class Vocos(NativeGenerator):
    kind = "vocos"

    def __init__(self, input_channels: int = 256, dim: int = 384, intermediate_dim: int = 1152, num_layers: int = 8,
                 n_fft: int = 800, hop_size: int = 200, padding: str = "same", adanorm_num_embeddings=None, cfg=None):
        super().__init__()

        def pick(name, default):
            return getattr(cfg, name) if cfg is not None and hasattr(cfg, name) else default

        input_channels = pick("input_channels", input_channels)
        dim = pick("dim", dim)
        intermediate_dim = pick("intermediate_dim", intermediate_dim)
        num_layers = pick("num_layers", num_layers)
        adanorm_num_embeddings = pick("adanorm_num_embeddings", adanorm_num_embeddings)
        n_fft = pick("n_fft", n_fft)
        hop_size = pick("hop_size", hop_size)
        padding = pick("padding", padding)
        if adanorm_num_embeddings is not None:
            # Vocos.forward passes no bandwidth_id, so the reference's AdaLayerNorm backbone asserts in forward
            raise ValueError("amphion_b200: Vocos with adanorm_num_embeddings (AdaLayerNorm) is not served: "
                             "Vocos.forward cannot pass the bandwidth_id it needs")
        if padding not in ["center", "same"]:
            raise ValueError("Padding must be 'center' or 'same'.")
        if padding != "same":
            raise NotImplementedError("amphion_b200: Vocos' ISTFT runs the 'same' padding mode")
        self.cfg = cfg
        self.input_channels, self.dim, self.intermediate_dim = int(input_channels), int(dim), int(intermediate_dim)
        self.num_layers, self.n_fft = int(num_layers), int(n_fft)
        self.hop_length = int(hop_size)
        self.backbone = VocosBackbone(self.input_channels, self.dim, self.intermediate_dim, self.num_layers)
        self.head = ISTFTHead(self.dim, self.n_fft, self.hop_length, padding)

    def _input_channels(self):
        return self.input_channels

    def _hop(self):
        return self.hop_length

    def _c_config(self):
        c = _capi.GeneratorConfig()
        c.kind = _capi.GEN_VOCOS
        c.n_mel = self.input_channels
        c.upsample_initial_channel = self.dim
        c.ffn_channels = self.intermediate_dim
        c.num_layers = self.num_layers
        c.istft_n_fft = self.n_fft
        c.istft_hop = self.hop_length
        return c
