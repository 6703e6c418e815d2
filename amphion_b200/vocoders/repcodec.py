"""RepCodec — drop-in for the semantic codec of MaskGCT, Metis and Vevo (``models/codec/kmeans/repcodec_model.py:34-196``):
the same constructor (keyword defaults, ``cfg`` fields override them, with the reference's rule that
``vocos_intermediate_dim`` and ``vocos_num_layers`` are read from ``cfg`` only when it has ``vocos_dim``) and the same
parameter tree, drawn in the same order, so the released ``semantic_codec/model.safetensors`` loads strictly.  Served
natively in eval:

- ``encoder`` / ``decoder``: ``nn.Sequential(VocosBackbone, nn.Linear(dim, hidden))`` on ``AB_GEN_VOCOS_LINEAR``,
  ``[B, hidden, T]`` (any strides) -> ``[B, T, hidden]`` fp32, children ``"0"`` and ``"1"`` as in the reference;
- ``quantizer``: the native ``ResidualVQ`` (``quantizer_type="fvq"``, ``use_l2_normlize=True``), fp32 at every
  precision;
- ``quantize(x [B, T, hidden]) -> (codes, quantized)`` and ``forward(x) -> (x_rec, codebook_loss, all_indices)``.

``down`` / ``up`` exist when ``downsample_scale > 1`` and are never run: the reference's downsampling code is commented
out.  Training mode (quantizer dropout, the commitment and codebook losses) is refused."""
from __future__ import annotations

import torch
from torch import nn

from .. import _capi
from .amphion_codec import ResidualVQ
from .facodec import _refuse_training
from .generator import NativeGenerator
from .vocos import VocosBackbone

_SERVED = "amphion_b200 serves RepCodec.quantize() / .forward() in eval, and its encoder / decoder on their own"


def init_weights(m):
    """repcodec_model.py:18-24: every Conv1d and Linear gets trunc_normal(std 0.02) weights and zero biases."""
    if isinstance(m, (nn.Conv1d, nn.Linear)):
        nn.init.trunc_normal_(m.weight, std=0.02)
        nn.init.constant_(m.bias, 0)


class VocosLinear(NativeGenerator):
    """``nn.Sequential(VocosBackbone(input_channels, dim, intermediate_dim, num_layers), nn.Linear(dim, out_features))``
    (repcodec_model.py:108-127) on the native pipeline (``AB_GEN_VOCOS_LINEAR``).  ``forward(x [B, input_channels, T])``
    (any strides, any float dtype) -> ``[B, T, out_features]`` fp32 contiguous, the layout ``nn.Linear`` returns."""

    kind = "vocos_linear"

    def __init__(self, input_channels: int, dim: int, intermediate_dim: int, num_layers: int, out_features: int):
        super().__init__()
        self.input_channels, self.dim, self.intermediate_dim = int(input_channels), int(dim), int(intermediate_dim)
        self.num_layers, self.out_features = int(num_layers), int(out_features)
        self.add_module("0", VocosBackbone(self.input_channels, self.dim, self.intermediate_dim, self.num_layers))
        self.add_module("1", nn.Linear(self.dim, self.out_features))

    def __getitem__(self, i):
        return self._modules[str(i)]

    def __len__(self):
        return 2

    def _input_channels(self):
        return self.input_channels

    def _hop(self):
        return 1

    def _c_config(self):
        c = _capi.GeneratorConfig()
        c.kind = _capi.GEN_VOCOS_LINEAR
        c.n_mel = self.input_channels
        c.upsample_initial_channel = self.dim
        c.ffn_channels = self.intermediate_dim
        c.num_layers = self.num_layers
        c.trunk_out_channels = self.out_features
        return c

    def forward(self, x, out=None):
        """``out`` (beyond the reference signature): a contiguous fp32 [B, T, out_features] tensor to write into."""
        if not isinstance(x, torch.Tensor) or x.dim() != 3 or x.shape[1] != self.input_channels:
            got = tuple(x.shape) if isinstance(x, torch.Tensor) else type(x).__name__
            raise ValueError(f"expected input of shape [B, {self.input_channels}, T], got {got}")
        if not x.is_floating_point():
            raise ValueError(f"amphion_b200: expected a floating-point input, got {x.dtype}")
        B, _, T = x.shape
        if B == 0 or T == 0:
            raise ValueError("amphion_b200: empty input batch")
        _capi.require_cuda(x, f"{type(self).__name__}.forward")
        if x.dtype != torch.float32:
            x = x.float()
        with self._launch(x.device) as h:
            need = _capi.lib.ab_generator_workspace_bytes(h, B, T)
            ws = self._scratch(need, x.device)
            y = self._output(out, (B, T, self.out_features), x.device)
            _capi.check(_capi.lib.ab_generator_forward(h, _capi.ptr(x), B, T, _capi.shape_array(x.stride()), _capi.ptr(y),
                                                       ws, need, _capi.stream_ptr()), "ab_generator_forward")
        return y


class RepCodec(nn.Module):
    """Drop-in for RepCodec (repcodec_model.py:34-196).  ``precision`` sets the encoder's and decoder's ("fp32",
    "tc_f16", "tc_bf16"); the quantizer runs in fp32 at every precision.  ``last_launches``: the kernel launches of the
    last ``quantize`` / ``forward`` (``quantize``: embed, LayerNorm, 3 per ConvNeXt block, final LayerNorm, Linear and
    the RVQ; 41 at 12 layers)."""

    def __init__(self, codebook_size=8192, hidden_size=1024, codebook_dim=8, vocos_dim=384, vocos_intermediate_dim=2048,
                 vocos_num_layers=12, num_quantizers=1, downsample_scale=1, cfg=None):
        super().__init__()

        def pick(name, default, key=None):
            return getattr(cfg, name) if cfg is not None and hasattr(cfg, key or name) else default

        codebook_size = pick("codebook_size", codebook_size)
        codebook_dim = pick("codebook_dim", codebook_dim)
        hidden_size = pick("hidden_size", hidden_size)
        vocos_dim = pick("vocos_dim", vocos_dim)
        # repcodec_model.py:67-76: both are read from cfg only when it has vocos_dim
        vocos_intermediate_dim = pick("vocos_intermediate_dim", vocos_intermediate_dim, "vocos_dim")
        vocos_num_layers = pick("vocos_num_layers", vocos_num_layers, "vocos_dim")
        num_quantizers = pick("num_quantizers", num_quantizers)
        downsample_scale = pick("downsample_scale", downsample_scale)

        self.codebook_size = codebook_size
        self.codebook_dim = codebook_dim
        self.hidden_size = hidden_size
        self.vocos_dim = vocos_dim
        self.vocos_intermediate_dim = vocos_intermediate_dim
        self.vocos_num_layers = vocos_num_layers
        self.num_quantizers = num_quantizers
        self.downsample_scale = downsample_scale

        if self.downsample_scale is not None and self.downsample_scale > 1:
            self.down = nn.Conv1d(self.hidden_size, self.hidden_size, kernel_size=3, stride=2, padding=1)
            self.up = nn.Conv1d(self.hidden_size, self.hidden_size, kernel_size=3, stride=1, padding=1)
        self.encoder = VocosLinear(self.hidden_size, self.vocos_dim, self.vocos_intermediate_dim, self.vocos_num_layers,
                                   self.hidden_size)
        self.decoder = VocosLinear(self.hidden_size, self.vocos_dim, self.vocos_intermediate_dim, self.vocos_num_layers,
                                   self.hidden_size)
        self.quantizer = ResidualVQ(input_dim=hidden_size, num_quantizers=num_quantizers, codebook_size=codebook_size,
                                    codebook_dim=codebook_dim, quantizer_type="fvq", quantizer_dropout=0.0,
                                    commitment=0.15, codebook_loss_weight=1.0, use_l2_normlize=True)
        self.last_launches = 0
        self.reset_parameters()

    @property
    def precision(self):
        return self.encoder.precision

    @precision.setter
    def precision(self, value):
        for m in (self.encoder, self.decoder, self.quantizer):
            m.precision = value

    def _encode(self, x, who):
        """x [B, T, hidden] -> the encoder's output as the [B, hidden, T] view the reference quantizes, and the RVQ's
        quantized_out [B, hidden, T] and codes [n, B, T]."""
        _refuse_training(self, "RepCodec", "quantizer dropout, commitment and codebook losses", _SERVED)
        if not isinstance(x, torch.Tensor) or x.dim() != 3 or x.shape[2] != self.hidden_size:
            got = tuple(x.shape) if isinstance(x, torch.Tensor) else type(x).__name__
            raise ValueError(f"RepCodec.{who} expects features of shape [B, T, {self.hidden_size}], got {got}")
        h = self.encoder(x.transpose(1, 2)).transpose(1, 2)
        qo, codes, _ = self.quantizer._quantize(h, self.num_quantizers, False)
        self.last_launches = self.encoder.last_launches + self.quantizer.last_launches
        return qo, codes

    def quantize(self, x):
        """x [B, T, hidden] -> (codes int64 [B, T] with one quantizer, else [n, B, T]; quantized [B, T, hidden], the
        transposed view of quantized_out, as the reference returns it)."""
        qo, codes = self._encode(x, "quantize")
        if codes.shape[0] == 1:
            return codes.squeeze(0), qo.transpose(1, 2)
        return codes, qo.transpose(1, 2)

    def forward(self, x):
        """x [B, T, hidden] -> (x_rec [B, T, hidden], codebook_loss (0-dim, zero in eval), all_indices [n, B, T])."""
        qo, codes = self._encode(x, "forward")
        launches = self.last_launches
        x_rec = self.decoder(qo)
        self.last_launches = launches + self.decoder.last_launches
        return x_rec, torch.zeros((), dtype=torch.float32, device=qo.device), codes

    def reset_parameters(self):
        self.apply(init_weights)
