"""CodecEncoder / CodecDecoder — drop-ins for the acoustic codec of MaskGCT, Metis and DebaTTS
(``models/codec/amphion_codec/codec.py:100-427``, ``quantizer_type="fvq"``, ``use_vocos=True``): the same constructors
(keyword defaults, ``cfg`` fields override them) and the same parameter trees, drawn in the same order, so the released
acoustic codec checkpoints load strictly.  Served natively:

- ``CodecEncoder.forward(wav [B, 1, N]) -> [B, out_channels, F]``, F = ``frames(N)``: the FACodec encoder's route
  (``AB_GEN_FACODEC_ENCODER``) with every activation a plain Snake1d (``AB_ACT_SNAKE1D``);
- ``CodecDecoder.quantizer`` is a native ``ResidualVQ`` (``AB_GEN_RVQ``): ``forward`` / ``quantize`` return the codes
  and the quantized latent, ``vq2emb`` turns codes back into the latent, on FACodec's RVQ kernels in fp32;
- ``CodecDecoder.model`` is the native ``Vocos``: ``forward(x)`` / ``decode(x)`` give the 24 kHz waveform.

The quantizer in training mode (quantizer dropout), ``latent2dist``, ``use_tanh=True``, ``use_vocos=False``, the ``"vq"``
and ``"lfq"`` quantizers and ``use_l2_normlize=False`` are not served: no config in the reference uses them."""
from __future__ import annotations

import numpy as np
import torch
from torch import nn
from torch.nn.utils import weight_norm

from .. import _capi
from .facodec import _FACodecGenerator, _block_config, _refuse_training
from .generator import NativeGenerator
from .vocos import Vocos

_SERVED = ("amphion_b200 serves CodecEncoder.forward(), CodecDecoder.forward() / .decode() (Vocos), and in eval "
           "CodecDecoder.forward(vq=True) / .quantize() / .vq2emb() and ResidualVQ.forward() / .vq2emb()")


def _native_only(name):
    raise RuntimeError(f"amphion_b200: the codec's {name} executes inside the native pipeline; {_SERVED}")


def _wn_conv(*args, **kwargs):
    return weight_norm(nn.Conv1d(*args, **kwargs))


def _init_weights(m):
    """codec.py:51-57: every Conv1d and Linear gets trunc_normal(std 0.02) weights and zero biases."""
    if isinstance(m, (nn.Conv1d, nn.Linear)):
        nn.init.trunc_normal_(m.weight, std=0.02)
        nn.init.constant_(m.bias, 0)


class Snake1d(nn.Module):
    """Parameter holder for codec.py:42-48: ``alpha`` [1, C, 1]."""

    def __init__(self, channels):
        super().__init__()
        self.alpha = nn.Parameter(torch.ones(1, channels, 1))

    def forward(self, x):
        _native_only("Snake1d")


class ResidualUnit(nn.Module):
    """Parameter holder for codec.py:60-76."""

    def __init__(self, dim: int = 16, dilation: int = 1):
        super().__init__()
        pad = ((7 - 1) * dilation) // 2
        self.block = nn.Sequential(Snake1d(dim), _wn_conv(dim, dim, kernel_size=7, dilation=dilation, padding=pad),
                                   Snake1d(dim), _wn_conv(dim, dim, kernel_size=1))

    def forward(self, x):
        _native_only("ResidualUnit")


class EncoderBlock(nn.Module):
    """Parameter holder for codec.py:79-97."""

    def __init__(self, dim: int = 16, stride: int = 1):
        super().__init__()
        self.block = nn.Sequential(
            ResidualUnit(dim // 2, dilation=1), ResidualUnit(dim // 2, dilation=3), ResidualUnit(dim // 2, dilation=9),
            Snake1d(dim // 2),
            _wn_conv(dim // 2, dim, kernel_size=2 * stride, stride=stride, padding=(stride + 1) // 2))

    def forward(self, x):
        _native_only("EncoderBlock")


class CodecEncoder(_FACodecGenerator):
    """Drop-in for CodecEncoder (codec.py:100-143).  ``forward(x)``: wav ``[B, 1, N]`` (any strides) ->
    ``[B, out_channels, F]`` fp32 on the wav's device, F = ``frames(N)``."""

    kind = "codec_encoder"

    def __init__(self, d_model: int = 64, up_ratios: list = (4, 5, 5, 6), out_channels: int = 256,
                 use_tanh: bool = False, cfg=None):
        super().__init__()
        d_model = cfg.d_model if cfg is not None else d_model
        up_ratios = cfg.up_ratios if cfg is not None else up_ratios
        out_channels = cfg.out_channels if cfg is not None else out_channels
        use_tanh = cfg.use_tanh if cfg is not None else use_tanh
        if use_tanh:
            raise NotImplementedError(f"amphion_b200: CodecEncoder(use_tanh=True) is not served (no reference config "
                                      f"sets it); {_SERVED}")
        self.ngf, self.up_ratios, self.out_channels = int(d_model), [int(u) for u in up_ratios], int(out_channels)
        self.hop_length = int(np.prod(self.up_ratios))
        block = [_wn_conv(1, d_model, kernel_size=7, padding=3)]
        for stride in up_ratios:
            d_model *= 2
            block.append(EncoderBlock(d_model, stride=stride))
        block += [Snake1d(d_model), _wn_conv(d_model, out_channels, kernel_size=3, padding=1)]
        self.block = nn.Sequential(*block)
        self.enc_dim = d_model
        self.reset_parameters()

    def reset_parameters(self):
        self.apply(_init_weights)

    # ---- NativeGenerator hooks -------------------------------------------------------
    def _input_channels(self):
        return 1

    def _c_config(self):
        if len(self.up_ratios) > _capi.AB_MAX_STAGES:
            raise ValueError("amphion_b200: too many up_ratios for the native encoder")
        c = _block_config(_capi.GEN_FACODEC_ENCODER, 1, self.ngf, self.up_ratios)
        c.activation, c.snake_logscale = _capi.ACT_SNAKE1D, 0
        c.trunk_out_channels = self.out_channels
        return c

    def frames(self, n_samples):
        """Output frames for n_samples input samples (0: a strided conv would have no output)."""
        t = int(n_samples)
        for s in self.up_ratios:
            pad = (s + 1) // 2
            if t <= 0 or t + 2 * pad < 2 * s:
                return 0
            t = (t + 2 * pad - 2 * s) // s + 1
        return t

    # ---- served methods --------------------------------------------------------------
    def forward(self, x, out=None):
        """wav [B, 1, N] (any strides) -> [B, out_channels, F] fp32.  ``out`` (beyond the reference signature): a
        contiguous fp32 [B, out_channels, F] tensor to write into."""
        if not isinstance(x, torch.Tensor) or x.dim() != 3 or x.shape[1] != 1:
            got = tuple(x.shape) if isinstance(x, torch.Tensor) else type(x).__name__
            raise ValueError(f"CodecEncoder expects a waveform of shape [B, 1, N], got {got}")
        B, _, N = x.shape
        if B == 0 or N == 0:
            raise ValueError("amphion_b200: empty waveform batch")
        F = self.frames(N)
        if F <= 0:
            raise ValueError(f"CodecEncoder: {N} samples are too short for up_ratios {self.up_ratios} (a strided conv's "
                             f"padded input would be shorter than its kernel)")
        _capi.require_cuda(x, "CodecEncoder.forward")
        if x.dtype != torch.float32:
            x = x.float()
        with self._launch(x.device) as h:
            need = _capi.lib.ab_generator_workspace_bytes(h, B, N)
            ws = self._scratch(need, x.device)
            y = self._output(out, (B, self.out_channels, F), x.device)
            _capi.check(_capi.lib.ab_facodec_encode(h, _capi.ptr(x), B, N, _capi.shape_array(x.stride()), _capi.ptr(y),
                                                    ws, need, _capi.stream_ptr()), "ab_facodec_encode")
        return y


class FactorizedVectorQuantize(nn.Module):
    """Parameter holder for quantize/factorized_vector_quantize.py:22-50 (input_dim != codebook_dim: weight-normed
    k = 1 ``in_project`` / ``out_project``, ``codebook``)."""

    def __init__(self, input_dim, codebook_size, codebook_dim, commitment=0.005, codebook_loss_weight=1.0,
                 use_l2_normlize=True):
        super().__init__()
        if not use_l2_normlize:
            raise NotImplementedError(f"amphion_b200: FactorizedVectorQuantize(use_l2_normlize=False) is not served (no "
                                      f"reference config sets it); {_SERVED}")
        if input_dim == codebook_dim:
            raise NotImplementedError("amphion_b200: FactorizedVectorQuantize with input_dim == codebook_dim (identity "
                                      "projections) is not served")
        self.input_dim, self.codebook_size, self.codebook_dim = input_dim, codebook_size, codebook_dim
        self.commitment, self.codebook_loss_weight, self.use_l2_normlize = commitment, codebook_loss_weight, use_l2_normlize
        self.in_project = _wn_conv(input_dim, codebook_dim, kernel_size=1)
        self.out_project = _wn_conv(codebook_dim, input_dim, kernel_size=1)
        self.codebook = nn.Embedding(codebook_size, codebook_dim)

    def forward(self, z):
        _native_only("FactorizedVectorQuantize (run the ResidualVQ)")


class ResidualVQ(NativeGenerator):
    """Drop-in for ResidualVQ (quantize/residual_vq.py:21-144) with ``quantizer_type="fvq"``, served in eval
    (``AB_GEN_RVQ``): every layer's projections, code search and straight-through step in fp32 on CUDA cores, at every
    precision.  ``forward(z, n_quantizers)`` -> ``(quantized_out [B, D, T], all_indices int64 [n, B, T],
    all_commit_losses [n], all_codebook_losses [n], all_quantized [n, B, D, T])``; ``vq2emb(vq, n_quantizers)``."""

    kind = "rvq"

    def __init__(self, input_dim: int = 256, num_quantizers: int = 8, codebook_size: int = 1024,
                 codebook_dim: int = 256, quantizer_type: str = "vq", quantizer_dropout: float = 0.5, **kwargs):
        super().__init__()
        if quantizer_type != "fvq":
            raise NotImplementedError(f"amphion_b200: ResidualVQ(quantizer_type={quantizer_type!r}) is not served, only "
                                      f"'fvq'; {_SERVED}")
        self.input_dim, self.num_quantizers = int(input_dim), int(num_quantizers)
        self.codebook_size, self.codebook_dim = int(codebook_size), int(codebook_dim)
        self.quantizer_type, self.quantizer_dropout = quantizer_type, quantizer_dropout
        self.quantizers = nn.ModuleList([FactorizedVectorQuantize(input_dim=input_dim, codebook_size=codebook_size,
                                                                  codebook_dim=codebook_dim, **kwargs)
                                         for _ in range(num_quantizers)])

    def _c_config(self):
        c = _capi.GeneratorConfig()
        c.kind, c.n_mel = _capi.GEN_RVQ, self.input_dim
        c.vq_num_q[0], c.vq_codebook_dim, c.vq_codebook_size = self.num_quantizers, self.codebook_dim, self.codebook_size
        return c

    def _n(self, n_quantizers, who):
        n = self.num_quantizers if n_quantizers is None else int(n_quantizers)
        if n < 1 or n > self.num_quantizers:
            raise ValueError(f"amphion_b200: {who}: n_quantizers {n_quantizers} outside 1..{self.num_quantizers}")
        return n

    def forward(self, z, n_quantizers: int = None):
        """z [B, input_dim, T] fp32 (any strides) on a CUDA device -> the reference's 5-tuple, without autograd
        history; the losses are the zeros the reference returns in eval."""
        _refuse_training(self, "the ResidualVQ", "quantizer dropout, commitment losses", _SERVED)
        n = self._n(n_quantizers, "ResidualVQ.forward")
        out, codes, layers = self._quantize(z, n, True)
        zeros = torch.zeros(n, dtype=torch.float32, device=out.device)
        return out, codes, zeros, zeros.clone(), layers

    def _quantize(self, z, n, with_layers):
        """quantized_out, codes and, with ``with_layers``, all_quantized (else None: nothing is written for it)."""
        if not isinstance(z, torch.Tensor) or z.dim() != 3 or z.shape[1] != self.input_dim:
            got = tuple(z.shape) if isinstance(z, torch.Tensor) else type(z).__name__
            raise ValueError(f"ResidualVQ expects z of shape [B, {self.input_dim}, T], got {got}")
        B, D, T = z.shape
        if B == 0 or T == 0:
            raise ValueError("amphion_b200: empty latent batch")
        _capi.require_cuda(z, "ResidualVQ.forward")
        z = z.float()
        dev = z.device
        with self._launch(dev) as h:
            out = torch.empty(B, D, T, dtype=torch.float32, device=dev)
            codes = torch.empty(n, B, T, dtype=torch.int64, device=dev)
            layers = torch.empty(n, B, D, T, dtype=torch.float32, device=dev) if with_layers else None
            _capi.check(_capi.lib.ab_rvq_quantize(h, _capi.ptr(z), _capi.shape_array(z.stride()), B, T, n, _capi.ptr(out),
                                                  _capi.ptr(codes), _capi.ptr(layers), _capi.stream_ptr()),
                        "ab_rvq_quantize")
        return out, codes, layers

    def vq2emb(self, vq, n_quantizers=None):
        """codes [>= n, B, T] (integer, any strides) -> [B, input_dim, T] fp32 on the codes' device."""
        n = self._n(n_quantizers, "ResidualVQ.vq2emb")
        if not isinstance(vq, torch.Tensor) or vq.dim() != 3 or vq.is_floating_point() or vq.is_complex() \
                or vq.dtype == torch.bool:
            got = f"{vq.dtype} {tuple(vq.shape)}" if isinstance(vq, torch.Tensor) else type(vq).__name__
            raise ValueError(f"ResidualVQ.vq2emb expects integer codes [n_q, B, T], got {got}")
        if vq.shape[0] < n:
            raise ValueError(f"ResidualVQ.vq2emb: {vq.shape[0]} code rows, fewer than n_quantizers = {n}")
        _, B, T = vq.shape
        if B == 0 or T == 0:
            raise ValueError("amphion_b200: empty code batch")
        _capi.require_cuda(vq, "ResidualVQ.vq2emb")
        vq = vq.long()
        lo, hi = int(vq[:n].min()), int(vq[:n].max())
        if lo < 0 or hi >= self.codebook_size:
            # the kernel would not read such a code (it writes NaN there): refuse it first, as F.embedding does
            raise ValueError(f"ResidualVQ.vq2emb: the codes hold {lo}..{hi}, outside the codebook [0, {self.codebook_size})")
        with self._launch(vq.device) as h:
            out = torch.empty(B, self.input_dim, T, dtype=torch.float32, device=vq.device)
            _capi.check(_capi.lib.ab_rvq_vq2emb(h, _capi.ptr(vq), _capi.shape_array(vq.stride()), n, B, T, _capi.ptr(out),
                                                _capi.stream_ptr()), "ab_rvq_vq2emb")
        return out

    def latent2dist(self, *args, **kwargs):
        raise NotImplementedError(f"amphion_b200: ResidualVQ.latent2dist is not served (no caller uses it); {_SERVED}")


class CodecDecoder(nn.Module):
    """Drop-in for CodecDecoder (codec.py:168-427) with ``quantizer_type="fvq"`` and ``use_vocos=True``: ``quantizer``
    is the native ``ResidualVQ`` and ``model`` the native ``Vocos``, so the state dict's keys are ``quantizer.*``,
    ``model.backbone.*`` and ``model.head.*``."""

    def __init__(self, in_channels: int = 256, upsample_initial_channel: int = 1536, up_ratios: list = (5, 5, 4, 2),
                 num_quantizers: int = 8, codebook_size: int = 1024, codebook_dim: int = 256,
                 quantizer_type: str = "vq", quantizer_dropout: float = 0.5, commitment: float = 0.25,
                 codebook_loss_weight: float = 1.0, use_l2_normlize: bool = False, codebook_type: str = "euclidean",
                 kmeans_init: bool = False, kmeans_iters: int = 10, decay: float = 0.8, eps: float = 1e-5,
                 threshold_ema_dead_code: int = 2, weight_init: bool = False, use_vocos: bool = False,
                 vocos_dim: int = 384, vocos_intermediate_dim: int = 1152, vocos_num_layers: int = 8, n_fft: int = 800,
                 hop_size: int = 200, padding: str = "same", cfg=None):
        super().__init__()

        def pick(name, default):
            return getattr(cfg, name) if cfg is not None and hasattr(cfg, name) else default

        in_channels = pick("in_channels", in_channels)
        num_quantizers = pick("num_quantizers", num_quantizers)
        codebook_size = pick("codebook_size", codebook_size)
        codebook_dim = pick("codebook_dim", codebook_dim)
        quantizer_type = pick("quantizer_type", quantizer_type)
        quantizer_dropout = pick("quantizer_dropout", quantizer_dropout)
        commitment = pick("commitment", commitment)
        codebook_loss_weight = pick("codebook_loss_weight", codebook_loss_weight)
        use_l2_normlize = pick("use_l2_normlize", use_l2_normlize)
        use_vocos = pick("use_vocos", use_vocos)
        vocos_dim = pick("vocos_dim", vocos_dim)
        vocos_intermediate_dim = pick("vocos_intermediate_dim", vocos_intermediate_dim)
        vocos_num_layers = pick("vocos_num_layers", vocos_num_layers)
        n_fft = pick("n_fft", n_fft)
        hop_size = pick("hop_size", hop_size)
        padding = pick("padding", padding)
        if quantizer_type not in ("vq", "fvq", "lfq"):
            raise ValueError(f"Unknown quantizer type {quantizer_type}")
        if quantizer_type != "fvq":
            raise NotImplementedError(f"amphion_b200: CodecDecoder(quantizer_type={quantizer_type!r}) is not served, only "
                                      f"'fvq'; {_SERVED}")
        if not use_l2_normlize:
            raise NotImplementedError(f"amphion_b200: CodecDecoder(use_l2_normlize=False) is not served (no reference "
                                      f"config sets it); {_SERVED}")
        if not use_vocos:
            raise NotImplementedError(f"amphion_b200: CodecDecoder(use_vocos=False), the DAC-style decoder, is not "
                                      f"served; {_SERVED}")
        self.quantizer = ResidualVQ(input_dim=in_channels, num_quantizers=num_quantizers, codebook_size=codebook_size,
                                    codebook_dim=codebook_dim, quantizer_type=quantizer_type,
                                    quantizer_dropout=quantizer_dropout, commitment=commitment,
                                    codebook_loss_weight=codebook_loss_weight, use_l2_normlize=use_l2_normlize)
        self.model = Vocos(input_channels=in_channels, dim=vocos_dim, intermediate_dim=vocos_intermediate_dim,
                           num_layers=vocos_num_layers, adanorm_num_embeddings=None, n_fft=n_fft, hop_size=hop_size,
                           padding=padding)
        self.reset_parameters()

    def forward(self, x=None, vq=False, eval_vq=False, n_quantizers=None):
        """``vq=True``: x = the encoder's output, returns the quantizer's 5-tuple; else x = the quantized latent,
        returns the waveform [B, 1, T * hop_size]."""
        if vq is True:
            if eval_vq:
                self.quantizer.eval()
            return self.quantizer(x, n_quantizers=n_quantizers)
        return self.model(x)

    def quantize(self, x, n_quantizers=None):
        self.quantizer.eval()
        quantized_out, vq, _, _, _ = self.quantizer(x, n_quantizers=n_quantizers)
        return quantized_out, vq

    def vq2emb(self, vq, n_quantizers=None):
        return self.quantizer.vq2emb(vq, n_quantizers=n_quantizers)

    def decode(self, x):
        return self.model(x)

    def latent2dist(self, x, n_quantizers=None):
        return self.quantizer.latent2dist(x, n_quantizers=n_quantizers)

    def reset_parameters(self):
        self.apply(_init_weights)
