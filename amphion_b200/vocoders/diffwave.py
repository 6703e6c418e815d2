"""DiffWave — drop-in for the reference class ``models/vocoders/diffusion/diffwave/diffwave.py:127`` (``_vocoders["diffwave"]``,
recipe ``egs/vocoder/diffusion/diffwave``): the same constructor, including its side effect of writing
``cfg.model.diffwave.noise_schedule``, the same parameter tree (``input_projection``, ``diffusion_embedding.projection{1,2}``
with the non-persistent ``diffusion_embedding.embedding`` table, ``spectrogram_upsampler.conv{1,2}``,
``residual_layers.{i}.{dilated_conv,diffusion_projection,conditioner_projection,output_projection}``, ``skip_projection``,
``output_projection``) drawn in the same order, and ``forward(audio, diffusion_step, spectrogram) -> eps [B, 1, L]`` on the
native pipeline (``AB_GEN_DIFFWAVE``: the residual layers on the tensor cores at ``tc_f16`` / ``tc_bf16``, on CUDA-core
FMAs at ``fp32``).  ``diffusion_vocoder_inference`` runs the reference's
sampler loop on top of the conditioning / step entry points."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch
from torch import nn

from .. import _capi
from .generator import NativeGenerator


def _native_only(name):
    raise RuntimeError(f"amphion_b200: DiffWave's {name} executes inside the CUDA pipeline; call DiffWave.forward()")


def _conv1d(*args, **kwargs):
    """nn.Conv1d redrawn with kaiming_normal_, as every Conv1d of the reference model is (diffwave.py:21-24)."""
    conv = nn.Conv1d(*args, **kwargs)
    nn.init.kaiming_normal_(conv.weight)
    return conv


def _step_table(rows):
    """[rows, 128]: sin / cos of step * 10^(4 j / 63), j < 64, computed with the reference's fp32 tensor ops."""
    step = torch.arange(rows).unsqueeze(1)
    freq = 10.0 ** (torch.arange(64).unsqueeze(0) * 4.0 / 63.0)
    angle = step * freq
    return torch.cat([torch.sin(angle), torch.cos(angle)], dim=1)


class DiffusionEmbedding(nn.Module):
    def __init__(self, max_steps):
        super().__init__()
        self.register_buffer("embedding", _step_table(max_steps), persistent=False)
        self.projection1 = nn.Linear(128, 512)
        self.projection2 = nn.Linear(512, 512)

    def forward(self, *args, **kwargs):
        _native_only("diffusion embedding")


class SpectrogramUpsampler(nn.Module):
    def __init__(self, upsample_factors):
        super().__init__()
        f1, f2 = (int(f) for f in upsample_factors)
        self.conv1 = nn.ConvTranspose2d(1, 1, [3, 2 * f1], stride=[1, f1], padding=[1, f1 // 2])
        self.conv2 = nn.ConvTranspose2d(1, 1, [3, 2 * f2], stride=[1, f2], padding=[1, f2 // 2])

    def forward(self, *args, **kwargs):
        _native_only("spectrogram upsampler")


class ResidualBlock(nn.Module):
    def __init__(self, n_mels, residual_channels, dilation):
        super().__init__()
        self.dilated_conv = _conv1d(residual_channels, 2 * residual_channels, 3, padding=dilation, dilation=dilation)
        self.diffusion_projection = nn.Linear(512, residual_channels)
        self.conditioner_projection = _conv1d(n_mels, 2 * residual_channels, 1)
        self.output_projection = _conv1d(residual_channels, 2 * residual_channels, 1)

    def forward(self, *args, **kwargs):
        _native_only("residual layers")


class DiffWave(NativeGenerator):
    kind = "diffwave"
    hp_key = "diffwave"

    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        hp = cfg.model.diffwave
        f = hp.noise_schedule_factors
        hp.noise_schedule = np.linspace(f[0], f[1], f[2]).tolist()   # read by the sampler
        C, L = int(hp.residual_channels), int(hp.residual_layers)
        self.upsample_factors = [int(f) for f in hp.upsample_factors]
        self.input_projection = _conv1d(1, C, 1)
        self.diffusion_embedding = DiffusionEmbedding(len(hp.noise_schedule))
        self.spectrogram_upsampler = SpectrogramUpsampler(self.upsample_factors)
        self.residual_layers = nn.ModuleList([ResidualBlock(cfg.preprocess.n_mel, C, 2 ** (i % hp.dilation_cycle_length))
                                              for i in range(L)])
        self.skip_projection = _conv1d(C, C, 1)
        self.output_projection = _conv1d(C, 1, 1)
        nn.init.zeros_(self.output_projection.weight)

    def _hop(self):
        return self.upsample_factors[0] * self.upsample_factors[1]

    def _input_channels(self):
        return int(self.cfg.preprocess.n_mel)

    def _check_factors(self):
        if len(self.upsample_factors) != 2 or any(f <= 0 or f % 2 for f in self.upsample_factors):
            raise ValueError(f"amphion_b200: DiffWave needs two even upsample_factors (got {self.upsample_factors}): an odd "
                             "factor makes the upsampled spectrogram one sample longer than the audio")

    def _c_config(self):
        hp = self.cfg.model.diffwave
        c = _capi.GeneratorConfig()
        c.kind = _capi.GEN_DIFFWAVE
        c.n_mel = int(self.cfg.preprocess.n_mel)
        c.upsample_initial_channel = int(hp.residual_channels)
        c.num_layers = int(hp.residual_layers)
        c.num_upsamples = len(self.upsample_factors)
        for i, f in enumerate(self.upsample_factors[:_capi.AB_MAX_STAGES]):
            c.upsample_rates[i] = f
        c.dilation_cycle = int(hp.dilation_cycle_length)
        c.embedding_rows = int(self.diffusion_embedding.embedding.shape[0])
        return c

    # ---- native entry points -----------------------------------------------------------------------------------
    def _check_mel(self, spectrogram, need_cuda=True):
        self._check_factors()
        if spectrogram.dim() != 3 or spectrogram.shape[1] != self._input_channels() or spectrogram.shape[0] == 0 \
                or spectrogram.shape[2] == 0:
            raise ValueError(f"expected a spectrogram of shape [B, {self._input_channels()}, F], got {tuple(spectrogram.shape)}")
        if need_cuda:
            _capi.require_cuda(spectrogram, "DiffWave")
        return spectrogram if spectrogram.dtype == torch.float32 else spectrogram.float()

    def _ensure_workspace(self, B, F, n_steps, device):
        need = _capi.lib.ab_diffwave_workspace_bytes(self._handle, B, F, n_steps)
        if need == 0:
            raise RuntimeError(f"amphion_b200: DiffWave workspace query failed: {_capi.last_error()}")
        return self._scratch(need, device), need

    def _condition(self, spectrogram, steps):
        """Upsampled mel and the diffusion projections of every value in ``steps`` (host floats) into the workspace;
        returns (workspace pointer, bytes)."""
        B, _, F = spectrogram.shape
        steps = np.ascontiguousarray(steps, dtype=np.float32)
        with self._launch(spectrogram.device) as h:
            ws, need = self._ensure_workspace(B, F, len(steps), spectrogram.device)
            _capi.check(_capi.lib.ab_diffwave_condition(
                h, _capi.ptr(spectrogram), B, F, _capi.shape_array(spectrogram.stride()),
                steps.ctypes.data_as(C.POINTER(C.c_float)), len(steps), ws, need, _capi.stream_ptr()),
                "ab_diffwave_condition")
        return ws, need

    def _step(self, audio, row, c1, c2, sigma, noise, ws, need):
        """One sampler update of ``audio`` [B, L] in place with conditioning row ``row``, on the workspace and the
        parameters ``_condition`` left (the sampler calls it under the audio's device)."""
        B, L = audio.shape
        _capi.check(_capi.lib.ab_diffwave_step(self._handle, _capi.ptr(audio), B, L // self._hop(), row, float(c1), float(c2),
                                               float(sigma), _capi.ptr(noise), None, ws, need, _capi.stream_ptr()),
                    "ab_diffwave_step")
        self._count_launches()

    def forward(self, audio, diffusion_step, spectrogram):
        """audio [B, L], diffusion_step [1] or [B] (integer: a table row; float: lerp between rows), spectrogram
        [B, n_mel, F] (any strides), all on one CUDA device, L = F * prod(upsample_factors) -> eps [B, 1, L] fp32."""
        spectrogram = self._check_mel(spectrogram, need_cuda=False)
        B, _, F = spectrogram.shape
        if audio.dim() != 2 or audio.shape[0] != B or audio.shape[1] != F * self._hop():
            raise ValueError(f"amphion_b200: DiffWave audio must be [{B}, {F * self._hop()}] for {F} frames and upsample "
                             f"factors {self.upsample_factors}, got {tuple(audio.shape)}")
        steps = torch.as_tensor(diffusion_step).detach().reshape(-1).to("cpu", torch.float32).numpy()
        if len(steps) not in (1, B):
            raise ValueError(f"amphion_b200: diffusion_step must hold 1 or {B} values, got {len(steps)}")
        _capi.require_cuda(spectrogram, "DiffWave.forward")
        _capi.require_cuda(audio, "DiffWave.forward")
        if audio.device != spectrogram.device:
            raise ValueError("amphion_b200: audio and spectrogram must be on the same device")
        audio = audio.float().contiguous()
        with self._launch(spectrogram.device) as h:
            ws, need = self._ensure_workspace(B, F, len(steps), spectrogram.device)
            eps = torch.empty(B, 1, audio.shape[1], dtype=torch.float32, device=audio.device)
            _capi.check(_capi.lib.ab_diffwave_forward(
                h, _capi.ptr(audio), B, F, _capi.ptr(spectrogram), _capi.shape_array(spectrogram.stride()),
                steps.ctypes.data_as(C.POINTER(C.c_float)), len(steps), _capi.ptr(eps), ws, need, _capi.stream_ptr()),
                "ab_diffwave_forward")
        return eps
