"""APNet generator — drop-in for ``models/vocoders/gan/generator/apnet.py:283-399`` (``_vocoders["apnet"]``,
models/vocoders/vocoder_inference.py:48): same constructor (``cfg``), same parameter names
(``ASP_input_conv``, ``ASP_ResNet.j.convs{1,2}.p``, ``ASP_output_conv``, ``PSP_*``), and
``forward(mel[B, n_mel, T]) -> (logamp, pha, rea, imag, audio[B, 1, T*hop])``.

Two frame-rate ResNet trunks (amplitude and phase streams) run on the native generator pipeline
(``AB_GEN_TRUNK``: the same tensor-core ResBlock kernels the HiFi-GAN stages use); the phase stream's two output
convolutions are one convolution with the R and I filters stacked.  ``ab_spectral_head_forward`` turns
(logamp, R, I) into phase / real / imaginary parts and the complex spectrum, and ``ab_istft_forward`` (cuFFT C2R +
windowed overlap-add, the reference's ``ISTFT`` with "same" padding, apnet.py:16-104) produces the audio."""
from __future__ import annotations

import ctypes as C

import torch
from torch import nn
from torch.nn.utils import remove_weight_norm, weight_norm

from .. import _capi
from .generator import ConvBlock, DEFAULT_PRECISION, NativeGenerator, get_padding, init_weights


class ISTFT(nn.Module):
    """apnet.py:16-104, ``padding="same"`` (the only mode APNet uses): spec complex [B, N, T] -> [B, T*hop]."""

    def __init__(self, n_fft: int, hop_length: int, win_length: int, padding: str = "same"):
        super().__init__()
        if padding not in ["center", "same"]:
            raise ValueError("Padding must be 'center' or 'same'.")
        if padding != "same":
            raise NotImplementedError("amphion_b200: ISTFT runs the 'same' padding mode (the one APNet constructs)")
        self.padding, self.n_fft, self.hop_length, self.win_length = padding, n_fft, hop_length, win_length
        self._handles = {}            # cuFFT plans belong to a device: one native handle per device

    def _mel_handle(self, device):
        key = str(device)
        if key not in self._handles:
            h = C.c_void_p()
            cfg = _capi.MelConfig(self.n_fft, self.hop_length, self.win_length, 0, 0, 0.0, 0.0)
            _capi.check(_capi.lib.ab_mel_create(C.byref(cfg), C.byref(h)), "ab_mel_create")
            self._handles[key] = h
        return self._handles[key]

    def forward_interleaved(self, spec_ri, B, T, window):
        """spec_ri: fp32 [B*T, N, 2] (frames-major, overwritten) -> audio [B, T*hop]."""
        lib = _capi.lib
        with torch.cuda.device(spec_ri.device):
            h = self._mel_handle(spec_ri.device)
            need = lib.ab_istft_workspace_bytes(h, B, T)
            if need == 0:
                raise RuntimeError("amphion_b200: " + _capi.last_error())
            ws = torch.empty(need + 256, dtype=torch.uint8, device=spec_ri.device)
            wbase = (ws.data_ptr() + 255) // 256 * 256
            pad = (self.win_length - self.hop_length) // 2
            L = (T - 1) * self.hop_length + self.win_length - 2 * pad
            wav = torch.empty(B, L, dtype=torch.float32, device=spec_ri.device)
            window = window.to(device=spec_ri.device, dtype=torch.float32).contiguous()
            _capi.check(lib.ab_istft_forward(h, _capi.ptr(spec_ri), B, T, _capi.ptr(window), _capi.ptr(wav),
                                             C.c_void_p(wbase), need, _capi.stream_ptr()), "ab_istft_forward")
        return wav

    def forward(self, spec: torch.Tensor, window) -> torch.Tensor:
        _capi.require_cuda(spec, "ISTFT.forward")
        assert spec.dim() == 3, "Expected a 3D tensor as input"
        B, N, T = spec.shape
        ri = torch.view_as_real(spec.to(torch.complex64)).permute(0, 2, 1, 3).contiguous().view(B * T, N, 2)
        return self.forward_interleaved(ri, B, T, window)

    def __getstate__(self):
        state = self.__dict__.copy()
        state["_handles"] = {}        # ctypes handles are derived state
        return state

    def __del__(self):
        try:
            for h in self._handles.values():
                _capi.lib.ab_mel_destroy(h)
        except Exception:
            pass


class _Trunk(NativeGenerator):
    """One stream of APNet as a native handle.  Holds no parameters of its own: ``tensors()`` of the owning APNet
    supplies them under the trunk's names (conv_pre / resblocks.j / conv_post)."""
    kind = "trunk"

    def __init__(self, owner, stream):
        super().__init__()
        object.__setattr__(self, "_owner", owner)     # not a submodule: the owner registers the parameters
        self._stream = stream
        self.cfg = owner.cfg

    def _c_config(self):
        hp = self.cfg.model.apnet
        s = self._stream
        c = _capi.GeneratorConfig()
        c.kind = _capi.GEN_TRUNK
        c.n_mel = int(self.cfg.preprocess.n_mel)
        c.upsample_initial_channel = int(getattr(hp, f"{s}_channel"))
        c.num_upsamples = 0
        c.resblock = 1
        rks = list(getattr(hp, f"{s}_resblock_kernel_sizes"))
        rds = [list(d) for d in getattr(hp, f"{s}_resblock_dilation_sizes")]
        if len(rks) > _capi.AB_MAX_KERNELS or any(len(d) > _capi.AB_MAX_DILATIONS for d in rds):
            raise ValueError("amphion_b200: too many kernels / dilations for the native generator")
        c.num_kernels = len(rks)
        for j, (k, ds) in enumerate(zip(rks, rds)):
            c.resblock_kernel_sizes[j] = int(k)
            c.num_dilations[j] = len(ds)
            for p, d in enumerate(ds):
                c.resblock_dilation_sizes[j][p] = int(d)
        c.activation = _capi.ACT_LRELU
        bins = int(self.cfg.preprocess.n_fft) // 2 + 1
        c.trunk_out_channels = bins if s == "ASP" else 2 * bins
        c.trunk_in_kernel = int(getattr(hp, f"{s}_input_conv_kernel_size"))
        c.trunk_out_kernel = int(hp.ASP_output_conv_kernel_size if s == "ASP" else hp.PSP_output_R_conv_kernel_size)
        return c

    # the owner's tensors under the trunk's names
    def named_parameters(self, *a, **k):
        return iter(self._owner._trunk_tensors(self._stream).items())

    def named_buffers(self, *a, **k):
        return iter(())

    def parameters(self, *a, **k):
        return iter(self._owner._trunk_tensors(self._stream).values())

    def buffers(self, *a, **k):
        return iter(())

    def _param_key(self, device):
        src = [t for n, t in self._owner.named_parameters() if n.startswith(self._stream)]
        return (str(device), self.precision, tuple((t.data_ptr(), t._version) for t in src))

    def run(self, mel):
        """mel [B, n_mel, T] -> [B, trunk_out_channels, T]"""
        _capi.require_cuda(mel, "APNet.forward")
        if mel.dtype != torch.float32:
            mel = mel.float()
        B, _, T = mel.shape
        with self._launch(mel.device) as h:
            need = _capi.lib.ab_generator_workspace_bytes(h, B, T)
            ws = self._scratch(need, mel.device)
            cout = self._c_config().trunk_out_channels
            out = torch.empty(B, cout, T, dtype=torch.float32, device=mel.device)
            _capi.check(_capi.lib.ab_generator_forward(h, _capi.ptr(mel), B, T, _capi.shape_array(mel.stride()),
                                                       _capi.ptr(out), ws, need, _capi.stream_ptr()),
                        "ab_generator_forward")
        return out


def _effective_weight(conv):
    """weight of a (possibly weight-normed) conv: w = g * v / ||v|| over all dims but 0 (torch.nn.utils.weight_norm)."""
    if hasattr(conv, "weight_g"):
        v, g = conv.weight_v.detach(), conv.weight_g.detach()
        return v * (g / v.flatten(1).norm(dim=1).view(-1, 1, 1))
    return conv.weight.detach()


class APNet(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        hp, pre = cfg.model.apnet, cfg.preprocess
        self.ASP_num_kernels = len(hp.ASP_resblock_kernel_sizes)
        self.PSP_num_kernels = len(hp.PSP_resblock_kernel_sizes)
        bins = pre.n_fft // 2 + 1

        def conv(cin, cout, k):
            return weight_norm(nn.Conv1d(cin, cout, k, 1, padding=get_padding(k, 1)))

        self.ASP_input_conv = conv(pre.n_mel, hp.ASP_channel, hp.ASP_input_conv_kernel_size)
        self.PSP_input_conv = conv(pre.n_mel, hp.PSP_channel, hp.PSP_input_conv_kernel_size)
        self.ASP_ResNet = nn.ModuleList(ConvBlock(cfg, hp.ASP_channel, k, d, "1")
                                        for k, d in zip(hp.ASP_resblock_kernel_sizes, hp.ASP_resblock_dilation_sizes))
        self.PSP_ResNet = nn.ModuleList(ConvBlock(cfg, hp.PSP_channel, k, d, "1")
                                        for k, d in zip(hp.PSP_resblock_kernel_sizes, hp.PSP_resblock_dilation_sizes))
        self.ASP_output_conv = conv(hp.ASP_channel, bins, hp.ASP_output_conv_kernel_size)
        self.PSP_output_R_conv = conv(hp.PSP_channel, bins, hp.PSP_output_R_conv_kernel_size)
        self.PSP_output_I_conv = conv(hp.PSP_channel, bins, hp.PSP_output_I_conv_kernel_size)
        if hp.PSP_output_R_conv_kernel_size != hp.PSP_output_I_conv_kernel_size:
            raise NotImplementedError("amphion_b200: the R and I output convolutions run as one stacked convolution "
                                      "(equal kernel sizes, as in egs/vocoder/gan/apnet/exp_config.json)")
        self.iSTFT = ISTFT(pre.n_fft, hop_length=pre.hop_size, win_length=pre.win_size)
        self.ASP_output_conv.apply(init_weights)
        self.PSP_output_R_conv.apply(init_weights)
        self.PSP_output_I_conv.apply(init_weights)
        self.precision = DEFAULT_PRECISION
        self._trunks = {"ASP": _Trunk(self, "ASP"), "PSP": _Trunk(self, "PSP")}   # plain dict: not submodules
        self._window = {}
        self.last_launches = 0

    # ---- the trunks' view of the parameters -------------------------------------------------
    def _trunk_tensors(self, s):
        out = {}
        inp = getattr(self, f"{s}_input_conv")
        out["conv_pre.weight"], out["conv_pre.bias"] = _effective_weight(inp), inp.bias.detach()
        for j, blk in enumerate(getattr(self, f"{s}_ResNet")):
            for name, group in (("convs1", blk.convs1), ("convs2", blk.convs2)):
                for p, c in enumerate(group):
                    out[f"resblocks.{j}.{name}.{p}.weight"] = _effective_weight(c)
                    out[f"resblocks.{j}.{name}.{p}.bias"] = c.bias.detach()
        if s == "ASP":
            out["conv_post.weight"], out["conv_post.bias"] = _effective_weight(self.ASP_output_conv), self.ASP_output_conv.bias.detach()
        else:   # R rows first, then I: one convolution instead of two reads of the phase stream
            out["conv_post.weight"] = torch.cat([_effective_weight(self.PSP_output_R_conv), _effective_weight(self.PSP_output_I_conv)], 0)
            out["conv_post.bias"] = torch.cat([self.PSP_output_R_conv.bias.detach(), self.PSP_output_I_conv.bias.detach()], 0)
        return out

    def remove_weight_norm(self):
        for c in (self.ASP_input_conv, self.PSP_input_conv, self.ASP_output_conv, self.PSP_output_R_conv, self.PSP_output_I_conv):
            remove_weight_norm(c)
        for blk in list(self.ASP_ResNet) + list(self.PSP_ResNet):
            blk.remove_weight_norm()

    def forward(self, mel):
        _capi.require_cuda(mel, "APNet.forward")
        if mel.dim() != 3 or mel.shape[1] != int(self.cfg.preprocess.n_mel):
            raise ValueError(f"expected mel of shape [B, {self.cfg.preprocess.n_mel}, T], got {tuple(mel.shape)}")
        B, _, T = mel.shape
        bins = int(self.cfg.preprocess.n_fft) // 2 + 1
        for t in self._trunks.values():
            t.precision = self.precision
        logamp = self._trunks["ASP"].run(mel)                       # [B, bins, T]
        ri = self._trunks["PSP"].run(mel)                           # [B, 2*bins, T]: R | I
        self.last_launches = self._trunks["ASP"].last_launches + self._trunks["PSP"].last_launches + 3
        pha, rea, imag = (torch.empty_like(logamp) for _ in range(3))
        spec = torch.empty(B * T, bins, 2, dtype=torch.float32, device=mel.device)
        with torch.cuda.device(mel.device):
            if B == 1:
                r_ptr, i_ptr = _capi.ptr(ri), C.c_void_p(ri.data_ptr() + bins * T * 4)
            else:   # R and I of one utterance are adjacent, not the batch: split once (a view would need a row stride)
                r, i = ri[:, :bins].contiguous(), ri[:, bins:].contiguous()
                r_ptr, i_ptr = _capi.ptr(r), _capi.ptr(i)
            _capi.check(_capi.lib.ab_spectral_head_forward(_capi.ptr(logamp), r_ptr, i_ptr, B, bins, T, 0.0, _capi.ptr(pha),
                                                           _capi.ptr(rea), _capi.ptr(imag), _capi.ptr(spec), _capi.stream_ptr()),
                        "ab_spectral_head_forward")
        key = (int(self.cfg.preprocess.win_size), str(mel.device))
        if key not in self._window:
            self._window[key] = torch.hann_window(self.cfg.preprocess.win_size).to(mel.device)
        audio = self.iSTFT.forward_interleaved(spec, B, T, self._window[key])
        return logamp, pha, rea, imag, audio.unsqueeze(1)

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)
        for t in getattr(self, "_trunks", {}).values():
            t.invalidate()
        return out

    def __getstate__(self):
        state = self.__dict__.copy()
        state["_trunks"], state["_window"] = None, {}
        return state

    def __setstate__(self, state):
        self.__dict__.update(state)
        self._trunks = {"ASP": _Trunk(self, "ASP"), "PSP": _Trunk(self, "PSP")}


class ISTFTHead(nn.Module):
    """Vocos' iSTFT head (models/codec/kmeans/vocos.py:313-361): ``out = Linear(dim, n_fft + 2)``; the first half of
    the outputs is the log-magnitude (exp, clipped at 1e2), the second half the phase; S = mag (cos p + i sin p);
    ISTFT with "same" padding.  x [B, L, H] -> audio [B, L * hop].  The linear layer is a library GEMM; magnitude /
    phase -> spectrum and the inverse STFT are the native kernels APNet uses."""

    def __init__(self, dim: int, n_fft: int, hop_length: int, padding: str = "same"):
        super().__init__()
        self.out = nn.Linear(dim, n_fft + 2)
        self.istft = ISTFT(n_fft=n_fft, hop_length=hop_length, win_length=n_fft, padding=padding)
        self.register_buffer("window", torch.hann_window(n_fft), persistent=False)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        _capi.require_cuda(x, "ISTFTHead.forward")
        y = self.out(x).transpose(1, 2).contiguous().float()        # [B, n_fft + 2, L]
        B, two_bins, L = y.shape
        bins = two_bins // 2
        spec = torch.empty(B * L, bins, 2, dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            if B == 1:
                m_ptr, p_ptr = _capi.ptr(y), C.c_void_p(y.data_ptr() + bins * L * 4)
            else:
                mag, pha = y[:, :bins].contiguous(), y[:, bins:].contiguous()
                m_ptr, p_ptr = _capi.ptr(mag), _capi.ptr(pha)
            _capi.check(_capi.lib.ab_spectral_head_forward(m_ptr, p_ptr, None, B, bins, L, 1e2, None, None, None,
                                                           _capi.ptr(spec), _capi.stream_ptr()), "ab_spectral_head_forward")
        return self.istft.forward_interleaved(spec, B, L, self.window)
