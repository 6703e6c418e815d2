"""Shared host logic of the native GAN generators (HiFi-GAN / BigVGAN).

The module keeps the reference's parameter names and weight-norm decomposition
(``weight_g`` / ``weight_v``) so reference checkpoints load unchanged
(SURVEY.md §10); ``forward`` hands raw device pointers to the C ABI.
"""
from __future__ import annotations

import ctypes as C
import os

import torch
from torch import nn
from torch.nn.utils import remove_weight_norm, weight_norm

from .. import _capi

LRELU_SLOPE = 0.1
DEFAULT_PRECISION = os.environ.get("AMPHION_B200_PRECISION", "tc_f16")


def get_padding(kernel_size, dilation=1):
    return int((kernel_size * dilation - dilation) / 2)


def init_weights(m, mean=0.0, std=0.01):
    if m.__class__.__name__.find("Conv") != -1:
        m.weight.data.normal_(mean, std)


def wn_conv(cin, cout, k, dilation=1):
    return weight_norm(nn.Conv1d(cin, cout, k, 1, dilation=dilation, padding=get_padding(k, dilation)))


class ConvBlock(nn.Module):
    """Parameter holder for ResBlock1/2 and AMPBlock1/2 (hifigan.py:17-148,
    bigvgan.py:23-229): ``convs1``/``convs2`` (type "1") or ``convs`` (type "2"),
    plus ``activations`` for the AMP variants."""

    def __init__(self, cfg, channels, kernel_size, dilation, block_type, make_activation=None):
        super().__init__()
        self.cfg = cfg
        self.block_type = str(block_type)
        if self.block_type == "1":
            self.convs1 = nn.ModuleList([wn_conv(channels, channels, kernel_size, d) for d in dilation])
            self.convs1.apply(init_weights)
            self.convs2 = nn.ModuleList([wn_conv(channels, channels, kernel_size, 1) for _ in dilation])
            self.convs2.apply(init_weights)
            self.num_layers = 2 * len(dilation)
        else:
            self.convs = nn.ModuleList([wn_conv(channels, channels, kernel_size, d) for d in dilation])
            self.convs.apply(init_weights)
            self.num_layers = len(dilation)
        if make_activation is not None:
            self.activations = nn.ModuleList([make_activation(channels) for _ in range(self.num_layers)])

    def _all_convs(self):
        if self.block_type == "1":
            return list(self.convs1) + list(self.convs2)
        return list(self.convs)

    def remove_weight_norm(self):
        for l in self._all_convs():
            remove_weight_norm(l)

    def forward(self, x):  # the blocks only run fused inside the generator kernels
        raise RuntimeError("amphion_b200: residual blocks execute inside the generator's CUDA pipeline; "
                           "call the generator's forward()")


class NativeGenerator(nn.Module):
    """Base class: owns the C-ABI handle, the packed-parameter arena and the workspace."""

    kind = None       # "hifigan" | "bigvgan" | "nsfhifigan"
    hp_key = None     # cfg.model.<hp_key>

    def __init__(self):
        super().__init__()
        self._handle = None
        self._arena = None
        self._arena_key = None
        self._workspace = None
        self.precision = DEFAULT_PRECISION
        self.last_launches = 0

    # ---- config -> C struct -------------------------------------------------
    def _hp(self):
        return getattr(self.cfg.model, self.hp_key)

    def _c_config(self):
        hp = self._hp()
        c = _capi.GeneratorConfig()
        c.kind = {"hifigan": _capi.GEN_HIFIGAN, "bigvgan": _capi.GEN_BIGVGAN, "nsfhifigan": _capi.GEN_NSFHIFIGAN}[self.kind]
        c.n_mel = int(self.cfg.preprocess.n_mel)
        c.upsample_initial_channel = int(hp.upsample_initial_channel)
        rates, ksz = list(hp.upsample_rates), list(hp.upsample_kernel_sizes)
        rks, rds = list(hp.resblock_kernel_sizes), [list(d) for d in hp.resblock_dilation_sizes]
        if len(rates) > _capi.AB_MAX_STAGES or len(rks) > _capi.AB_MAX_KERNELS or \
                any(len(d) > _capi.AB_MAX_DILATIONS for d in rds):
            raise ValueError("amphion_b200: too many stages / kernels / dilations for the native generator")
        c.num_upsamples = len(rates)
        for i, (u, k) in enumerate(zip(rates, ksz)):
            c.upsample_rates[i], c.upsample_kernel_sizes[i] = int(u), int(k)
        c.resblock = 1 if str(hp.resblock) == "1" else 2
        c.num_kernels = len(rks)
        for j, (k, ds) in enumerate(zip(rks, rds)):
            c.resblock_kernel_sizes[j] = int(k)
            c.num_dilations[j] = len(ds)
            for p, d in enumerate(ds):
                c.resblock_dilation_sizes[j][p] = int(d)
        if self.kind == "bigvgan":
            c.activation = _capi.ACT_SNAKE if hp.activation == "snake" else _capi.ACT_SNAKEBETA
            c.snake_logscale = int(bool(hp.snake_logscale))
        else:
            c.activation = _capi.ACT_LRELU
        c.gin_channels = int(getattr(self, "gin_channels", 0))
        c.conv_post_no_bias = int(getattr(self, "conv_post_no_bias", False))
        return c

    # ---- parameter packing ---------------------------------------------------
    def _param_key(self, device):
        ts = list(self.parameters()) + list(self.buffers())
        return (str(device), self.precision, tuple((t.data_ptr(), t._version) for t in ts))

    def _ensure_handle(self):
        if self._handle is None:
            h = C.c_void_p()
            cfg = self._c_config()
            _capi.check(_capi.lib.ab_generator_create(C.byref(cfg), C.byref(h)), "ab_generator_create")
            self._handle = h
        return self._handle

    def _sync_params(self, device):
        key = self._param_key(device)
        if key == self._arena_key:
            return
        if self.precision not in _capi.PRECISIONS:
            raise ValueError(f"amphion_b200: unknown precision '{self.precision}' (use {list(_capi.PRECISIONS)})")
        h = self._ensure_handle()
        lib = _capi.lib
        need = lib.ab_generator_param_bytes(h)
        self._arena = torch.empty(need + 256, dtype=torch.uint8, device=device)
        base = (self._arena.data_ptr() + 255) // 256 * 256
        _capi.check(lib.ab_generator_bind_params(h, C.c_void_p(base), need), "ab_generator_bind_params")
        st = _capi.stream_ptr()
        sd = {k: v.detach() for k, v in list(self.named_parameters()) + list(self.named_buffers())}
        keep = []
        for i in range(lib.ab_generator_num_tensors(h)):
            name = lib.ab_generator_tensor_name(h, i).decode()
            if name in sd:
                t = sd[name].to(device=device, dtype=torch.float32).contiguous()
                keep.append(t)
                _capi.check(lib.ab_generator_load_tensor(h, name.encode(), _capi.ptr(t), _capi.shape_array(t.shape),
                                                         t.dim(), st), f"load_tensor({name})")
            elif name.endswith(".weight") and name + "_v" in sd:
                v = sd[name + "_v"].to(device=device, dtype=torch.float32).contiguous()
                g = sd[name + "_g"].to(device=device, dtype=torch.float32).contiguous()
                keep += [v, g]
                _capi.check(lib.ab_generator_load_weight_norm(h, name.encode(), _capi.ptr(g), _capi.ptr(v),
                                                              _capi.shape_array(v.shape), v.dim(), st),
                            f"load_weight_norm({name})")
            else:
                raise RuntimeError(f"amphion_b200: the module has no parameter for '{name}'")
        _capi.check(lib.ab_generator_finalize(h, _capi.PRECISIONS[self.precision], st), "ab_generator_finalize")
        self._arena_key = key
        del keep  # stream-ordered: the caching allocator keeps the blocks alive until the copies ran

    # ---- forward ---------------------------------------------------------------
    def forward(self, x, out=None, tail_events=None):
        """mel [B, n_mel, T] (any strides) -> wav [B, 1, T*hop], fp32, same device.

        ``out`` (optional, beyond the reference signature): a contiguous fp32 [B, 1, T*hop] tensor to write into
        (e.g. a slice of a gathered batch).  ``tail_events``: a list of ``torch.cuda.Event``; the last layer runs in
        ``len(tail_events)`` batch chunks and event i is recorded when utterances [B*i/n, B*(i+1)/n) are complete."""
        return self._forward_native(x, out=out, tail_events=tail_events)

    def _forward_native(self, x, g=None, out=None, tail_events=None, out_samples=None):
        """``g`` [B, gin_channels] (HiFiGAN_vits conditioning) or None."""
        _capi.require_cuda(x, f"{type(self).__name__}.forward")
        if x.dim() != 3 or x.shape[1] != int(self.cfg.preprocess.n_mel):
            raise ValueError(f"expected mel of shape [B, {self.cfg.preprocess.n_mel}, T], got {tuple(x.shape)}")
        if x.dtype != torch.float32:
            x = x.float()
        B, _, T = x.shape
        if B == 0 or T == 0:
            raise ValueError("amphion_b200: empty mel batch")
        with torch.cuda.device(x.device):
            self._sync_params(x.device)
            lib, h = _capi.lib, self._handle
            hop = 1
            for u in self._hp().upsample_rates:
                hop *= int(u)
            need = lib.ab_generator_workspace_bytes(h, B, T)
            if self._workspace is None or self._workspace.numel() < need + 256 or self._workspace.device != x.device:
                self._workspace = None
                self._workspace = torch.empty(need + 256, dtype=torch.uint8, device=x.device)
            wbase = (self._workspace.data_ptr() + 255) // 256 * 256
            n_out = T * hop if out_samples is None else int(out_samples)
            if out is None:
                wav = torch.empty(B, 1, n_out, dtype=torch.float32, device=x.device)
            else:
                if (tuple(out.shape) != (B, 1, n_out) or out.dtype != torch.float32 or out.device != x.device
                        or not out.is_contiguous()):
                    raise ValueError(f"out must be a contiguous fp32 [{B}, 1, {n_out}] tensor on {x.device}")
                wav = out
            if tail_events:
                for ev in tail_events:
                    ev.record()   # creates the underlying cudaEvent_t (torch creates it lazily); re-recorded below
                arr = (C.c_void_p * len(tail_events))(*[C.c_void_p(ev.cuda_event) for ev in tail_events])
                _capi.check(lib.ab_generator_set_tail_events(h, arr, len(tail_events)), "ab_generator_set_tail_events")
            strides = _capi.shape_array(x.stride())
            if g is None:
                _capi.check(lib.ab_generator_forward(h, _capi.ptr(x), B, T, strides, _capi.ptr(wav), C.c_void_p(wbase),
                                                     need, _capi.stream_ptr()), "ab_generator_forward")
            else:
                _capi.check(lib.ab_generator_forward_cond(h, _capi.ptr(x), B, T, strides, _capi.ptr(g), g.stride(0),
                                                          _capi.ptr(wav), C.c_void_p(wbase), need, _capi.stream_ptr()),
                            "ab_generator_forward_cond")
            self.last_launches = lib.ab_generator_last_launches(h)
        return wav

    def set_option(self, key: str, value: int):
        """Execution-plan knob of the C ABI (`ab_generator_set_option`), e.g. ("nsf_source_frames", n)."""
        _capi.check(_capi.lib.ab_generator_set_option(self._ensure_handle(), key.encode(), int(value)), "set_option")

    # ---- per-kernel-class device timing (bench.py roofline) ------------------------
    def set_profiling(self, enable: bool):
        _capi.check(_capi.lib.ab_generator_set_profiling(self._ensure_handle(), int(enable)), "set_profiling")

    def get_profile(self):
        """{class: dict(launches, ms, flops, bytes)} accumulated since the last call (synchronises)."""
        arr = (_capi.ProfileEntry * 8)()
        n = C.c_int32(0)
        _capi.check(_capi.lib.ab_generator_get_profile(self._ensure_handle(), arr, 8, C.byref(n)), "get_profile")
        return {arr[i].name.decode(): dict(launches=arr[i].launches, ms=arr[i].ms, flops=arr[i].flops,
                                           bytes=arr[i].bytes) for i in range(n.value)}

    # ---- native state is derived: never copied / pickled, rebuilt on the next forward ---------------
    def invalidate(self):
        """Drop the packed weight arena so the next forward re-reads the parameters.  Needed after edits that do
        not bump a tensor's version counter (``p.data.copy_()``, ``m.weight.data.normal_()``); ``load_state_dict``,
        ``.to()`` / ``.cuda()`` and ``remove_weight_norm`` call it themselves."""
        self._arena_key = None

    def load_state_dict(self, *args, **kwargs):
        out = super().load_state_dict(*args, **kwargs)
        self.invalidate()
        return out

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)
        self.invalidate()
        return out

    def __getstate__(self):
        state = self.__dict__.copy()
        for k in ("_handle", "_arena", "_arena_key", "_workspace"):   # ctypes handle / device scratch: not state
            state[k] = None
        return state

    def __deepcopy__(self, memo):
        import copy
        cls = self.__class__
        new = cls.__new__(cls)
        memo[id(self)] = new
        for k, v in self.__getstate__().items():
            setattr(new, k, copy.deepcopy(v, memo))
        return new

    def __del__(self):
        try:
            if self._handle is not None:
                _capi.lib.ab_generator_destroy(self._handle)
        except Exception:
            pass
