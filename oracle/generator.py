"""Oracle: HiFi-GAN / BigVGAN generator forward, restated on CPU.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Parameters are a plain ``dict[str, np.ndarray]`` keyed by the reference
state-dict names (SURVEY.md §10): weight-normed convs appear either as
``<name>.weight_g`` + ``<name>.weight_v`` or already folded as ``<name>.weight``.

Two sets of primitives are provided:
  * ``*_np``  : pure numpy loops/einsum — slow, for small cases, no torch.
  * default   : the same maths through ``torch.nn.functional`` on CPU fp32,
                used for speed; cross-checked against ``*_np`` in
                tests/test_oracle.py.
All citations are to files of the reference (open-mmlab/Amphion).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

LRELU_SLOPE = 0.1  # models/vocoders/gan/generator/hifigan.py:14, bigvgan.py:17


# --------------------------------------------------------------------------
# parameters
# --------------------------------------------------------------------------
def fold_weight_norm(v: np.ndarray, g: np.ndarray) -> np.ndarray:
    """w = g * v / ||v||, norm over every dim except 0 (old-style
    torch.nn.utils.weight_norm, dim=0; used by every conv in hifigan.py:157-199
    and bigvgan.py:241-303).  For ConvTranspose1d dim 0 is C_in (SURVEY Q6)."""
    v64 = v.astype(np.float32)
    n = np.sqrt((v64 * v64).reshape(v.shape[0], -1).sum(axis=1, dtype=np.float32))
    n = n.reshape((-1,) + (1,) * (v.ndim - 1))
    return (v64 * (g.astype(np.float32) / n)).astype(np.float32)


def get_weight(params: dict, name: str) -> np.ndarray:
    if name + ".weight" in params:
        return np.asarray(params[name + ".weight"], dtype=np.float32)
    return fold_weight_norm(params[name + ".weight_v"], params[name + ".weight_g"])


def get_padding(kernel_size: int, dilation: int = 1) -> int:
    # modules/vocoder_blocks/gan_utils.py:12-13
    return int((kernel_size * dilation - dilation) / 2)


# --------------------------------------------------------------------------
# primitives — pure numpy
# --------------------------------------------------------------------------
def conv1d_np(x, w, b, dilation=1, padding=0):
    """y[n,co,t] = b[co] + sum_ci sum_j w[co,ci,j] * xpad[n,ci,t+j*dilation]."""
    n, cin, t = x.shape
    cout, _, k = w.shape
    xp = np.zeros((n, cin, t + 2 * padding), np.float32)
    xp[:, :, padding:padding + t] = x
    tout = t + 2 * padding - dilation * (k - 1)
    y = np.zeros((n, cout, tout), np.float32)
    for j in range(k):
        y += np.einsum("oc,nct->not", w[:, :, j], xp[:, :, j * dilation:j * dilation + tout],
                       dtype=np.float32)
    if b is not None:
        y += b[None, :, None]
    return y


def conv_transpose1d_np(x, w, b, stride, padding):
    """ConvTranspose1d (hifigan.py:176-186): w is [C_in, C_out, k];
    full[n,co,s*stride+j] += x[n,ci,s]*w[ci,co,j]; out = full[padding : padding+T*stride]
    (k - stride even, so T_out = T*stride)."""
    n, cin, t = x.shape
    _, cout, k = w.shape
    full = np.zeros((n, cout, (t - 1) * stride + k), np.float32)
    for j in range(k):
        full[:, :, j:j + (t - 1) * stride + 1:stride] += np.einsum(
            "co,nct->not", w[:, :, j], x, dtype=np.float32)
    tout = (t - 1) * stride - 2 * padding + k
    y = full[:, :, padding:padding + tout]
    if b is not None:
        y = y + b[None, :, None]
    return y.astype(np.float32)


def leaky_relu_np(x, slope):
    return np.where(x >= 0, x, x * np.float32(slope)).astype(np.float32)


def snake_np(x, alpha, beta, logscale):
    """modules/activation_functions/snake.py:51-61 (Snake: beta is alpha) and
    :110-122 (SnakeBeta): x + 1/(b+1e-9) * sin(x*a)^2, a/b = exp(.) if logscale."""
    a = alpha.astype(np.float32)[None, :, None]
    b = beta.astype(np.float32)[None, :, None]
    if logscale:
        a = np.exp(a)
        b = np.exp(b)
    return (x + (np.float32(1.0) / (b + np.float32(1e-9))) * np.sin(x * a) ** 2).astype(np.float32)


def upsample2x_np(x, f):
    """modules/anti_aliasing/resample.py:36-45 with ratio=2, kernel 12, in the
    closed form of SURVEY §8 a10: replicate-pad 5/5, depthwise transposed conv
    stride 2, times 2, crop 15/15."""
    n, c, t = x.shape
    f = np.asarray(f, np.float32).reshape(-1)
    assert f.size == 12
    idx = np.clip(np.arange(-3, t + 3), 0, t - 1)  # xhat[q-3 .. q+2+...]
    xh = x[:, :, idx]  # xh[..., i] = xhat[i-3]
    u = np.zeros((n, c, 2 * t), np.float32)
    for m in range(6):
        u[:, :, 0::2] += f[11 - 2 * m] * xh[:, :, m:m + t]          # xhat[q-3+m]
        u[:, :, 1::2] += f[10 - 2 * m] * xh[:, :, m + 1:m + 1 + t]  # xhat[q-2+m]
    return (np.float32(2.0) * u).astype(np.float32)


def downsample2x_np(v, f):
    """modules/anti_aliasing/filter.py:92-99 via resample.py:62-65: replicate
    pad 5 left / 6 right, depthwise conv stride 2 (SURVEY §8 a11)."""
    n, c, t2 = v.shape
    f = np.asarray(f, np.float32).reshape(-1)
    t = t2 // 2
    y = np.zeros((n, c, t), np.float32)
    base = 2 * np.arange(t) - 5
    for j in range(12):
        y += f[j] * v[:, :, np.clip(base + j, 0, t2 - 1)]
    return y


def activation1d_np(x, alpha, beta, logscale, f_up, f_down):
    # modules/anti_aliasing/act.py:31-36
    return downsample2x_np(snake_np(upsample2x_np(x, f_up), alpha, beta, logscale), f_down)


# --------------------------------------------------------------------------
# primitives — CPU torch (same maths, used for speed)
# --------------------------------------------------------------------------
def _t(a):
    return a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))


def conv1d(x, w, b, dilation=1, padding=0):
    return F.conv1d(_t(x), _t(w), None if b is None else _t(b), dilation=dilation, padding=padding)


def conv_transpose1d(x, w, b, stride, padding):
    return F.conv_transpose1d(_t(x), _t(w), None if b is None else _t(b), stride=stride, padding=padding)


def snake(x, alpha, beta, logscale):
    a = _t(alpha)[None, :, None]
    b = _t(beta)[None, :, None]
    if logscale:
        a, b = torch.exp(a), torch.exp(b)
    return x + (1.0 / (b + 1e-9)) * torch.sin(x * a) ** 2


def upsample2x(x, f):
    c = x.shape[1]
    fk = _t(f).reshape(1, 1, 12).expand(c, -1, -1)
    xp = F.pad(x, (5, 5), mode="replicate")
    y = 2 * F.conv_transpose1d(xp, fk, stride=2, groups=c)
    return y[..., 15:-15]


def downsample2x(v, f):
    c = v.shape[1]
    fk = _t(f).reshape(1, 1, 12).expand(c, -1, -1)
    return F.conv1d(F.pad(v, (5, 6), mode="replicate"), fk, stride=2, groups=c)


def activation1d(x, alpha, beta, logscale, f_up, f_down):
    return downsample2x(snake(upsample2x(x, f_up), alpha, beta, logscale), f_down)


# --------------------------------------------------------------------------
# anti-alias filter (only used when a state dict carries no filter buffers)
# --------------------------------------------------------------------------
def kaiser_sinc_filter12() -> np.ndarray:
    """modules/anti_aliasing/filter.py:30-61 at cutoff 0.25, half_width 0.3,
    kernel 12 (the only instance on the path: resample.py:28-31, :54-59)."""
    cutoff, half_width, ks = 0.25, 0.3, 12
    half = ks // 2
    delta_f = 4 * half_width
    a = 2.285 * (half - 1) * np.pi * delta_f + 7.95
    if a > 50.0:
        beta = 0.1102 * (a - 8.7)
    elif a >= 21.0:
        beta = 0.5842 * (a - 21) ** 0.4 + 0.07886 * (a - 21.0)
    else:
        beta = 0.0
    window = torch.kaiser_window(ks, beta=beta, periodic=False)
    time = torch.arange(-half, half) + 0.5
    filt = 2 * cutoff * window * torch.sinc(2 * cutoff * time)
    filt = filt / filt.sum()
    return filt.numpy().astype(np.float32)


# --------------------------------------------------------------------------
# blocks
# --------------------------------------------------------------------------
def _bias(params, name):
    return np.asarray(params[name + ".bias"], np.float32)


def resblock1(params, prefix, x, k, dilations):
    """hifigan.py:93-100."""
    for p, d in enumerate(dilations):
        xt = F.leaky_relu(x, LRELU_SLOPE)
        xt = conv1d(xt, get_weight(params, f"{prefix}.convs1.{p}"), _bias(params, f"{prefix}.convs1.{p}"),
                    dilation=d, padding=get_padding(k, d))
        xt = F.leaky_relu(xt, LRELU_SLOPE)
        xt = conv1d(xt, get_weight(params, f"{prefix}.convs2.{p}"), _bias(params, f"{prefix}.convs2.{p}"),
                    dilation=1, padding=get_padding(k, 1))
        x = xt + x
    return x


def resblock2(params, prefix, x, k, dilations):
    """hifigan.py:139-144."""
    for p, d in enumerate(dilations):
        xt = F.leaky_relu(x, LRELU_SLOPE)
        xt = conv1d(xt, get_weight(params, f"{prefix}.convs.{p}"), _bias(params, f"{prefix}.convs.{p}"),
                    dilation=d, padding=get_padding(k, d))
        x = xt + x
    return x


def _act(params, prefix, x, kind, logscale):
    """One Activation1d(Snake|SnakeBeta) module, state-dict prefix e.g.
    ``resblocks.3.activations.2`` (bigvgan.py:106-131, act.py:14-36)."""
    alpha = np.asarray(params[prefix + ".act.alpha"], np.float32)
    beta = np.asarray(params[prefix + ".act.beta"], np.float32) if kind == "snakebeta" else alpha
    f_up = params.get(prefix + ".upsample.filter")
    f_dn = params.get(prefix + ".downsample.lowpass.filter")
    if f_up is None:
        f_up = kaiser_sinc_filter12()
    if f_dn is None:
        f_dn = kaiser_sinc_filter12()
    return activation1d(x, alpha, beta, logscale, np.asarray(f_up).reshape(-1), np.asarray(f_dn).reshape(-1))


def ampblock1(params, prefix, x, k, dilations, kind, logscale):
    """bigvgan.py:137-146: acts1 = activations[::2], acts2 = activations[1::2]."""
    for p, d in enumerate(dilations):
        xt = _act(params, f"{prefix}.activations.{2 * p}", x, kind, logscale)
        xt = conv1d(xt, get_weight(params, f"{prefix}.convs1.{p}"), _bias(params, f"{prefix}.convs1.{p}"),
                    dilation=d, padding=get_padding(k, d))
        xt = _act(params, f"{prefix}.activations.{2 * p + 1}", xt, kind, logscale)
        xt = conv1d(xt, get_weight(params, f"{prefix}.convs2.{p}"), _bias(params, f"{prefix}.convs2.{p}"),
                    dilation=1, padding=get_padding(k, 1))
        x = xt + x
    return x


def ampblock2(params, prefix, x, k, dilations, kind, logscale):
    """bigvgan.py:222-228."""
    for p, d in enumerate(dilations):
        xt = _act(params, f"{prefix}.activations.{p}", x, kind, logscale)
        xt = conv1d(xt, get_weight(params, f"{prefix}.convs.{p}"), _bias(params, f"{prefix}.convs.{p}"),
                    dilation=d, padding=get_padding(k, d))
        x = xt + x
    return x


# --------------------------------------------------------------------------
# generators.  ``hp`` is a plain dict of the cfg.model.{hifigan,bigvgan} keys.
# --------------------------------------------------------------------------
def hifigan_forward(params, hp, mel, return_stages=False):
    """hifigan.py:203-219.  mel [B, n_mel, T] -> wav [B, 1, T*prod(rates)]."""
    x = _t(np.asarray(mel, np.float32)) if not isinstance(mel, torch.Tensor) else mel.float()
    stages = []
    with torch.no_grad():
        x = conv1d(x, get_weight(params, "conv_pre"), _bias(params, "conv_pre"), padding=3)
        nk = len(hp["resblock_kernel_sizes"])
        rb = resblock1 if str(hp["resblock"]) == "1" else resblock2
        for i, (u, k) in enumerate(zip(hp["upsample_rates"], hp["upsample_kernel_sizes"])):
            x = F.leaky_relu(x, LRELU_SLOPE)
            x = conv_transpose1d(x, get_weight(params, f"ups.{i}"), _bias(params, f"ups.{i}"),
                                 stride=u, padding=(k - u) // 2)
            xs = None
            for j in range(nk):
                r = rb(params, f"resblocks.{i * nk + j}", x, hp["resblock_kernel_sizes"][j],
                       hp["resblock_dilation_sizes"][j])
                xs = r if xs is None else xs + r
            x = xs / nk
            stages.append(x.numpy().copy())
        x = F.leaky_relu(x)  # default slope 0.01 (hifigan.py:215, SURVEY Q1)
        x = conv1d(x, get_weight(params, "conv_post"), _bias(params, "conv_post"), padding=3)
        x = torch.tanh(x)
    out = x.numpy()
    return (out, stages) if return_stages else out


def bigvgan_forward(params, hp, mel, return_stages=False):
    """bigvgan.py:313-331."""
    x = _t(np.asarray(mel, np.float32)) if not isinstance(mel, torch.Tensor) else mel.float()
    kind, logscale = hp["activation"], bool(hp["snake_logscale"])
    stages = []
    with torch.no_grad():
        x = conv1d(x, get_weight(params, "conv_pre"), _bias(params, "conv_pre"), padding=3)
        nk = len(hp["resblock_kernel_sizes"])
        rb = ampblock1 if str(hp["resblock"]) == "1" else ampblock2
        for i, (u, k) in enumerate(zip(hp["upsample_rates"], hp["upsample_kernel_sizes"])):
            # no activation before the transposed conv (bigvgan.py:316-318, SURVEY Q2)
            x = conv_transpose1d(x, get_weight(params, f"ups.{i}.0"), _bias(params, f"ups.{i}.0"),
                                 stride=u, padding=(k - u) // 2)
            xs = None
            for j in range(nk):
                r = rb(params, f"resblocks.{i * nk + j}", x, hp["resblock_kernel_sizes"][j],
                       hp["resblock_dilation_sizes"][j], kind, logscale)
                xs = r if xs is None else xs + r
            x = xs / nk
            stages.append(x.numpy().copy())
        x = _act(params, "activation_post", x, kind, logscale)
        x = conv1d(x, get_weight(params, "conv_post"), _bias(params, "conv_post"), padding=3)
        x = torch.tanh(x)
    out = x.numpy()
    return (out, stages) if return_stages else out


def hifigan_vits_forward(params, hp, x, g=None):
    """HiFiGAN_vits.forward (hifigan.py:427-445): plain conv_pre, ``x + cond(g)`` with g [B, gin, 1], HiFi-GAN
    stages (the residual blocks are called without a mask, :437-441), bias-free conv_post."""
    x = _t(np.asarray(x, np.float32)) if not isinstance(x, torch.Tensor) else x.float()
    with torch.no_grad():
        x = conv1d(x, get_weight(params, "conv_pre"), _bias(params, "conv_pre"), padding=3)
        if g is not None:
            x = x + conv1d(_t(np.asarray(g, np.float32)), get_weight(params, "cond"), _bias(params, "cond"))
        nk = len(hp["resblock_kernel_sizes"])
        rb = resblock1 if str(hp["resblock"]) == "1" else resblock2
        for i, (u, k) in enumerate(zip(hp["upsample_rates"], hp["upsample_kernel_sizes"])):
            x = F.leaky_relu(x, LRELU_SLOPE)
            x = conv_transpose1d(x, get_weight(params, f"ups.{i}"), _bias(params, f"ups.{i}"),
                                 stride=u, padding=(k - u) // 2)
            xs = None
            for j in range(nk):
                r = rb(params, f"resblocks.{i * nk + j}", x, hp["resblock_kernel_sizes"][j],
                       hp["resblock_dilation_sizes"][j])
                xs = r if xs is None else xs + r
            x = xs / nk
        x = F.leaky_relu(x)
        x = conv1d(x, get_weight(params, "conv_post"), None, padding=3)
        x = torch.tanh(x)
    return x.numpy()


def nsfhifigan_forward(params, hp, mel, f0, return_stages=False):
    """nsfhifigan.py:262-283.  ``har_source`` (:263) is [B, 1, T_f0 * upp]; ``noise_convs[i]`` (:223-236) maps it
    to length floor((L + 2*(s//2) - 2s) / s) + 1 with s = prod(rates[i+1:]) (kernel 1 for the last stage), and
    its VALUES are dropped by ``x_source = x[:, :, :length]`` (:269) — so only that length is restated here
    (the source itself draws torch.rand / torch.randn, sine_excitation.py:42,84, and cannot be a fixture)."""
    x = _t(np.asarray(mel, np.float32)) if not isinstance(mel, torch.Tensor) else mel.float()
    rates = [int(u) for u in hp["upsample_rates"]]
    upp = int(np.prod(rates))
    src_len = int(np.asarray(f0).shape[1]) * upp
    stages = []
    with torch.no_grad():
        x = conv1d(x, get_weight(params, "conv_pre"), _bias(params, "conv_pre"), padding=3)
        nk = len(hp["resblock_kernel_sizes"])
        for i, (u, k) in enumerate(zip(rates, hp["upsample_kernel_sizes"])):
            x = F.leaky_relu(x, LRELU_SLOPE)
            x = conv_transpose1d(x, get_weight(params, f"ups.{i}"), _bias(params, f"ups.{i}"),
                                 stride=u, padding=(k - u) // 2)
            if i + 1 < len(rates):
                s = int(np.prod(rates[i + 1:]))
                x_source_len = (src_len + 2 * (s // 2) - 2 * s) // s + 1
            else:
                x_source_len = src_len
            length = min(x.shape[-1], x_source_len)
            x = x[:, :, :length]
            x_source = x[:, :, :length]          # sic (:269)
            x = x + x_source
            xs = None
            for j in range(nk):
                r = resblock1(params, f"resblocks.{i * nk + j}", x, hp["resblock_kernel_sizes"][j],
                              hp["resblock_dilation_sizes"][j])
                xs = r if xs is None else xs + r
            x = xs / nk
            stages.append(x.numpy().copy())
        x = F.leaky_relu(x)
        x = conv1d(x, get_weight(params, "conv_post"), _bias(params, "conv_post"), padding=3)
        x = torch.tanh(x)
    out = x.numpy()
    return (out, stages) if return_stages else out


def istft_same(rea, imag, n_fft, hop, win):
    """ISTFT.forward with padding="same" (apnet.py:46-104), from the definitions: numpy irfft (norm "backward"),
    periodic hann window, overlap-add by explicit accumulation, divided by the overlap-added squared window,
    (win - hop) // 2 samples trimmed per side.  rea / imag [B, N, T] -> [B, T * hop] float32."""
    rea, imag = np.asarray(rea, np.float64), np.asarray(imag, np.float64)
    B, _, T = rea.shape
    n = np.arange(win)
    window = (0.5 - 0.5 * np.cos(2 * np.pi * n / win)).astype(np.float32).astype(np.float64)   # torch.hann_window (periodic)
    frames = np.fft.irfft(rea + 1j * imag, n_fft, axis=1) * window[None, :, None]               # [B, n_fft, T]
    size = (T - 1) * hop + win
    y, env = np.zeros((B, size)), np.zeros(size)
    for t in range(T):
        y[:, t * hop: t * hop + win] += frames[:, :, t]
        env[t * hop: t * hop + win] += window ** 2
    pad = (win - hop) // 2
    y, env = y[:, pad: size - pad], env[pad: size - pad]
    assert (env > 1e-11).all()
    return (y / env).astype(np.float32)


def apnet_forward(params, hp, mel, n_fft, hop, win):
    """apnet.py:357-399.  ``hp`` = cfg.model.apnet as a dict.  Returns (logamp, pha, rea, imag, audio [B, 1, T*hop])."""
    x = _t(np.asarray(mel, np.float32)) if not isinstance(mel, torch.Tensor) else mel.float()

    def stream(s):
        k_in = hp[f"{s}_input_conv_kernel_size"]
        h = conv1d(x, get_weight(params, f"{s}_input_conv"), _bias(params, f"{s}_input_conv"), padding=get_padding(k_in, 1))
        acc = None
        ks, ds = hp[f"{s}_resblock_kernel_sizes"], hp[f"{s}_resblock_dilation_sizes"]
        for j in range(len(ks)):
            r = resblock1(params, f"{s}_ResNet.{j}", h, ks[j], ds[j])      # ASPResBlock / PSPResBlock = ResBlock1 (:113-278)
            acc = r if acc is None else acc + r
        return F.leaky_relu(acc / len(ks))                                   # default slope 0.01 (:366, :377)

    with torch.no_grad():
        a = stream("ASP")
        k = hp["ASP_output_conv_kernel_size"]
        logamp = conv1d(a, get_weight(params, "ASP_output_conv"), _bias(params, "ASP_output_conv"), padding=get_padding(k, 1))
        p = stream("PSP")
        kr, ki = hp["PSP_output_R_conv_kernel_size"], hp["PSP_output_I_conv_kernel_size"]
        R = conv1d(p, get_weight(params, "PSP_output_R_conv"), _bias(params, "PSP_output_R_conv"), padding=get_padding(kr, 1))
        I = conv1d(p, get_weight(params, "PSP_output_I_conv"), _bias(params, "PSP_output_I_conv"), padding=get_padding(ki, 1))
        pha = torch.atan2(I, R)
        rea = torch.exp(logamp) * torch.cos(pha)
        imag = torch.exp(logamp) * torch.sin(pha)
    audio = istft_same(rea.numpy(), imag.numpy(), n_fft, hop, win)
    return logamp.numpy(), pha.numpy(), rea.numpy(), imag.numpy(), audio[:, None, :]


def generator_forward(kind, params, hp, mel, return_stages=False, f0=None):
    if kind == "nsfhifigan":
        return nsfhifigan_forward(params, hp, mel, f0, return_stages)
    fn = hifigan_forward if kind == "hifigan" else bigvgan_forward
    return fn(params, hp, mel, return_stages)


# --------------------------------------------------------------------------
# plumbing above the generator
# --------------------------------------------------------------------------
def vocoder_inference(kind, params, hp, mels, f0s=None):
    """models/vocoders/gan/gan_vocoder_inference.py:11-38 -> [B, T*hop]."""
    return generator_forward(kind, params, hp, mels, f0=f0s)[:, 0, :]


def pad_mels(mels, batched=None):
    """utils/util.py:114-182: zero-pad a list of [n_mel, T_i] into batches of
    ``batched`` (None = one batch); returns (list of [b, n_mel, Tmax], list of frame counts)."""
    groups = [mels] if batched is None else [mels[s:s + batched] for s in range(0, len(mels), batched)]
    tensors, frames = [], []
    for g in groups:
        if not g:
            continue
        size = max(m.shape[-1] for m in g)
        t = np.zeros((len(g), g[0].shape[0], size), np.float32)
        for i, m in enumerate(g):
            t[i, :, :m.shape[-1]] = m
        tensors.append(t)
        frames.append(np.array([m.shape[-1] for m in g], np.int32))
    return tensors, frames


def pad_f0s(f0s, batched=None):
    """utils/util.py:61-111: zero-pad a list of [T_i] f0 tracks into [b, Tmax] batches."""
    groups = [f0s] if batched is None else [f0s[s:s + batched] for s in range(0, len(f0s), batched)]
    tensors = []
    for g in groups:
        if not g:
            continue
        t = np.zeros((len(g), max(f.shape[-1] for f in g)), np.float32)
        for i, f in enumerate(g):
            t[i, :f.shape[-1]] = f
        tensors.append(t)
    return tensors


def synthesis_audios(kind, params, hp, mels, hop_size, batch_size=None, f0s=None):
    """gan_vocoder_inference.py:41-96: per-utterance B=1 forward on the
    zero-padded mel (and f0), trimmed to frames*hop (SURVEY Q12)."""
    out = []
    batches, frames = pad_mels(mels, batch_size)
    f0_batches = pad_f0s(f0s, batch_size) if f0s is not None else [None] * len(batches)
    for mb, fr, fb in zip(batches, frames, f0_batches):
        for i in range(mb.shape[0]):
            a = vocoder_inference(kind, params, hp, mb[i:i + 1], None if fb is None else fb[i:i + 1])[0]
            out.append(a[: int(fr[i]) * hop_size])
    return out
