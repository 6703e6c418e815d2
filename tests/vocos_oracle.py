"""CPU oracle of Vocos.forward (models/codec/amphion_codec/vocos.py:824-881, non-conditional backbone, "same" ISTFT),
restated op by op in float64 numpy on a state dict: embed conv, LayerNorm, ConvNeXt blocks (depthwise conv, LayerNorm,
Linear, erf-GELU, Linear, layer scale, residual), final LayerNorm, the head's Linear, exp / clip / cos / sin, then irfft,
window, overlap-add, division by the window envelope and the "same" trim.

``operands="f16" | "bf16"`` rounds the operands of every GEMM the tensor-core path runs (embed input and weight, the
pointwise layers' inputs and weights, the head's input and weight) as the kernels do, so that what remains is the
fp32 accumulation order."""
import numpy as np
import torch
from scipy.special import erf

# tag -> (hyper-parameters, B, L); the fixtures of tests/golden/vocos.npz (tests/golden/gen_vocos.py)
GOLDEN_VOCOS = {
    "a": (dict(input_channels=20, dim=48, intermediate_dim=144, num_layers=3, n_fft=64, hop_size=16), 2, 24),
    "b": (dict(input_channels=12, dim=40, intermediate_dim=120, num_layers=2, n_fft=48, hop_size=12), 1, 7),
}
# Vevo's vocoder (models/vc/vevo/config/Vocoder.json): 24 kHz, 128 mels
HP_VOCOS_RECIPE = dict(input_channels=128, dim=1024, intermediate_dim=4096, num_layers=30, n_fft=1920, hop_size=480)


def _round(a, operands):
    if operands is None:
        return a
    dt = {"f16": torch.float16, "bf16": torch.bfloat16}[operands]
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dt).to(torch.float64).numpy()


def _layer_norm(x, w, b, eps=1e-6):
    """x [..., C] over the last axis: two-pass mean and biased variance, as torch.layer_norm."""
    mu = x.mean(-1, keepdims=True)
    var = ((x - mu) ** 2).mean(-1, keepdims=True)
    return (x - mu) / np.sqrt(var + eps) * w + b


def _conv1d(x, w, b, pad):
    """x [B, Cin, T], w [Cout, Cin, k], zero padding pad."""
    B, Cin, T = x.shape
    k = w.shape[2]
    xp = np.pad(x, ((0, 0), (0, 0), (pad, pad)))
    y = np.zeros((B, w.shape[0], T))
    for j in range(k):
        y += np.einsum("oc,bct->bot", w[:, :, j], xp[:, :, j:j + T])
    return y + b[None, :, None]


def _dwconv(x, w, b):
    """depthwise k = 7, padding 3: x [B, C, T], w [C, 1, 7]."""
    T = x.shape[2]
    xp = np.pad(x, ((0, 0), (0, 0), (3, 3)))
    y = np.zeros_like(x)
    for j in range(7):
        y += w[None, :, 0, j, None] * xp[:, :, j:j + T]
    return y + b[None, :, None]


def _gelu(x):
    return 0.5 * x * (1.0 + erf(x / np.sqrt(2.0)))


def istft_same(spec, window, n_fft, hop):
    """spec complex [B, bins, L] -> [B, L * hop] (vocos.py:129-167)."""
    B, _, L = spec.shape
    frames = np.fft.irfft(spec, n_fft, axis=1) * window[None, :, None]      # norm "backward"
    out = (L - 1) * hop + n_fft
    y = np.zeros((B, out))
    env = np.zeros(out)
    for f in range(L):
        y[:, f * hop:f * hop + n_fft] += frames[:, :, f]
        env[f * hop:f * hop + n_fft] += window ** 2
    pad = (n_fft - hop) // 2
    return y[:, pad:out - pad] / env[pad:out - pad]


def vocos_forward(sd, hp, mel, operands=None, stages=False):
    """mel [B, input_channels, L] -> wav [B, 1, L * hop] (float32); with stages, also each block's output and the
    backbone's output ([B, L, dim])."""
    g = {k: np.asarray(v, dtype=np.float64) for k, v in sd.items()}
    r = lambda a: _round(a, operands)   # noqa: E731
    x = _conv1d(r(np.asarray(mel, np.float64)), r(g["backbone.embed.weight"]), g["backbone.embed.bias"], 3)
    x = _layer_norm(x.transpose(0, 2, 1), g["backbone.norm.weight"], g["backbone.norm.bias"]).transpose(0, 2, 1)
    outs = []
    for i in range(hp["num_layers"]):
        p = f"backbone.convnext.{i}."
        h = _dwconv(x, g[p + "dwconv.weight"], g[p + "dwconv.bias"]).transpose(0, 2, 1)    # [B, T, C]
        h = _layer_norm(h, g[p + "norm.weight"], g[p + "norm.bias"])
        h = _gelu(r(h) @ r(g[p + "pwconv1.weight"]).T + g[p + "pwconv1.bias"])
        h = r(h) @ r(g[p + "pwconv2.weight"]).T + g[p + "pwconv2.bias"]
        x = x + (g[p + "gamma"] * h).transpose(0, 2, 1)
        outs.append(x.astype(np.float32))
    feat = _layer_norm(x.transpose(0, 2, 1), g["backbone.final_layer_norm.weight"], g["backbone.final_layer_norm.bias"])
    y = (r(feat) @ r(g["head.out.weight"]).T + g["head.out.bias"]).transpose(0, 2, 1)       # [B, n_fft + 2, L]
    bins = y.shape[1] // 2
    mag = np.minimum(np.exp(y[:, :bins]), 1e2)
    S = mag * (np.cos(y[:, bins:]) + 1j * np.sin(y[:, bins:]))
    wav = istft_same(S, g["head.istft.window"], hp["n_fft"], hp["hop_size"])[:, None, :].astype(np.float32)
    if stages:
        return wav, outs, feat.astype(np.float32)
    return wav
