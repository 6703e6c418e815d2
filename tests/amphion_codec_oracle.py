"""Float64 restatement of the acoustic codec of MaskGCT, Metis and DebaTTS (models/codec/amphion_codec/codec.py): the
CodecEncoder (the FACodec encoder's structure with a plain Snake1d), the ResidualVQ of FactorizedVectorQuantize layers
and, for the waveform, Vocos (tests/vocos_oracle.py).  Imports nothing from the product.

``operands="f16" | "bf16"`` rounds the operands of every encoder convolution the tensor-core path runs (all but
conv_pre, whose single input channel stays on the fp32 CUDA cores), as the 16-bit operand images do."""
from __future__ import annotations

import hashlib
import math

import numpy as np
import torch
import torch.nn.functional as F

from facodec_oracle import _conv, _round, _t, weight
from facodec_quantize_oracle import TAU   # noqa: F401  (the codes' margin rule, used by the tests)
from vocos_oracle import vocos_forward

# tag -> (encoder arguments, decoder arguments, B, N, n_quantizers); the fixtures of tests/golden/amphion_codec*.npz
# (tests/golden/gen_amphion_codec.py).  "a" is MaskGCT's layout scaled down; "b" odd ratios, a codebook of 100 rows
# (a ragged last chunk of the 256-row codebook stream) and one quantizer.
_DEC = dict(quantizer_type="fvq", use_l2_normlize=True, use_vocos=True, quantizer_dropout=0.5, commitment=0.25)
GOLDEN_CODEC = {
    "a": (dict(d_model=8, up_ratios=[3, 4, 5, 8], out_channels=64),
          dict(_DEC, in_channels=64, num_quantizers=12, codebook_size=1024, codebook_dim=8, vocos_dim=64,
               vocos_intermediate_dim=192, vocos_num_layers=3, n_fft=1920, hop_size=480), 2, 24 * 480 + 7, 12),
    "b": (dict(d_model=8, up_ratios=[3, 2], out_channels=24),
          dict(_DEC, in_channels=24, num_quantizers=3, codebook_size=100, codebook_dim=8, vocos_dim=32,
               vocos_intermediate_dim=64, vocos_num_layers=2, n_fft=24, hop_size=6), 1, 29, 1),
}
SEEDS = {"a": 311, "b": 313}
# MaskGCT's acoustic codec (models/tts/maskgct/config/maskgct.json: model.acoustic_codec)
MASKGCT_ENCODER = dict(d_model=96, up_ratios=[3, 4, 5, 8], out_channels=256, use_tanh=False)
MASKGCT_DECODER = dict(_DEC, in_channels=256, num_quantizers=12, codebook_size=1024, codebook_dim=8, vocos_dim=512,
                       vocos_intermediate_dim=4096, vocos_num_layers=30, n_fft=1920, hop_size=480)


def perturb(named_parameters, seed):
    """Redraw every bias and every Snake1d alpha, in state-dict order: the reference's init zeroes the biases and sets
    alpha to 1, which would hide a wrong bias or a wrong alpha.  About a third of the alphas are negative."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in named_parameters:
            if name.endswith(".alpha"):
                mag = torch.rand(p.shape, generator=g) * 1.2 + 0.3
                sign = torch.where(torch.rand(p.shape, generator=g) < 0.3, -1.0, 1.0)
                p.copy_(mag * sign)
            elif name.endswith(".bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)


def digests(sd):
    """SHA-256 of every tensor (fp32 bytes), by name."""
    return {k: hashlib.sha256(np.ascontiguousarray(np.asarray(v, np.float32)).tobytes()).hexdigest() for k, v in sd.items()}


def snake1d(x, alpha):
    """codec.py:34-39: x + (alpha + 1e-9)^-1 sin(alpha x)^2 per channel."""
    a = _t(alpha).reshape(1, -1, 1)
    return x + (1.0 / (a + 1e-9)) * torch.sin(a * x) ** 2


def encoder(sd, up_ratios, wav, operands=None, return_stages=False):
    """CodecEncoder.forward(wav) -> [B, out_channels, F] float64; with return_stages also each EncoderBlock's output."""
    x = F.conv1d(_t(wav), weight(sd, "block.0"), _t(sd["block.0.bias"]), padding=3)
    stages = []
    for i, s in enumerate(up_ratios):
        pre = f"block.{1 + i}.block."
        for p, d in enumerate((1, 3, 9)):
            r = f"{pre}{p}.block."
            h = _conv(sd, r + "1", snake1d(x, sd[r + "0.alpha"]), operands, dilation=d, padding=3 * d)
            x = x + _conv(sd, r + "3", snake1d(h, sd[r + "2.alpha"]), operands)
        h = snake1d(x, sd[pre + "3.alpha"])
        x = F.conv1d(_round(h, operands), _round(weight(sd, pre + "4"), operands), _t(sd[pre + "4.bias"]), stride=s,
                     padding=s // 2 + s % 2)
        stages.append(x)
    n = len(up_ratios)
    h = snake1d(x, sd[f"block.{1 + n}.alpha"])
    cout, cin = weight(sd, f"block.{2 + n}").shape[:2]
    post_tc = cin != cout and cin <= 512 and cout > 4   # the generators' conv_post routing
    out = _conv(sd, f"block.{2 + n}", h, operands if post_tc else None, padding=1)
    return (out, stages) if return_stages else out


def _layer(sd, i):
    pre = f"quantizer.quantizers.{i}."
    w_in = weight(sd, pre + "in_project")[:, :, 0]     # [D_cb, C]
    w_out = weight(sd, pre + "out_project")[:, :, 0]   # [C, D_cb]
    return w_in, _t(sd[pre + "in_project.bias"]), w_out, _t(sd[pre + "out_project.bias"]), _t(sd[pre + "codebook.weight"])


def quantize(sd, z, n_quantizers, forced=None):
    """ResidualVQ.forward in eval (residual_vq.py:69-134, factorized_vector_quantize.py:52-129) in float64.  forced:
    codes [n, B, T] to continue with instead of the argmin (teacher forcing).  Returns quantized_out [B, C, T], codes
    int64 [n, B, T], all_quantized [n, B, C, T] and the gap between the best and the runner-up distance [n, B, T]."""
    r = _t(z).permute(0, 2, 1)   # [B, T, C]
    out, codes, layers, gaps = 0.0, [], [], []
    for i in range(n_quantizers):
        w_in, b_in, w_out, b_out, cb = _layer(sd, i)
        z_e = r @ w_in.T + b_in
        e = z_e / torch.clamp(torch.linalg.norm(z_e, dim=-1, keepdim=True), min=1e-12)
        cn = cb / torch.clamp(torch.linalg.norm(cb, dim=-1, keepdim=True), min=1e-12)
        dist = (e * e).sum(-1, keepdim=True) - 2 * e @ cn.T + (cn * cn).sum(-1)[None, None, :]
        srt = torch.sort(dist, dim=-1).values
        gaps.append(srt[..., 1] - srt[..., 0] if cb.shape[0] > 1 else torch.full(srt.shape[:2], math.inf))
        code = torch.argmin(dist, dim=-1) if forced is None else torch.as_tensor(np.asarray(forced[i]), dtype=torch.int64)
        codes.append(code)
        q = cb[code] @ w_out.T + b_out
        out = out + q
        r = r - q
        layers.append(q.permute(0, 2, 1))
    return out.permute(0, 2, 1), torch.stack(codes), torch.stack(layers), torch.stack(gaps)


def vq2emb(sd, codes, n_quantizers):
    """ResidualVQ.vq2emb (residual_vq.py:136-144) in float64."""
    out = 0.0
    for i in range(n_quantizers):
        _, _, w_out, b_out, cb = _layer(sd, i)
        out = out + (cb[torch.as_tensor(np.asarray(codes[i]), dtype=torch.int64)] @ w_out.T + b_out)
    return out.permute(0, 2, 1)


def decode(sd, dec_hp, x, operands=None):
    """CodecDecoder.forward(x) = Vocos(x) (codec.py:409), through tests/vocos_oracle.py on the ``model.*`` entries."""
    vsd = {k[len("model."):]: np.asarray(v) for k, v in sd.items() if k.startswith("model.")}
    hp = dict(input_channels=dec_hp["in_channels"], dim=dec_hp["vocos_dim"], intermediate_dim=dec_hp["vocos_intermediate_dim"],
              num_layers=dec_hp["vocos_num_layers"], n_fft=dec_hp["n_fft"], hop_size=dec_hp["hop_size"])
    return vocos_forward(vsd, hp, np.asarray(x, np.float64), operands=operands)


def one_hot_projections(sd, seed):
    """Make every layer's folded in_project and out_project one-hot (weight_v one-hot with weight_g 1, so the fold
    w = g v / |v| is exactly 0 or 1): each projection is then one exact term plus its bias, and the RVQ's fp32 result
    depends only on the order of its adds (quantize_kernel_order)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for k in list(sd):
            if k.endswith(("in_project.weight_v", "out_project.weight_v")):
                v = sd[k]
                v.zero_()
                pick = torch.randint(0, v.shape[1], (v.shape[0],), generator=g)
                v[torch.arange(v.shape[0]), pick, 0] = 1.0
            elif k.endswith(("in_project.weight_g", "out_project.weight_g")):
                sd[k].fill_(1.0)


def quantize_kernel_order(sd, z, n_quantizers):
    """ResidualVQ.forward with one-hot projections, in numpy float32 in the kernel's operation order: z_e = r[d] +
    b_in, z_q = z_e + (codebook[code] - z_e), q = z_q[d'] + b_out, r = r - q, quantized_out = ((0 + q_0) + q_1) + ...
    Codes are the float64 argmin (the test data keeps the distances apart)."""
    r = np.asarray(z, np.float32)
    acc, codes, layers = np.zeros_like(r), [], []
    for i in range(n_quantizers):
        w_in, b_in, w_out, b_out, cb = (a.numpy() for a in _layer(sd, i))
        b_in, b_out, cb32 = b_in.astype(np.float32), b_out.astype(np.float32), cb.astype(np.float32)
        z_e = (np.einsum("dc,bct->btd", w_in.astype(np.float32), r) + b_in).astype(np.float32)
        e = z_e.astype(np.float64)
        e = e / np.maximum(np.linalg.norm(e, axis=-1, keepdims=True), 1e-12)
        cn = cb / np.maximum(np.linalg.norm(cb, axis=-1, keepdims=True), 1e-12)
        code = np.argmin((e * e).sum(-1, keepdims=True) - 2 * e @ cn.T + (cn * cn).sum(-1), axis=-1)
        z_q = (z_e + (cb32[code] - z_e).astype(np.float32)).astype(np.float32)
        q = (np.einsum("cd,btd->bct", w_out.astype(np.float32), z_q) + b_out[None, :, None]).astype(np.float32)
        r = (r - q).astype(np.float32)
        acc = (acc + q).astype(np.float32)
        codes.append(code)
        layers.append(q)
    return acc, np.stack(codes).astype(np.int64), np.stack(layers)
