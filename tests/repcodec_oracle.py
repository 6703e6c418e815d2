"""Float64 restatement of RepCodec, the semantic codec of MaskGCT, Metis and Vevo (models/codec/kmeans/repcodec_model.py):
the encoder and decoder are ``nn.Sequential(VocosBackbone, nn.Linear)`` (restated with tests/vocos_oracle.py's
backbone helpers), the quantizer the codec's ResidualVQ (tests/amphion_codec_oracle.py).  Imports nothing from the
product.

``operands="f16" | "bf16"`` rounds the operands of every GEMM the tensor-core path runs: the pointwise layers' and the
Linear's inputs and weights, and the embed conv's when it is routed to the tensor cores (C_in <= 512; RepCodec's
1024-wide embed stays on the fp32 CUDA cores)."""
from __future__ import annotations

import numpy as np
import torch

from amphion_codec_oracle import TAU, digests, quantize, quantize_kernel_order   # noqa: F401  (used by the tests)
from vocos_oracle import _conv1d, _dwconv, _gelu, _layer_norm, _round

# tag -> (constructor arguments, B, T); the fixtures of tests/golden/repcodec*.npz (tests/golden/gen_repcodec.py).
# "a" is the released geometry; "b" small odd sizes, two quantizers (the [n, B, T] codes) and downsample_scale 2 (the
# down / up keys).
GOLDEN_REPCODEC = {
    "a": (dict(codebook_size=8192, hidden_size=1024, codebook_dim=8, vocos_dim=384, vocos_intermediate_dim=2048,
               vocos_num_layers=12, num_quantizers=1, downsample_scale=1), 2, 24),
    "b": (dict(codebook_size=300, hidden_size=48, codebook_dim=5, vocos_dim=40, vocos_intermediate_dim=96,
               vocos_num_layers=2, num_quantizers=2, downsample_scale=2), 3, 7),
}
SEEDS = {"a": 401, "b": 403}
# MaskGCT's semantic codec (models/tts/maskgct/config/maskgct.json: model.semantic_codec)
MASKGCT_SEMANTIC = dict(codebook_size=8192, hidden_size=1024, codebook_dim=8, vocos_dim=384, vocos_intermediate_dim=2048,
                        vocos_num_layers=12)


def perturb(named_parameters, seed):
    """Redraw every bias, LayerNorm affine and layer scale, in state-dict order: the reference's init zeroes the biases
    and leaves the affines at 1 / 0 and gamma at 1 / num_layers, which would hide a wrong or misplaced one."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in named_parameters:
            if name.endswith(".bias") or name.endswith(".gamma"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
            elif name.endswith("norm.weight"):
                p.copy_(1.0 + torch.randn(p.shape, generator=g) * 0.1)


def vocos_linear(sd, prefix, x, operands=None):
    """``prefix`` + nn.Sequential(VocosBackbone, nn.Linear) (vocos.py:764-783, repcodec_model.py:108-127): x
    [B, C_in, T] -> [B, T, out] float64."""
    g = {k[len(prefix):]: np.asarray(v, dtype=np.float64) for k, v in sd.items() if k.startswith(prefix)}
    r = lambda a: _round(a, operands)   # noqa: E731
    w = g["0.embed.weight"]
    cout, cin = w.shape[:2]
    re = r if cin != cout and cin <= 512 and cout > 4 else (lambda a: a)   # the embed conv's routing   # noqa: E731
    x = _conv1d(re(np.asarray(x, np.float64)), re(w), g["0.embed.bias"], 3)
    x = _layer_norm(x.transpose(0, 2, 1), g["0.norm.weight"], g["0.norm.bias"]).transpose(0, 2, 1)
    i = 0
    while f"0.convnext.{i}.gamma" in g:
        p = f"0.convnext.{i}."
        h = _layer_norm(_dwconv(x, g[p + "dwconv.weight"], g[p + "dwconv.bias"]).transpose(0, 2, 1), g[p + "norm.weight"],
                        g[p + "norm.bias"])
        h = _gelu(r(h) @ r(g[p + "pwconv1.weight"]).T + g[p + "pwconv1.bias"])
        h = r(h) @ r(g[p + "pwconv2.weight"]).T + g[p + "pwconv2.bias"]
        x = x + (g[p + "gamma"] * h).transpose(0, 2, 1)
        i += 1
    feat = _layer_norm(x.transpose(0, 2, 1), g["0.final_layer_norm.weight"], g["0.final_layer_norm.bias"])
    return r(feat) @ r(g["1.weight"]).T + g["1.bias"]


def encoder(sd, x, operands=None):
    """RepCodec's ``encoder(x.transpose(1, 2))``: x [B, T, hidden] -> [B, T, hidden] float64."""
    return vocos_linear(sd, "encoder.", np.asarray(x, np.float64).transpose(0, 2, 1), operands)


def rvq(sd, enc, n, forced=None):
    """The quantizer on the encoder output [B, T, hidden]: quantized_out [B, hidden, T], codes [n, B, T], the layers
    and the distance gaps (amphion_codec_oracle.quantize)."""
    return quantize(sd, np.asarray(enc, np.float64).transpose(0, 2, 1), n, forced=forced)


def decoder(sd, qo, operands=None):
    """RepCodec's ``decoder(quantized_out)``: [B, hidden, T] -> x_rec [B, T, hidden] float64."""
    return vocos_linear(sd, "decoder.", np.asarray(qo, np.float64), operands)
