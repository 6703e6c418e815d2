"""Float64 restatement of NaturalSpeech 3's FACodecEncoder (models/codec/ns3_codec/facodec.py:121-194): conv_pre, the
EncoderBlocks (three ResidualUnits, the anti-aliased SnakeBeta, a strided conv), the final activation and conv_post.
Imports nothing from the product.

``operands="f16" | "bf16"`` rounds the operands of every convolution the tensor-core path runs (all but conv_pre,
whose single input channel stays on the fp32 CUDA cores) to that format, as the 16-bit operand images do; the
arithmetic stays float64.  ``dtype=torch.float32`` runs the same restatement in fp32 arithmetic: with rounded operands
the distance between the two is the floor any fp32-accumulating implementation of those operands sits at (a
rounding boundary crossed by fp32 round-off moves an operand by a whole 16-bit ulp, and the deeper layers carry it)."""
from __future__ import annotations

import torch
import torch.nn.functional as F

import numpy as np

from facodec_oracle import _conv, _round, _t, activation1d, weight

# variant -> (constructor arguments, B, N); N is not a multiple of the hop.  "a" has odd strides and C_in = 8 (a
# strided conv from fp32 input), "b" stride 8 and out_channels % 16 != 0
GOLDEN_FACODEC_ENCODE = {
    "a": (dict(ngf=8, up_ratios=[2, 3, 5], out_channels=48), 2, 1001),
    "b": (dict(ngf=16, up_ratios=[4, 8], out_channels=40), 1, 517),
}
README_FACODEC_ENCODER = dict(ngf=32, up_ratios=[2, 4, 5, 5], out_channels=256)


def frames(up_ratios, n):
    """Output frames of n samples; 0 when a strided conv's padded input is shorter than its kernel."""
    for s in up_ratios:
        pad = s // 2 + s % 2
        if n + 2 * pad < 2 * s:
            return 0
        n = (n + 2 * pad - 2 * s) // s + 1
    return n


def _in(dtype):
    """The helpers of facodec_oracle (float64) at another arithmetic dtype."""
    if dtype == torch.float64:
        return _t, _round, weight, activation1d, _conv

    def t(a):
        return (a if isinstance(a, torch.Tensor) else torch.from_numpy(np.asarray(a))).to(dtype)

    def rnd(x, operands):
        return x if operands is None else x.to(torch.float16 if operands == "f16" else torch.bfloat16).to(dtype)

    def w(sd, name):
        return weight(sd, name).to(dtype)

    def act(sd, prefix, x):
        a = torch.exp(t(sd[prefix + ".act.alpha"]))[None, :, None]
        b = torch.exp(t(sd[prefix + ".act.beta"]))[None, :, None]
        c = x.shape[1]
        fu = t(sd[prefix + ".upsample.filter"]).reshape(1, 1, 12).expand(c, -1, -1)
        fd = t(sd[prefix + ".downsample.lowpass.filter"]).reshape(1, 1, 12).expand(c, -1, -1)
        u = 2 * F.conv_transpose1d(F.pad(x, (5, 5), mode="replicate"), fu, stride=2, groups=c)[..., 15:-15]
        u = u + (1.0 / (b + 1e-9)) * torch.sin(u * a) ** 2
        return F.conv1d(F.pad(u, (5, 6), mode="replicate"), fd, stride=2, groups=c)

    def conv(sd, name, x, operands, dilation=1, padding=0):
        return F.conv1d(rnd(x, operands), rnd(w(sd, name), operands), t(sd[name + ".bias"]), dilation=dilation,
                        padding=padding)

    return t, rnd, w, act, conv


def encoder(sd, up_ratios, wav, operands=None, return_stages=False, dtype=torch.float64):
    """FACodecEncoder.forward(wav) -> [B, out_channels, F] (dtype); with return_stages also each EncoderBlock's output."""
    _t, _round, weight, activation1d, _conv = _in(dtype)
    x = F.conv1d(_t(wav), weight(sd, "block.0"), _t(sd["block.0.bias"]), padding=3)
    stages = []
    for i, s in enumerate(up_ratios):
        pre = f"block.{1 + i}.block."
        for p, d in enumerate((1, 3, 9)):
            r = f"{pre}{p}.block."
            h = _conv(sd, r + "1", activation1d(sd, r + "0", x), operands, dilation=d, padding=3 * d)
            x = x + _conv(sd, r + "3", activation1d(sd, r + "2", h), operands)
        h = activation1d(sd, pre + "3", x)
        x = F.conv1d(_round(h, operands), _round(weight(sd, pre + "4"), operands), _t(sd[pre + "4.bias"]), stride=s,
                     padding=s // 2 + s % 2)
        stages.append(x)
    n = len(up_ratios)
    h = activation1d(sd, f"block.{1 + n}", x)
    cout, cin = weight(sd, f"block.{2 + n}").shape[:2]
    post_tc = cin != cout and cin <= 512 and cout > 4   # the generators' conv_post routing
    out = _conv(sd, f"block.{2 + n}", h, operands if post_tc else None, padding=1)
    return (out, stages) if return_stages else out
