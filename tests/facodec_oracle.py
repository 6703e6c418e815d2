"""Float64 restatement of NaturalSpeech 3's FACodec decoder path (models/codec/ns3_codec/facodec.py:121-133, :220-240,
:556-576; quantize/fvq.py:86-96, rvq.py:75-81; the anti-aliased SnakeBeta of alias_free_torch): vq2emb, the timbre FiLM
prologue and the generator.  Imports nothing from the product.

``operands="f16" | "bf16"`` rounds the operands of every convolution the tensor-core path runs (all but the C -> 1
conv_post) to that format, as the 16-bit operand images do; the arithmetic stays float64."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

# variant -> (constructor arguments, B, T); "readme" is the geometry of models/codec/ns3_codec/README.md
GOLDEN_FACODEC = {
    "a": (dict(in_channels=32, upsample_initial_channel=128, up_ratios=[5, 4, 2], vq_dim=32), 2, 12),
    "b": (dict(in_channels=16, upsample_initial_channel=64, up_ratios=[3, 2], vq_dim=16, codebook_size_prosody=4,
               codebook_size_content=4, codebook_size_residual=4), 1, 5),
}
README_FACODEC = dict(in_channels=256, upsample_initial_channel=1024, ngf=32, up_ratios=[5, 5, 4, 2], vq_num_q_c=2,
                      vq_num_q_p=1, vq_num_q_r=3, vq_dim=256, codebook_dim=8, codebook_size_prosody=10,
                      codebook_size_content=10, codebook_size_residual=10, use_gr_x_timbre=True,
                      use_gr_residual_f0=True, use_gr_residual_phone=True)


def _t(a):
    return (a if isinstance(a, torch.Tensor) else torch.from_numpy(np.asarray(a))).to(torch.float64)


def _round(x, operands):
    if operands is None:
        return x
    return x.to(torch.float16 if operands == "f16" else torch.bfloat16).to(torch.float64)


def weight(sd, name):
    """``name``.weight, folding torch.nn.utils.weight_norm (dim 0: norm over every other dim) when stored so."""
    if name + ".weight" in sd:
        return _t(sd[name + ".weight"])
    v, g = _t(sd[name + ".weight_v"]), _t(sd[name + ".weight_g"])
    dims = tuple(range(1, v.dim()))
    return g * v / torch.sqrt((v * v).sum(dim=dims, keepdim=True))


def vq2emb(sd, codes, n_q=(1, 2, 3), use_residual=True):
    """codes [n_q, B, T] -> [B, vq_dim, T]: each ResidualVQ sums its layers, then prosody + content [+ residual]."""
    codes = torch.as_tensor(np.asarray(codes)).long()
    out, row = 0, 0
    for q, n in enumerate(n_q):
        if q == 2 and (n == 0 or not use_residual):
            break
        grp = 0
        for j in range(n):
            pre = f"quantizer.{q}.layers.{j}."
            emb = _t(sd[pre + "_codebook.weight"])[codes[row]]                       # [B, T, D]
            grp = grp + (emb @ weight(sd, pre + "out_proj").T + _t(sd[pre + "out_proj.bias"]))
            row += 1
        out = out + grp
    return out.transpose(1, 2)


def film(sd, x, spk):
    """LayerNorm over channels (no affine, eps 1e-5), then x * gamma + beta with (gamma, beta) = timbre_linear(spk)."""
    x, spk = _t(x), _t(spk)
    style = spk @ _t(sd["timbre_linear.weight"]).T + _t(sd["timbre_linear.bias"])
    C = x.shape[1]
    gamma, beta = style[:, :C, None], style[:, C:, None]
    mu = x.mean(dim=1, keepdim=True)
    var = ((x - mu) ** 2).mean(dim=1, keepdim=True)
    return (x - mu) / torch.sqrt(var + 1e-5) * gamma + beta


def activation1d(sd, prefix, x):
    """Activation1d(SnakeBeta(alpha_logscale=True)): 2x up (replicate pad 5, transposed conv, crop 15), snake-beta,
    low-pass 2x down (replicate pad 5 / 6)."""
    a = torch.exp(_t(sd[prefix + ".act.alpha"]))[None, :, None]
    b = torch.exp(_t(sd[prefix + ".act.beta"]))[None, :, None]
    c = x.shape[1]
    fu = _t(sd[prefix + ".upsample.filter"]).reshape(1, 1, 12).expand(c, -1, -1)
    fd = _t(sd[prefix + ".downsample.lowpass.filter"]).reshape(1, 1, 12).expand(c, -1, -1)
    u = 2 * F.conv_transpose1d(F.pad(x, (5, 5), mode="replicate"), fu, stride=2, groups=c)[..., 15:-15]
    u = u + (1.0 / (b + 1e-9)) * torch.sin(u * a) ** 2
    return F.conv1d(F.pad(u, (5, 6), mode="replicate"), fd, stride=2, groups=c)


def _conv(sd, name, x, operands, dilation=1, padding=0):
    return F.conv1d(_round(x, operands), _round(weight(sd, name), operands), _t(sd[name + ".bias"]), dilation=dilation,
                    padding=padding)


def generator(sd, up_ratios, x, operands=None, return_stages=False):
    """self.model(x): conv_pre, the DecoderBlocks, the final act, conv_post (fp32-exact path) and tanh."""
    x = _conv(sd, "model.0", _t(x), operands, padding=3)
    stages = []
    for i, u in enumerate(up_ratios):
        pre = f"model.{1 + i}.block."
        h = activation1d(sd, pre + "0", x)
        x = F.conv_transpose1d(_round(h, operands), _round(weight(sd, pre + "1"), operands), _t(sd[pre + "1.bias"]),
                               stride=u, padding=u // 2 + u % 2, output_padding=u % 2)
        for p, d in enumerate((1, 3, 9)):
            r = f"{pre}{2 + p}.block."
            h = _conv(sd, r + "1", activation1d(sd, r + "0", x), operands, dilation=d, padding=3 * d)
            x = x + _conv(sd, r + "3", activation1d(sd, r + "2", h), operands)
        stages.append(x)
    n = len(up_ratios)
    h = activation1d(sd, f"model.{1 + n}", x)
    wav = torch.tanh(F.conv1d(h, weight(sd, f"model.{2 + n}"), _t(sd[f"model.{2 + n}.bias"]), padding=3))
    return (wav, stages) if return_stages else wav


def inference(sd, up_ratios, x, spk, operands=None):
    """FACodecDecoder.inference(x, speaker_embedding) -> [B, 1, T * prod(up_ratios)] (float64)."""
    return generator(sd, up_ratios, _round(film(sd, x, spk), operands), operands)
