"""Float64 restatement of NaturalSpeech 3's FACodecDecoder.forward(vq=True) in eval (models/codec/ns3_codec/facodec.py:
408-471, quantize/rvq.py:27-76, quantize/fvq.py:43-111, transformer.py:35-217): the three ResidualVQs and the timbre
encoder with the time mean.  Imports nothing from the product.

``operands="f16" | "bf16"`` rounds the timbre encoder's tensor-core operands (the LayerNorm outputs feeding a GEMM,
the attention output, relu(ffn_1) and the GEMM weights) to that format, as the 16-bit operand images do; the
arithmetic stays float64.  ``dtype=torch.float32`` runs the same restatement in fp32 arithmetic.  The quantizer is fp32
on CUDA cores at every precision, so it has no operand rounding; ``quantize_kernel_order`` restates it in the fp32
operation order of the kernel, exact for one-hot projections."""
from __future__ import annotations

import hashlib
import math

import numpy as np
import torch
import torch.nn.functional as F

# variant -> (constructor arguments, B, T, n_quantizers).  "a" is the README quantizer (1 + 2 + 3 layers of 2^10 x 8),
# "b" has no residual group, codebooks of 2^4 and keeps one layer per group
_SMALL = dict(in_channels=256, vq_dim=256, upsample_initial_channel=32, up_ratios=[2], codebook_dim=8)
GOLDEN_FACODEC_QUANTIZE = {
    "a": (dict(_SMALL, vq_num_q_p=1, vq_num_q_c=2, vq_num_q_r=3, codebook_size_prosody=10, codebook_size_content=10,
               codebook_size_residual=10), 3, 24, None),
    "b": (dict(_SMALL, vq_num_q_p=1, vq_num_q_c=2, vq_num_q_r=0, codebook_size_prosody=4, codebook_size_content=4,
               codebook_size_residual=4), 2, 7, 1),
}
TAU = 1e-5   # codes are compared where the float64 gap between the best and the runner-up distance exceeds this
C_TIMBRE = 256


def positional_encoding(d_model=C_TIMBRE, max_len=5000):
    """transformer.py:35-47: the ``pe`` buffer [max_len, 1, d_model] (fp32, as the reference computes it)."""
    position = torch.arange(max_len).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, d_model, 2) * (-math.log(10000.0) / d_model))
    pe = torch.zeros(max_len, 1, d_model)
    pe[:, 0, 0::2] = torch.sin(position * div_term)
    pe[:, 0, 1::2] = torch.cos(position * div_term)
    return pe


def perturb(named_parameters, seed):
    """Redraw the quantizers' and the timbre encoder's parameters, in state-dict order, at scales where every
    sublayer matters (the reference's 0.02 FFN init would leave the residual branches negligible)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in named_parameters:
            if not name.startswith(("quantizer.", "timbre_encoder.")):
                continue
            fan_in = p.shape[1] * (p.shape[2] if p.dim() > 2 else 1) if p.dim() > 1 else 1
            if name.endswith("weight_g"):
                v = torch.rand(p.shape, generator=g) * 0.6 + 0.6
            elif name.endswith("weight_v") or name.endswith("_codebook.weight"):
                v = torch.randn(p.shape, generator=g)
            elif ".ln_" in name or "last_ln" in name:
                v = torch.randn(p.shape, generator=g) * (0.2 if name.endswith("weight") else 0.1)
                if name.endswith("weight"):
                    v = v + 1.0
            elif name.endswith("in_proj_weight"):
                v = torch.randn(p.shape, generator=g) / math.sqrt(fan_in)
            elif name.endswith("weight"):   # out_proj, ffn_1, ffn_2
                v = torch.randn(p.shape, generator=g) * (0.5 / math.sqrt(fan_in))
            else:
                v = torch.randn(p.shape, generator=g) * 0.1
            p.copy_(v)


def digests(sd):
    """SHA-256 of every quantizer / timbre-encoder tensor (fp32 bytes), by name."""
    return {k: hashlib.sha256(np.ascontiguousarray(np.asarray(v, np.float32)).tobytes()).hexdigest()
            for k, v in sd.items() if k.startswith(("quantizer.", "timbre_encoder."))}


def _t(a, dtype=torch.float64):
    return (a if isinstance(a, torch.Tensor) else torch.from_numpy(np.asarray(a))).to(dtype)


def _weight(sd, name, dtype=torch.float64):
    if name + ".weight" in sd:
        return _t(sd[name + ".weight"], dtype)
    v, g = _t(sd[name + ".weight_v"], dtype), _t(sd[name + ".weight_g"], dtype)
    return g * v / torch.sqrt((v * v).sum(dim=tuple(range(1, v.dim())), keepdim=True))


def _rnd(x, operands):
    if operands is None:
        return x
    return x.to(torch.float16 if operands == "f16" else torch.bfloat16).to(x.dtype)


def _groups(nq):
    """(group, first layer row, layers) of the ResidualVQs that exist."""
    out, q0 = [], 0
    for gi, n in enumerate(nq):
        if n > 0:
            out.append((gi, q0, n))
        q0 += n
    return out


def quantize(sd, x, nq, n_quantizers=None, forced=None):
    """facodec.py:408-445 in float64.  nq = (prosody, content, residual) layers.  forced: codes [n_used, B, T] to
    continue with instead of the argmin (teacher forcing).  Returns outs [B, C, T], qs int64 [n_used, B, T], the
    groups' sums, and the gap between the best and the runner-up distance [n_used, B, T] (inf with one code)."""
    x = _t(x)
    B, C, T = x.shape
    k = max(nq) if n_quantizers is None else n_quantizers
    outs, qs, bufs, gaps = 0, [], [], []
    row = 0
    for gi, q0, n in _groups(nq):
        inp = x if gi < 2 else x - (bufs[0] + bufs[1])
        r, acc = inp.permute(0, 2, 1), 0
        for j in range(min(k, n)):
            pre = f"quantizer.{gi}.layers.{j}."
            z_e = r @ _weight(sd, pre + "in_proj").T + _t(sd[pre + "in_proj.bias"])
            cb = _t(sd[pre + "_codebook.weight"])
            e = z_e / torch.clamp(torch.linalg.norm(z_e, dim=-1, keepdim=True), min=1e-12)
            cn = cb / torch.clamp(torch.linalg.norm(cb, dim=-1, keepdim=True), min=1e-12)
            dist = (e * e).sum(-1, keepdim=True) - 2 * e @ cn.T + (cn * cn).sum(-1)[None, None, :]
            srt = torch.sort(dist, dim=-1).values
            gaps.append(srt[..., 1] - srt[..., 0] if cb.shape[0] > 1 else torch.full(srt.shape[:2], math.inf))
            code = torch.argmin(dist, dim=-1) if forced is None else _t(forced[row], torch.int64)
            qs.append(code)
            q = cb[code] @ _weight(sd, pre + "out_proj").T + _t(sd[pre + "out_proj.bias"])
            r, acc = r - q, acc + q
            row += 1
        buf = acc.permute(0, 2, 1)
        bufs.append(buf)
        outs = outs + buf
    return outs, torch.stack(qs), bufs, torch.stack(gaps)


def quantize_kernel_order(sd, x, nq, n_quantizers=None):
    """The RVQ in the kernel's fp32 operation order (numpy float32), for weight-normed projections whose folded weights
    are one-hot (each in_proj row and each out_proj row a single 1): every dot product is then one exact term.  Codes
    are the float64 argmin (the test data keeps the distances apart, or ties them exactly)."""
    x = np.asarray(x, np.float32)
    B, C, T = x.shape
    k = max(nq) if n_quantizers is None else n_quantizers
    qs, bufs = [], []
    for gi, q0, n in _groups(nq):
        r = x.copy() if gi < 2 else (x - (bufs[0] + bufs[1])).astype(np.float32)
        acc = np.zeros_like(x)
        for j in range(min(k, n)):
            pre = f"quantizer.{gi}.layers.{j}."
            w_in = _weight(sd, pre + "in_proj").numpy().astype(np.float32)     # [D, C] one-hot rows
            w_out = _weight(sd, pre + "out_proj").numpy().astype(np.float32)   # [C, D] one-hot rows
            b_in = np.asarray(sd[pre + "in_proj.bias"], np.float32)
            b_out = np.asarray(sd[pre + "out_proj.bias"], np.float32)
            cb = np.asarray(sd[pre + "_codebook.weight"], np.float32)
            z_e = (np.einsum("dc,bct->btd", w_in, r).astype(np.float32) + b_in).astype(np.float32)
            e = z_e.astype(np.float64)
            e = e / np.maximum(np.linalg.norm(e, axis=-1, keepdims=True), 1e-12)
            c64 = cb.astype(np.float64)
            cn = c64 / np.maximum(np.linalg.norm(c64, axis=-1, keepdims=True), 1e-12)
            dist = (e * e).sum(-1, keepdims=True) - 2 * e @ cn.T + (cn * cn).sum(-1)
            code = np.argmin(dist, axis=-1)
            qs.append(code)
            z_q = (z_e + (cb[code] - z_e).astype(np.float32)).astype(np.float32)
            q = (np.einsum("cd,btd->bct", w_out, z_q).astype(np.float32) + b_out[None, :, None]).astype(np.float32)
            r = (r - q).astype(np.float32)
            acc = (acc + q).astype(np.float32)
        bufs.append(acc)
    outs = bufs[0] + bufs[1]
    if len(bufs) > 2:
        outs = (outs + bufs[2]).astype(np.float32)
    return outs, np.stack(qs).astype(np.int64), bufs


def timbre(sd, x, operands=None, dtype=torch.float64, return_layers=False):
    """transformer.py:206-217 on x.transpose(1, 2), then the time mean (facodec.py:465-469) -> spk [B, 256]."""
    x = _t(x, dtype)
    B, C, T = x.shape
    pe = _t(sd["timbre_encoder.position_emb.pe"], dtype)
    h = x.transpose(1, 2) + pe[:B]                     # [B, T, C] + [B, 1, C]: the batch index is the position
    layers = []
    nh, hd = 4, C // 4

    def ln(v, name):
        return F.layer_norm(v, (C,), _t(sd[name + ".weight"], dtype), _t(sd[name + ".bias"], dtype), 1e-5)

    def w(name):
        return _rnd(_t(sd[name], dtype), operands)

    for i in range(4):
        pre = f"timbre_encoder.layers.{i}."
        a = _rnd(ln(h, pre + "ln_1"), operands)
        qkv = a @ w(pre + "self_attn.in_proj_weight").T + _t(sd[pre + "self_attn.in_proj_bias"], dtype)
        q, k, v = (qkv[..., j * C:(j + 1) * C].reshape(B, T, nh, hd).transpose(1, 2) for j in range(3))
        p = torch.softmax(q @ k.transpose(-1, -2) / 8.0, dim=-1)
        o = _rnd((p @ v).transpose(1, 2).reshape(B, T, C), operands)
        h = h + (o @ w(pre + "self_attn.out_proj.weight").T + _t(sd[pre + "self_attn.out_proj.bias"], dtype))
        a = _rnd(ln(h, pre + "ln_2"), operands)
        f = F.conv1d(a.transpose(1, 2), w(pre + "ffn.ffn_1.weight"), _t(sd[pre + "ffn.ffn_1.bias"], dtype), padding=2)
        f = _rnd(torch.relu(f), operands).transpose(1, 2)
        h = h + (f @ w(pre + "ffn.ffn_2.weight").T + _t(sd[pre + "ffn.ffn_2.bias"], dtype))
        layers.append(h)
    y = ln(h, "timbre_encoder.last_ln")
    spk = y.mean(dim=1)
    return (spk, layers) if return_layers else spk
