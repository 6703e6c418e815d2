"""Float64 restatement of NaturalSpeech 3's FACodecRedecoder in eval (models/codec/ns3_codec/facodec.py:602-769,
transformer.py:13-234): ``vq2emb`` with its style-conditioned prosody transformer, and ``inference`` (the decoder's FiLM
and generator: facodec_oracle.inference).  Imports nothing from the product.

``operands="f16" | "bf16"`` rounds the prosody transformer's tensor-core operands (the style LayerNorm outputs feeding a
GEMM, the attention output, relu(ffn_1) and the GEMM weights) to that format, as the 16-bit operand images do; the
arithmetic stays float64.  ``dtype=torch.float32`` runs the same restatement in fp32 arithmetic.  The style Linears read
``mean(condition, dim=1)`` of the speaker embedding expanded over time, as the reference does (``literal_mean=True``);
``literal_mean=False`` reads the embedding itself, as the native path does."""
from __future__ import annotations

import hashlib
import math

import numpy as np
import torch
import torch.nn.functional as F

import facodec_oracle as fo

_GROUPS = ("prosody", "content", "residual")
# variant -> (constructor arguments, B, T).  "a" is the README layout (1 + 2 + 3 tables of 2^10) on a small generator;
# "b" has two prosody tables (the transformer runs once per table), no residual group and odd ratios
GOLDEN_FACODEC_REDECODE = {
    "a": (dict(in_channels=256, upsample_initial_channel=64, up_ratios=[5, 4], vq_num_q_p=1, vq_num_q_c=2, vq_num_q_r=3,
               vq_dim=256, codebook_size_prosody=10, codebook_size_content=10, codebook_size_residual=10), 3, 24),
    "b": (dict(in_channels=256, upsample_initial_channel=64, up_ratios=[3, 2], vq_num_q_p=2, vq_num_q_c=1, vq_num_q_r=0,
               vq_dim=256, codebook_size_prosody=4, codebook_size_content=5, codebook_size_residual=4), 2, 7),
}
# the released checkpoint (ns3_facodec_redecoder.bin): the default constructor
RELEASED = dict(in_channels=256, upsample_initial_channel=1280, up_ratios=[5, 5, 4, 2], vq_num_q_c=2, vq_num_q_p=1,
                vq_num_q_r=3, vq_dim=256, codebook_size_prosody=10, codebook_size_content=10, codebook_size_residual=10)
C_PROSODY = 256
PREFIX = "timbre_cond_prosody_enc."


def n_tables(hp):
    return hp.get("vq_num_q_p", 1), hp.get("vq_num_q_c", 2), hp.get("vq_num_q_r", 3)


def perturb(named_parameters, seed, n_stages):
    """Redraw every parameter in sorted-name order (independent of the module's registration order), at scales where
    every sublayer matters: the reference draws its embeddings at std 1e-5 (they would vanish under ``pe``), starts
    the style Linears at gamma = 1, beta = 0 and SnakeBeta at alpha = beta = 0, and zeroes the conv biases."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in sorted(named_parameters, key=lambda kv: kv[0]):
            fan_in = p.shape[1] * (p.shape[2] if p.dim() > 2 else 1) if p.dim() > 1 else 1
            if name.startswith(tuple(f"{k}_embs." for k in _GROUPS)):
                v = torch.randn(p.shape, generator=g)
            elif name.endswith("weight_g"):
                # conv_post small enough that tanh stays near its linear range, a ResidualUnit's k = 1 conv small
                scale = 0.1 if name.startswith(f"model.{n_stages + 2}.") else \
                    0.25 if (name.startswith("model.") and name.endswith(".block.3.weight_g") and
                             name.split(".")[3] in ("2", "3", "4")) else 1.0
                v = (torch.rand(p.shape, generator=g) * 0.6 + 0.6) * scale
            elif name.endswith("weight_v"):
                v = torch.randn(p.shape, generator=g)
            elif name.endswith((".alpha", ".beta")):   # SnakeBeta, log scale
                v = torch.randn(p.shape, generator=g) * 0.3
            elif name == "timbre_linear.weight" or name.endswith(".style.weight"):
                v = torch.randn(p.shape, generator=g) * (0.3 / math.sqrt(fan_in))
            elif name == "timbre_linear.bias" or name.endswith(".style.bias"):
                v = torch.randn(p.shape, generator=g) * 0.1
                v[:p.shape[0] // 2] += 1.0
            elif name.endswith("in_proj_weight"):
                v = torch.randn(p.shape, generator=g) / math.sqrt(fan_in)
            elif name.endswith("weight"):   # out_proj, ffn_1, ffn_2
                v = torch.randn(p.shape, generator=g) * (0.5 / math.sqrt(fan_in))
            else:
                v = torch.randn(p.shape, generator=g) * 0.1
            p.copy_(v)


def positional_encoding(d_model=C_PROSODY, max_len=5000):
    """transformer.py:35-47: the ``pe`` buffer [max_len, 1, d_model] (fp32, as the reference computes it)."""
    position = torch.arange(max_len).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, d_model, 2) * (-math.log(10000.0) / d_model))
    pe = torch.zeros(max_len, 1, d_model)
    pe[:, 0, 0::2] = torch.sin(position * div_term)
    pe[:, 0, 1::2] = torch.cos(position * div_term)
    return pe


def digests(sd):
    """SHA-256 of every state-dict tensor (fp32 bytes), by name."""
    return {k: hashlib.sha256(np.ascontiguousarray(np.asarray(v, np.float32)).tobytes()).hexdigest()
            for k, v in sd.items()}


def _t(a, dtype=torch.float64):
    return (a if isinstance(a, torch.Tensor) else torch.from_numpy(np.asarray(a))).to(dtype)


def _rnd(x, operands):
    if operands is None:
        return x
    return x.to(torch.float16 if operands == "f16" else torch.bfloat16).to(x.dtype)


def style(sd, name, spk, T, dtype=torch.float64, literal_mean=True):
    """StyleAdaptiveLayerNorm.style(mean(condition, dim=1)) -> (gamma, beta), each [B, 1, C]."""
    s = _t(spk, dtype)
    cond = s[:, None, :].expand(-1, T, -1).mean(dim=1) if literal_mean else s
    st = cond @ _t(sd[name + ".style.weight"], dtype).T + _t(sd[name + ".style.bias"], dtype)
    C = st.shape[1] // 2
    return st[:, None, :C], st[:, None, C:]


def prosody_encoder(sd, x, spk, operands=None, dtype=torch.float64, literal_mean=True):
    """TransformerEncoder(use_cln=True).forward(x [B, T, C], None, spk expanded over T) -> (x, each layer's output)."""
    x = _t(x, dtype)
    B, T, C = x.shape
    h = x + _t(sd[PREFIX + "position_emb.pe"], dtype)[:B]   # [B, T, C] + [B, 1, C]: the batch index is the position
    nh, hd = 4, C // 4

    def saln(v, name):
        gamma, beta = style(sd, name, spk, T, dtype, literal_mean)
        return gamma * F.layer_norm(v, (C,), eps=1e-5) + beta

    def w(name):
        return _rnd(_t(sd[name], dtype), operands)

    layers = []
    for i in range(4):
        pre = f"{PREFIX}layers.{i}."
        a = _rnd(saln(h, pre + "ln_1"), operands)
        qkv = a @ w(pre + "self_attn.in_proj_weight").T + _t(sd[pre + "self_attn.in_proj_bias"], dtype)
        q, k, v = (qkv[..., j * C:(j + 1) * C].reshape(B, T, nh, hd).transpose(1, 2) for j in range(3))
        p = torch.softmax(q @ k.transpose(-1, -2) / 8.0, dim=-1)
        o = _rnd((p @ v).transpose(1, 2).reshape(B, T, C), operands)
        h = h + (o @ w(pre + "self_attn.out_proj.weight").T + _t(sd[pre + "self_attn.out_proj.bias"], dtype))
        a = _rnd(saln(h, pre + "ln_2"), operands)
        f = F.conv1d(a.transpose(1, 2), w(pre + "ffn.ffn_1.weight"), _t(sd[pre + "ffn.ffn_1.bias"], dtype), padding=2)
        f = _rnd(torch.relu(f), operands).transpose(1, 2)
        h = h + (f @ w(pre + "ffn.ffn_2.weight").T + _t(sd[pre + "ffn.ffn_2.bias"], dtype))
        layers.append(h)
    return saln(h, PREFIX + "last_ln"), layers


def vq2emb(sd, codes, spk, n, use_residual=True, operands=None, dtype=torch.float64, literal_mean=True,
           return_layers=False):
    """FACodecRedecoder.vq2emb(codes [>= rows, B, T], spk [B, 256]) -> [B, 256, T].  n = (prosody, content, residual)
    tables.  The transformer runs inside the prosody loop, once per prosody table.  return_layers: also each run's
    layer outputs ([run][layer] -> [B, T, 256])."""
    codes = torch.as_tensor(np.asarray(codes)).long()
    p, c, r = n
    x_t, runs = 0, []
    for i in range(p):
        x_t = x_t + _t(sd[f"prosody_embs.{i}.weight"], dtype)[codes[i]]
        x_t, layers = prosody_encoder(sd, x_t, spk, operands, dtype, literal_mean)
        runs.append(layers)
    out = x_t
    for i in range(c):
        out = out + _t(sd[f"content_embs.{i}.weight"], dtype)[codes[p + i]]
    if use_residual:
        for i in range(r):
            out = out + _t(sd[f"residual_embs.{i}.weight"], dtype)[codes[p + c + i]]
    out = out.transpose(1, 2)
    return (out, runs) if return_layers else out


def inference(sd, up_ratios, x, spk, operands=None, dtype=torch.float64):
    """FACodecRedecoder.inference: FACodecDecoder.inference with the same parameter names (facodec_oracle.inference).
    dtype=torch.float32 runs that restatement in fp32 arithmetic, by swapping its float64 conversions for the call."""
    if dtype == torch.float64:
        return fo.inference(sd, up_ratios, x, spk, operands)
    saved = fo._t, fo._round
    fo._t = lambda a: _t(a, dtype)
    fo._round = lambda v, op: _rnd(v, op)
    try:
        return fo.inference(sd, up_ratios, x, spk, operands)
    finally:
        fo._t, fo._round = saved


def tail_kernel_order(sd, codes, beta, n, use_residual):
    """vq2emb when last_ln's output is beta exactly (its style weight zero): numpy float32 ((beta + c0) + c1) + r0 ...,
    one rounding per add, in the reference's order."""
    codes = np.asarray(codes)
    p, c, r = n
    out = np.broadcast_to(np.asarray(beta, np.float32)[:, None, :], codes.shape[1:] + (beta.shape[-1],)).copy()
    rows = [(f"content_embs.{i}.weight", p + i) for i in range(c)]
    if use_residual:
        rows += [(f"residual_embs.{i}.weight", p + c + i) for i in range(r)]
    for name, q in rows:
        out = (out + np.asarray(sd[name], np.float32)[codes[q]]).astype(np.float32)
    return np.ascontiguousarray(out.transpose(0, 2, 1))
