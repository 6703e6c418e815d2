"""Float64 restatement of NaturalSpeech 3's FACodecDecoderV2.forward(vq=True) in eval (models/codec/ns3_codec/facodec.py:
1027-1094): the prosody transformer melspec_encoder(melspec_linear(prosody_feature^T)), the three ResidualVQs (the
prosody group reads the transformer's output, the content group x, the residual group x - (prosody + content)) and the
timbre encoder.  Reuses tests/facodec_quantize_oracle.py's pieces; imports nothing from the product.

The prosody transformer runs in fp32 on CUDA cores at every precision, so it has no operand rounding here."""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

import facodec_quantize_oracle as fqo

BINS = 20
# variant -> (encoder arguments, decoder arguments, B, samples, n_quantizers).  "a": hop 200 and the README quantizer
# (1 + 2 + 3 layers of 2^10 x 8); "b": no residual group, codebooks of 2^4, one layer per group, an odd frame count
_ENC = dict(ngf=2, up_ratios=(2, 4, 5, 5), out_channels=256)
GOLDEN_FACODEC_V2 = {
    "a": (_ENC, dict(fqo.GOLDEN_FACODEC_QUANTIZE["a"][0]), 2, 24 * 200, None),
    "b": (_ENC, dict(fqo.GOLDEN_FACODEC_QUANTIZE["b"][0]), 2, 7 * 200, 1),
}
PREFIXES = ("quantizer.", "timbre_encoder.", "melspec_linear.", "melspec_encoder.", "timbre_linear.")


def perturb(named_parameters, seed):
    """Redraw the quantizers', both transformers', melspec_linear's and timbre_linear's parameters in state-dict order:
    the quantizers and the timbre encoder as facodec_quantize_oracle.perturb draws them, melspec_encoder by the same
    rules from seed + 1, melspec_linear (Linear 20 -> 256) and timbre_linear (gamma around 1, beta around 0) from
    seed + 2.  timbre_linear is redrawn because a module's constructor draws it after the transformers, whose
    construction consumes the random stream differently in the reference and in the product."""
    params = list(named_parameters)
    fqo.perturb(params, seed)
    fqo.perturb([("timbre_encoder." + n[len("melspec_encoder."):], p) for n, p in params
                 if n.startswith("melspec_encoder.")], seed + 1)
    g = torch.Generator().manual_seed(seed + 2)
    with torch.no_grad():
        for n, p in params:
            if n == "melspec_linear.weight":
                p.copy_(torch.randn(p.shape, generator=g) / math.sqrt(BINS))
            elif n == "melspec_linear.bias":
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
            elif n == "timbre_linear.weight":
                p.copy_(torch.randn(p.shape, generator=g) * (0.5 / math.sqrt(p.shape[1])))
            elif n == "timbre_linear.bias":
                c = p.shape[0] // 2
                p.copy_(torch.randn(p.shape, generator=g) * 0.1 + torch.cat([torch.ones(c), torch.zeros(c)]))


def digests(sd):
    """SHA-256 of every redrawn tensor (fp32 bytes), by name."""
    d = fqo.digests(sd)
    d.update(fqo.digests({"timbre_encoder." + k: v for k, v in sd.items() if k.startswith(PREFIXES[2:])}))
    return d


def prosody_stream(sd, pf, dtype=torch.float64, return_layers=False):
    """melspec_encoder(melspec_linear(pf^T))^T (facodec.py:1034-1038) -> [B, 256, T]; with return_layers also each
    layer's output [B, T, 256]."""
    pf = fqo._t(pf, dtype)
    lin = pf.transpose(1, 2) @ fqo._t(sd["melspec_linear.weight"], dtype).T + fqo._t(sd["melspec_linear.bias"], dtype)
    enc = {"timbre_encoder." + k[len("melspec_encoder."):]: v for k, v in sd.items() if k.startswith("melspec_encoder.")}
    _, layers = fqo.timbre(enc, lin.transpose(1, 2), dtype=dtype, return_layers=True)
    y = F.layer_norm(layers[-1], (lin.shape[-1],), fqo._t(sd["melspec_encoder.last_ln.weight"], dtype),
                     fqo._t(sd["melspec_encoder.last_ln.bias"], dtype), 1e-5)
    y = y.transpose(1, 2)
    return (y, layers) if return_layers else y


def quantize(sd, x, prosody, nq, n_quantizers=None, forced=None):
    """facodec.py:1029-1062 in float64: fqo.quantize with the prosody group reading `prosody`.  Returns outs, qs, the
    groups' sums and the best / runner-up gaps."""
    x, prosody = fqo._t(x), fqo._t(prosody)
    k = max(nq) if n_quantizers is None else n_quantizers
    outs, qs, bufs, gaps, row = 0, [], [], [], 0
    for gi, q0, n in fqo._groups(nq):
        inp = prosody if gi == 0 else x if gi == 1 else x - (bufs[0] + bufs[1])
        r, acc = inp.permute(0, 2, 1), 0
        for j in range(min(k, n)):
            pre = f"quantizer.{gi}.layers.{j}."
            z_e = r @ fqo._weight(sd, pre + "in_proj").T + fqo._t(sd[pre + "in_proj.bias"])
            cb = fqo._t(sd[pre + "_codebook.weight"])
            e = z_e / torch.clamp(torch.linalg.norm(z_e, dim=-1, keepdim=True), min=1e-12)
            cn = cb / torch.clamp(torch.linalg.norm(cb, dim=-1, keepdim=True), min=1e-12)
            dist = (e * e).sum(-1, keepdim=True) - 2 * e @ cn.T + (cn * cn).sum(-1)[None, None, :]
            srt = torch.sort(dist, dim=-1).values
            gaps.append(srt[..., 1] - srt[..., 0] if cb.shape[0] > 1 else torch.full(srt.shape[:2], math.inf))
            code = torch.argmin(dist, dim=-1) if forced is None else fqo._t(forced[row], torch.int64)
            qs.append(code)
            q = cb[code] @ fqo._weight(sd, pre + "out_proj").T + fqo._t(sd[pre + "out_proj.bias"])
            r, acc = r - q, acc + q
            row += 1
        buf = acc.permute(0, 2, 1)
        bufs.append(buf)
        outs = outs + buf
    return outs, torch.stack(qs), bufs, torch.stack(gaps)


def quantize_kernel_order(sd, x, prosody, nq, n_quantizers=None):
    """The V2 RVQ in the kernel's fp32 operation order (numpy float32) for one-hot projections, as
    fqo.quantize_kernel_order: the prosody group starts from `prosody`, the residual group from x - (prosody sum +
    content sum).  Codes are the float64 argmin; among exactly equal distances the lowest code."""
    x, prosody = np.asarray(x, np.float32), np.asarray(prosody, np.float32)
    k = max(nq) if n_quantizers is None else n_quantizers
    qs, bufs = [], []
    for gi, q0, n in fqo._groups(nq):
        r = prosody.copy() if gi == 0 else x.copy() if gi == 1 else (x - (bufs[0] + bufs[1]).astype(np.float32)).astype(np.float32)
        acc = np.zeros_like(x)
        for j in range(min(k, n)):
            pre = f"quantizer.{gi}.layers.{j}."
            w_in = fqo._weight(sd, pre + "in_proj").numpy().astype(np.float32)
            w_out = fqo._weight(sd, pre + "out_proj").numpy().astype(np.float32)
            b_in = np.asarray(sd[pre + "in_proj.bias"], np.float32)
            b_out = np.asarray(sd[pre + "out_proj.bias"], np.float32)
            cb = np.asarray(sd[pre + "_codebook.weight"], np.float32)
            z_e = (np.einsum("dc,bct->btd", w_in, r).astype(np.float32) + b_in).astype(np.float32)
            e = z_e.astype(np.float64)
            e = e / np.maximum(np.linalg.norm(e, axis=-1, keepdims=True), 1e-12)
            c64 = cb.astype(np.float64)
            cn = c64 / np.maximum(np.linalg.norm(c64, axis=-1, keepdims=True), 1e-12)
            code = np.argmin((e * e).sum(-1, keepdims=True) - 2 * e @ cn.T + (cn * cn).sum(-1), axis=-1)
            qs.append(code)
            z_q = (z_e + (cb[code] - z_e).astype(np.float32)).astype(np.float32)
            q = (np.einsum("cd,btd->bct", w_out, z_q).astype(np.float32) + b_out[None, :, None]).astype(np.float32)
            r = (r - q).astype(np.float32)
            acc = (acc + q).astype(np.float32)
        bufs.append(acc)
    outs = (bufs[0] + bufs[1]).astype(np.float32)
    if len(bufs) > 2:
        outs = (outs + bufs[2]).astype(np.float32)
    return outs, np.stack(qs).astype(np.int64), bufs


def prosody_input_exact(w, bias, pe, pf):
    """The prosody input kernel's fp32 operation order: per (b, c, t) an FMA chain over the 20 rows from 0, + bias[c],
    + pe[b][c], each step rounded to fp32 (the FMA exactly, by diffwave_exact_oracle.fma)."""
    import diffwave_exact_oracle as dxo
    w, bias, pf = np.asarray(w, np.float32), np.asarray(bias, np.float32), np.asarray(pf, np.float32)
    pe = np.asarray(pe, np.float32).reshape(-1, w.shape[0])
    B, _, T = pf.shape
    a = np.zeros((B, w.shape[0], T), np.float32)
    for i in range(BINS):
        a = dxo.fma(np.broadcast_to(w[None, :, i, None], a.shape), np.broadcast_to(pf[:, i:i + 1, :], a.shape), a)
    a = (a + bias[None, :, None]).astype(np.float32)
    return (a + pe[:B, :, None]).astype(np.float32)
