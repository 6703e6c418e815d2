"""Benchmark MaskGCT's acoustic codec (models/tts/maskgct/config/maskgct.json: d_model 96, ratios [3, 4, 5, 8], 256
channels; 12 quantizers of 1024 x 8; Vocos 512 / 4096 / 30 layers, n_fft 1920, hop 480) on B utterances of 10 s at
24 kHz: the three calls of a MaskGCT synthesis, each timed natively at every precision and as the reference's op
sequence run eagerly in torch.nn.functional (cuDNN, fp32, TF32 off and on):

- encode: CodecEncoder.forward(wav);
- quantize: CodecDecoder.quantize(latent) (the prompt's codes, maskgct_utils.py:124-127);
- decode: CodecDecoder.vq2emb(codes) then CodecDecoder.forward (maskgct_utils.py:223-230).

Weights are seeded, with the biases and Snake1d alphas redrawn (the reference's init zeroes the biases).  The card's
name, power limit and the median SM clock over the timed windows come from read-only nvidia-smi queries; one JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from amphion_b200.vocoders import CodecDecoder, CodecEncoder  # noqa: E402
from bench_melgan import ClockSampler, card, time_steps  # noqa: E402
from bench_vocos import eager_backbone, eager_head  # noqa: E402

ENC = dict(d_model=96, up_ratios=[3, 4, 5, 8], out_channels=256)
DEC = dict(in_channels=256, num_quantizers=12, codebook_size=1024, codebook_dim=8, quantizer_type="fvq",
           use_l2_normlize=True, use_vocos=True, vocos_dim=512, vocos_intermediate_dim=4096, vocos_num_layers=30,
           n_fft=1920, hop_size=480)


def snake(x, alpha):
    """codec.py:34-39."""
    return x + (alpha + 1e-9).reciprocal() * torch.sin(alpha * x).pow(2)


def eager_encode(m, x):
    """CodecEncoder.forward (codec.py:60-143) after remove_weight_norm."""
    seq = m.block
    x = F.conv1d(x, seq[0].weight, seq[0].bias, padding=3)
    for i, s in enumerate(m.up_ratios):
        blk = seq[1 + i].block
        for ru in blk[:3]:
            b = ru.block
            h = F.conv1d(snake(x, b[0].alpha), b[1].weight, b[1].bias, dilation=b[1].dilation, padding=b[1].padding)
            x = x + F.conv1d(snake(h, b[2].alpha), b[3].weight, b[3].bias)
        x = F.conv1d(snake(x, blk[3].alpha), blk[4].weight, blk[4].bias, stride=s, padding=(s + 1) // 2)
    n = len(m.up_ratios)
    return F.conv1d(snake(x, seq[1 + n].alpha), seq[2 + n].weight, seq[2 + n].bias, padding=1)


def eager_quantize(rvq, z, n):
    """ResidualVQ.forward in eval (residual_vq.py:69-134, factorized_vector_quantize.py:52-129)."""
    out, r, codes = 0.0, z, []
    for q in rvq.quantizers[:n]:
        z_e = F.conv1d(r, q.in_project.weight, q.in_project.bias)
        e = F.normalize(z_e.transpose(1, 2).reshape(-1, z_e.shape[1]))
        cb = F.normalize(q.codebook.weight)
        dist = e.pow(2).sum(1, keepdim=True) - 2 * e @ cb.t() + cb.pow(2).sum(1, keepdim=True).t()
        idx = (-dist).max(1)[1].view(z.shape[0], -1)
        z_q = F.embedding(idx, q.codebook.weight).transpose(1, 2)
        z_q = F.conv1d(z_e + (z_q - z_e), q.out_project.weight, q.out_project.bias)
        out, r = out + z_q, r - z_q
        codes.append(idx)
    return out, torch.stack(codes)


def eager_decode(dec, codes, n):
    """ResidualVQ.vq2emb (residual_vq.py:136-144), then Vocos.forward."""
    emb = 0.0
    for i, q in enumerate(dec.quantizer.quantizers[:n]):
        emb = emb + F.conv1d(F.embedding(codes[i], q.codebook.weight).transpose(1, 2), q.out_project.weight,
                             q.out_project.bias)
    return eager_head(dec.model, eager_backbone(dec.model, emb))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_amphion_codec: needs a CUDA device")
    torch.manual_seed(0)
    enc, dec = CodecEncoder(**ENC).eval(), CodecDecoder(**DEC).eval()
    with torch.no_grad():
        g = torch.Generator().manual_seed(2)
        for m in (enc, dec):
            for name, p in m.named_parameters():
                if name.endswith(".alpha"):
                    p.copy_((torch.rand(p.shape, generator=g) + 0.3) * torch.where(torch.rand(p.shape, generator=g) < 0.3, -1.0, 1.0))
                elif name.endswith("bias"):
                    p.copy_(torch.randn(p.shape, generator=g) * 0.1)
    enc.remove_weight_norm()
    enc, dec = enc.cuda(), dec.cuda()
    n_samples = int(a.seconds * 24000)
    x = torch.randn(a.batch, 1, n_samples, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1)) * 0.3
    nq = DEC["num_quantizers"]
    sampler = ClockSampler()
    res = dict(workload="maskgct_acoustic_codec", batch=a.batch, samples=n_samples, frames=enc.frames(n_samples),
               steps=a.steps, warmup=a.warmup)
    res["card"], res["power_limit"] = card()
    with torch.no_grad():
        for prec in ("tc_f16", "tc_bf16", "fp32"):
            for m in (enc, dec.quantizer, dec.model):
                m.precision = prec
            z = enc(x)
            qo, codes = dec.quantize(z)
            r = dict(encode_ms=time_steps(lambda: enc(x), a.steps, a.warmup, sampler),
                     quantize_ms=time_steps(lambda: dec.quantize(z), a.steps, a.warmup, sampler),
                     decode_ms=time_steps(lambda: dec(dec.vq2emb(codes)), a.steps, a.warmup, sampler))
            res[prec] = {k: round(v, 3) for k, v in r.items()}
            if prec == "fp32":
                native = (z, codes, dec(dec.vq2emb(codes)))
        wn = CodecDecoder(**DEC).eval()   # eager needs the folded weights of the quantizer's projections
        wn.load_state_dict(dec.state_dict())
        for q in wn.quantizer.quantizers:
            torch.nn.utils.remove_weight_norm(q.in_project)
            torch.nn.utils.remove_weight_norm(q.out_project)
        wn = wn.cuda()
        z32, codes32, y32 = native
        for tf32 in (False, True):
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32
            r = dict(encode_ms=time_steps(lambda: eager_encode(enc, x), a.steps, a.warmup, sampler),
                     quantize_ms=time_steps(lambda: eager_quantize(wn.quantizer, z32, nq), a.steps, a.warmup, sampler),
                     decode_ms=time_steps(lambda: eager_decode(wn, codes32, nq), a.steps, a.warmup, sampler))
            key = "eager_tf32" if tf32 else "eager_fp32"
            res[key] = {k: round(v, 3) for k, v in r.items()}
            if not tf32:
                ze = eager_encode(enc, x)
                _, ce = eager_quantize(wn.quantizer, z32, nq)
                ye = eager_decode(wn, codes32, nq)
                res["fp32_vs_eager_fp32"] = dict(
                    encode_rel=float((z32 - ze).abs().max() / ze.abs().max()),
                    codes_differing=int((ce != codes32).sum()), codes=int(codes32.numel()),
                    decode_rel=float((y32 - ye).abs().max() / ye.abs().max()))
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    res["median_sm_clock_mhz"] = sampler.median()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
