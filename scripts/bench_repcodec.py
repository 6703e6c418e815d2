"""Benchmark MaskGCT's semantic codec (models/tts/maskgct/config/maskgct.json: RepCodec with hidden 1024, Vocos
backbones 384 / 2048 / 12 layers, one quantizer of 8192 x 8) on B utterances of 10 s of 50 Hz w2v-BERT features
(500 frames): the two calls of the codec, each timed natively at every precision and as the reference's op sequence
run eagerly in torch.nn.functional (cuDNN / cuBLAS, fp32 with TF32 off and on, and under autocast fp16):

- quantize: RepCodec.quantize(feat) (the prompt's semantic codes, maskgct_utils.py:111-121);
- forward: RepCodec.forward(feat) (encoder, quantizer, decoder).

Weights are seeded, with the biases, LayerNorm affines and layer scales redrawn (the reference's init zeroes the
biases).  The card's name, power limit and the median SM clock over the timed windows come from read-only nvidia-smi
queries; one JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from amphion_b200.vocoders import RepCodec  # noqa: E402
from bench_melgan import ClockSampler, card, time_steps  # noqa: E402

CODEC = dict(codebook_size=8192, hidden_size=1024, codebook_dim=8, vocos_dim=384, vocos_intermediate_dim=2048,
             vocos_num_layers=12)


def eager_vocos_linear(seq, x):
    """nn.Sequential(VocosBackbone, nn.Linear) (kmeans/vocos.py:764-783, repcodec_model.py:108-127): [B, C, T] ->
    [B, T, out]."""
    bb, lin = seq[0], seq[1]
    dim = bb.embed.weight.shape[0]
    x = F.conv1d(x, bb.embed.weight, bb.embed.bias, padding=3)
    x = F.layer_norm(x.transpose(1, 2), (dim,), bb.norm.weight, bb.norm.bias, 1e-6).transpose(1, 2)
    for blk in bb.convnext:
        h = F.conv1d(x, blk.dwconv.weight, blk.dwconv.bias, padding=3, groups=dim).transpose(1, 2)
        h = F.layer_norm(h, (dim,), blk.norm.weight, blk.norm.bias, 1e-6)
        h = F.linear(F.gelu(F.linear(h, blk.pwconv1.weight, blk.pwconv1.bias)), blk.pwconv2.weight, blk.pwconv2.bias)
        x = x + (blk.gamma * h).transpose(1, 2)
    x = F.layer_norm(x.transpose(1, 2), (dim,), bb.final_layer_norm.weight, bb.final_layer_norm.bias, 1e-6)
    return F.linear(x, lin.weight, lin.bias)


def eager_quantize(rvq, z):
    """One FactorizedVectorQuantize layer of ResidualVQ.forward in eval (factorized_vector_quantize.py:52-129), on the
    folded weights."""
    q = rvq.quantizers[0]
    z_e = F.conv1d(z, q.in_project.weight, q.in_project.bias)
    e = F.normalize(z_e.transpose(1, 2).reshape(-1, z_e.shape[1]))
    cb = F.normalize(q.codebook.weight)
    dist = e.pow(2).sum(1, keepdim=True) - 2 * e @ cb.t() + cb.pow(2).sum(1, keepdim=True).t()
    idx = (-dist).max(1)[1].view(z.shape[0], -1)
    z_q = F.embedding(idx, q.codebook.weight).transpose(1, 2)
    return F.conv1d(z_e + (z_q - z_e), q.out_project.weight, q.out_project.bias), idx


def eager_codec(m, x, decode):
    """RepCodec.quantize (decode False: codes, quantized) or RepCodec.forward (decode True: x_rec, codes)."""
    h = eager_vocos_linear(m.encoder, x.transpose(1, 2)).transpose(1, 2)
    qo, idx = eager_quantize(m.quantizer, h.float())
    if decode:
        return eager_vocos_linear(m.decoder, qo), idx
    return idx, qo.transpose(1, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_repcodec: needs a CUDA device")
    torch.manual_seed(0)
    m = RepCodec(**CODEC).eval()
    with torch.no_grad():
        g = torch.Generator().manual_seed(2)
        for name, p in m.named_parameters():
            if name.endswith(".bias") or name.endswith(".gamma"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
            elif name.endswith("norm.weight"):
                p.copy_(1.0 + torch.randn(p.shape, generator=g) * 0.1)
    m = m.cuda()
    frames = int(a.seconds * 50)
    x = torch.randn(a.batch, frames, CODEC["hidden_size"], device="cuda",
                    generator=torch.Generator(device="cuda").manual_seed(1))
    sampler = ClockSampler()
    res = dict(workload="maskgct_semantic_codec", batch=a.batch, frames=frames, steps=a.steps, warmup=a.warmup)
    res["card"], res["power_limit"] = card()
    with torch.no_grad():
        for prec in ("tc_f16", "tc_bf16", "fp32"):
            m.precision = prec
            r = dict(quantize_ms=time_steps(lambda: m.quantize(x), a.steps, a.warmup, sampler),
                     forward_ms=time_steps(lambda: m(x), a.steps, a.warmup, sampler))
            res[prec] = {k: round(v, 3) for k, v in r.items()}
            res[prec]["launches_forward"] = m.last_launches
            if prec == "fp32":
                codes32, _ = m.quantize(x)
                rec32 = m(x)[0]
        wn = RepCodec(**CODEC).eval()   # eager needs the folded weights of the quantizer's projections
        wn.load_state_dict(m.state_dict())
        for q in wn.quantizer.quantizers:
            torch.nn.utils.remove_weight_norm(q.in_project)
            torch.nn.utils.remove_weight_norm(q.out_project)
        wn = wn.cuda()
        for key, tf32, amp in (("eager_fp32", False, False), ("eager_tf32", True, False), ("eager_autocast_f16", False, True)):
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32
            with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
                r = dict(quantize_ms=time_steps(lambda: eager_codec(wn, x, False), a.steps, a.warmup, sampler),
                         forward_ms=time_steps(lambda: eager_codec(wn, x, True), a.steps, a.warmup, sampler))
                res[key] = {k: round(v, 3) for k, v in r.items()}
                if key == "eager_fp32":
                    ce, _ = eager_codec(wn, x, False)
                    re_, _ = eager_codec(wn, x, True)
                    res["fp32_vs_eager_fp32"] = dict(codes_differing=int((ce != codes32).sum()), codes=int(codes32.numel()),
                                                     x_rec_rel=float((rec32 - re_).abs().max() / re_.abs().max()))
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    res["median_sm_clock_mhz"] = sampler.median()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
