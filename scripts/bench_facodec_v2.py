"""Time FACodec V2 (models/codec/ns3_codec/facodec.py:772-1199) at the README geometry on cuda:0: B = 16 waveforms of
10 s at 16 kHz (800 frames at hop 200), FACodecEncoderV2.get_prosody_feature, FACodecDecoderV2.forward(x,
prosody_feature, vq=True) with its per-class profile, and the README's whole A -> B conversion (encoder and prosody
feature on both batches, forward(vq=True) x 2, vq2emb(codes of A, use_residual=False), inference with B's speaker
embedding), at each precision; forward(vq=True) against the same computation restated eagerly (fp32 with TF32 off and
on), with the codes that differ from eager fp32.  One JSON line.

    python scripts/bench_facodec_v2.py [--batch 16] [--frames 800] [--steps 5] [--warmup 2]

ms per call come from CUDA events around `steps` calls after `warmup` untimed ones.  The card's name, power limit and
the median SM clock over the timed windows come from read-only nvidia-smi queries."""
import argparse
import json
import math
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from amphion_b200.vocoders import FACodecDecoderV2, FACodecEncoderV2  # noqa: E402
from bench_facodec_quantize import ENC, HP  # noqa: E402
from bench_melgan import ClockSampler, card, time_steps  # noqa: E402


def init(m, seed):
    """bench_facodec_quantize.init's scales for the quantizers and both transformers, and the positional encodings."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if not name.startswith(("quantizer.", "timbre_encoder.", "melspec_encoder.", "melspec_linear.")):
                continue
            fan_in = p.shape[1] * (p.shape[2] if p.dim() > 2 else 1) if p.dim() > 1 else 1
            if name.endswith("weight_g"):
                p.copy_(torch.rand(p.shape, generator=g) * 0.6 + 0.6)
            elif name.endswith(("weight_v", "_codebook.weight")):
                p.copy_(torch.randn(p.shape, generator=g))
            elif ".ln_" in name or "last_ln" in name:
                p.copy_(1.0 + 0.2 * torch.randn(p.shape, generator=g) if name.endswith("weight")
                        else 0.1 * torch.randn(p.shape, generator=g))
            elif name.endswith("weight"):
                p.copy_(torch.randn(p.shape, generator=g) / math.sqrt(fan_in))
            else:
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
        pos = torch.arange(5000).unsqueeze(1)
        div = torch.exp(torch.arange(0, 256, 2) * (-math.log(10000.0) / 256))
        for te in (m.timbre_encoder, m.melspec_encoder):
            pe = te.position_emb.pe
            pe[:, 0, 0::2] = torch.sin(pos * div)
            pe[:, 0, 1::2] = torch.cos(pos * div)
    m.invalidate()


def transformer(te, h):
    """transformer.py:206-234 on [B, T, 256] (eval): pe[:B], 4 pre-LN layers, last_ln."""
    h = h + te.position_emb.pe[:h.shape[0]]
    for layer in te.layers:
        a = F.layer_norm(h, (256,), layer.ln_1.weight, layer.ln_1.bias, 1e-5)
        h = h + layer.self_attn(a, a, a, need_weights=False)[0]
        a = F.layer_norm(h, (256,), layer.ln_2.weight, layer.ln_2.bias, 1e-5)
        f = F.relu(F.conv1d(a.transpose(1, 2), layer.ffn.ffn_1.weight, layer.ffn.ffn_1.bias, padding=2))
        h = h + F.linear(f.transpose(1, 2), layer.ffn.ffn_2.weight, layer.ffn.ffn_2.bias)
    return F.layer_norm(h, (256,), te.last_ln.weight, te.last_ln.bias, 1e-5)


def eager(m, x, pf):
    """facodec.py:1027-1094 in eval: the prosody transformer, the RVQ with the prosody group reading its output, and the
    timbre encoder's time mean."""
    P = transformer(m.melspec_encoder, F.linear(pf.transpose(1, 2), m.melspec_linear.weight, m.melspec_linear.bias))
    P = P.transpose(1, 2)
    qs, bufs = [], []
    for gi, rvq in enumerate(m.quantizer):
        r = P if gi == 0 else x if gi == 1 else x - (bufs[0] + bufs[1])
        acc = 0
        for layer in rvq.layers:
            w_in = torch._weight_norm(layer.in_proj.weight_v, layer.in_proj.weight_g, 0)
            w_out = torch._weight_norm(layer.out_proj.weight_v, layer.out_proj.weight_g, 0)
            z_e = F.linear(r.transpose(1, 2), w_in, layer.in_proj.bias)
            cb = layer._codebook.weight
            e, cn = F.normalize(z_e.reshape(-1, z_e.shape[-1])), F.normalize(cb)
            dist = e.pow(2).sum(1, keepdim=True) - 2 * e @ cn.t() + cn.pow(2).sum(1, keepdim=True).t()
            code = (-dist).max(1)[1].reshape(z_e.shape[:2])
            q = F.linear(z_e + (F.embedding(code, cb) - z_e), w_out, layer.out_proj.bias).transpose(1, 2)
            r, acc = r - q, acc + q
            qs.append(code)
        bufs.append(acc)
    spk = transformer(m.timbre_encoder, x.transpose(1, 2)).mean(1)
    return sum(bufs), torch.stack(qs), bufs, spk


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--frames", type=int, default=800)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_facodec_v2: needs a CUDA device")
    torch.manual_seed(0)
    dec = FACodecDecoderV2(**HP).eval()
    init(dec, 3)
    enc = FACodecEncoderV2(**ENC).eval()
    dec, enc = dec.cuda(), enc.cuda()
    g = torch.Generator(device="cuda").manual_seed(1)
    N = a.frames * 200
    wav_a = torch.randn(a.batch, 1, N, device="cuda", generator=g) * 0.3
    wav_b = torch.randn(a.batch, 1, N, device="cuda", generator=g) * 0.3
    sampler = ClockSampler()
    res = dict(workload="facodec_v2_readme", batch=a.batch, frames=a.frames, samples=N, steps=a.steps, warmup=a.warmup)
    res["card"], res["power_limit"] = card()
    outs = {}
    with torch.no_grad():
        res["get_prosody_feature"] = dict(ms_per_call=round(time_steps(lambda: enc.get_prosody_feature(wav_a), a.steps,
                                                                       a.warmup, sampler), 3))
        pf = enc.get_prosody_feature(wav_a)
        for prec in ("tc_f16", "tc_bf16", "fp32"):
            enc.precision = dec.precision = prec
            x = enc(wav_a)
            T = min(x.shape[2], pf.shape[2])   # trim to the common frame count, as a caller must
            x, p = x[:, :, :T].contiguous(), pf[:, :, :T].contiguous()
            ms = time_steps(lambda: dec(x, p, vq=True), a.steps, a.warmup, sampler)
            dec.set_profiling(True)
            dec(x, p, vq=True)
            prof = dec.get_profile()
            dec.set_profiling(False)
            res[prec] = dict(frames=T, ms_per_call=round(ms, 3), launches=dec.last_launches,
                             profile={k: dict(launches=v["launches"], ms=round(v["ms"], 3),
                                              gflop=round(v["flops"] / 1e9, 2), gb=round(v["bytes"] / 1e9, 3))
                                      for k, v in prof.items() if v["launches"]})

            def convert():
                ha, hb = enc(wav_a), enc(wav_b)
                pa, pb = enc.get_prosody_feature(wav_a), enc.get_prosody_feature(wav_b)
                ta, tb = min(ha.shape[2], pa.shape[2]), min(hb.shape[2], pb.shape[2])
                _, qa, _, _, _ = dec(ha[:, :, :ta], pa[:, :, :ta], vq=True)
                _, _, _, _, spk_b = dec(hb[:, :, :tb], pb[:, :, :tb], vq=True)
                return dec.inference(dec.vq2emb(qa, use_residual=False), spk_b)

            res[prec]["readme_conversion_ms"] = round(time_steps(convert, a.steps, a.warmup, sampler), 3)
        # the code comparison reads the fp32 encoder's latent at every precision
        for prec in ("tc_f16", "tc_bf16", "fp32"):
            dec.precision = prec
            outs[prec] = dec(x, p, vq=True)
        for tf32 in (False, True):
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32
            ms = time_steps(lambda: eager(dec, x, p), a.steps, a.warmup, sampler)
            res["eager_tf32" if tf32 else "eager_fp32"] = dict(ms_per_call=round(ms, 3))
            if not tf32:
                ref = eager(dec, x, p)
                for prec, o in outs.items():
                    res[prec]["codes_differing_from_eager_fp32"] = int((o[1] != ref[1]).sum())
                    res[prec]["max_abs_diff_outs_vs_eager_fp32"] = float((o[0] - ref[0]).abs().max())
                    res[prec]["max_abs_diff_spk_vs_eager_fp32"] = float((o[4] - ref[3]).abs().max())
                res["eager_fp32"]["peak_outs"] = float(ref[0].abs().max())
                del ref
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    res["median_sm_clock_mhz"] = sampler.median()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
