"""Time FACodecDecoder.forward(vq=True) (quantization, the timbre encoder and the speaker embedding) at the README
geometry (models/codec/ns3_codec/README.md: in_channels 256, 1 + 2 + 3 codebooks of 2^10 x 8) on cuda:0, B = 16 latents
of 800 frames (10 s at 16 kHz), against the same computation restated eagerly in torch.nn.functional (fp32 with TF32
off and on), then the whole README round trip (encoder, forward(vq=True), vq2emb, inference) at tc_f16; one JSON line.

    python scripts/bench_facodec_quantize.py [--batch 16] [--frames 800] [--steps 5] [--warmup 2]

ms per call come from CUDA events around `steps` calls after `warmup` untimed ones; the per-class profile of the C ABI
from one extra profiled call.  The card's name, power limit and the median SM clock over the timed windows come from
read-only nvidia-smi queries."""
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

from amphion_b200.vocoders import FACodecDecoder, FACodecEncoder  # noqa: E402
from bench_melgan import ClockSampler, card, time_steps  # noqa: E402

HP = dict(in_channels=256, upsample_initial_channel=1024, ngf=32, up_ratios=[5, 5, 4, 2], vq_num_q_c=2, vq_num_q_p=1,
          vq_num_q_r=3, vq_dim=256, codebook_dim=8, codebook_size_prosody=10, codebook_size_content=10,
          codebook_size_residual=10)
ENC = dict(ngf=32, up_ratios=[2, 4, 5, 5], out_channels=256)


def init(m, seed):
    """Trained-like scales for the quantizers and the timbre encoder (the reference's 0.02 FFN init and zero biases
    would leave the residual branches negligible), and the reference's positional encoding."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if not name.startswith(("quantizer.", "timbre_encoder.")):
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
        pe = m.timbre_encoder.position_emb.pe
        pos = torch.arange(pe.shape[0]).unsqueeze(1)
        div = torch.exp(torch.arange(0, 256, 2) * (-math.log(10000.0) / 256))
        pe[:, 0, 0::2] = torch.sin(pos * div)
        pe[:, 0, 1::2] = torch.cos(pos * div)
    m.invalidate()


def wn(lin):
    return torch._weight_norm(lin.weight_v, lin.weight_g, 0)


def eager(m, x):
    """facodec.py:408-471 in eval: the ResidualVQs (fvq.py:52-91) and the timbre encoder (transformer.py:206-217)."""
    outs, qs, bufs = 0, [], []
    for gi, rvq in enumerate(m.quantizer):
        r = x if gi < 2 else x - (bufs[0] + bufs[1])
        acc = 0
        for layer in rvq.layers:
            z_e = F.linear(r.transpose(1, 2), wn(layer.in_proj), layer.in_proj.bias)
            cb = layer._codebook.weight
            e, cn = F.normalize(z_e.reshape(-1, z_e.shape[-1])), F.normalize(cb)
            dist = e.pow(2).sum(1, keepdim=True) - 2 * e @ cn.t() + cn.pow(2).sum(1, keepdim=True).t()
            code = (-dist).max(1)[1].reshape(z_e.shape[:2])
            z_q = z_e + (F.embedding(code, cb) - z_e)
            q = F.linear(z_q, wn(layer.out_proj), layer.out_proj.bias).transpose(1, 2)
            r, acc = r - q, acc + q
            qs.append(code)
        bufs.append(acc)
        outs = outs + acc
    te = m.timbre_encoder
    h = x.transpose(1, 2) + te.position_emb.pe[:x.shape[0]]
    for layer in te.layers:
        a = F.layer_norm(h, (256,), layer.ln_1.weight, layer.ln_1.bias, 1e-5)
        h = h + layer.self_attn(a, a, a, need_weights=False)[0]
        a = F.layer_norm(h, (256,), layer.ln_2.weight, layer.ln_2.bias, 1e-5)
        f = F.relu(F.conv1d(a.transpose(1, 2), layer.ffn.ffn_1.weight, layer.ffn.ffn_1.bias, padding=2))
        h = h + F.linear(f.transpose(1, 2), layer.ffn.ffn_2.weight, layer.ffn.ffn_2.bias)
    y = F.layer_norm(h, (256,), te.last_ln.weight, te.last_ln.bias, 1e-5)
    return outs, torch.stack(qs), bufs, y.mean(1)


def flops(B, T):
    """GEMMs, attention and the RVQ's projections and distances, 2 x MACs."""
    gemm = 2.0 * B * T * 4 * (256 * 768 + 256 * 256 + 256 * 1024 * 5 + 1024 * 256)
    attn = 4 * 1024.0 * B * T * T
    rvq = 2.0 * B * T * 6 * (256 * 8 + 8 * 256 + 1024 * 8)
    return gemm, attn, rvq


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--frames", type=int, default=800)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_facodec_quantize: needs a CUDA device")
    torch.manual_seed(0)
    model = FACodecDecoder(**HP).eval()
    init(model, 3)
    model = model.cuda()
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(a.batch, 256, a.frames, device="cuda", generator=g)
    gemm, attn, rvq = flops(a.batch, a.frames)
    sampler = ClockSampler()
    res = dict(workload="facodec_quantize_readme", batch=a.batch, frames=a.frames, steps=a.steps, warmup=a.warmup,
               gflop_gemm=round(gemm / 1e9, 1), gflop_attention=round(attn / 1e9, 1), gflop_rvq=round(rvq / 1e9, 2))
    res["card"], res["power_limit"] = card()
    outs = {}
    with torch.no_grad():
        for prec in ("tc_f16", "tc_bf16", "fp32"):
            model.precision = prec
            ms = time_steps(lambda: model(x, vq=True), a.steps, a.warmup, sampler)
            model.set_profiling(True)
            outs[prec] = model(x, vq=True)
            prof = model.get_profile()
            model.set_profiling(False)
            res[prec] = dict(ms_per_call=round(ms, 3), launches=model.last_launches,
                             profile={k: dict(launches=v["launches"], ms=round(v["ms"], 3),
                                              gflop=round(v["flops"] / 1e9, 2), gb=round(v["bytes"] / 1e9, 3))
                                      for k, v in prof.items() if v["launches"]})
        for tf32 in (False, True):
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32
            ms = time_steps(lambda: eager(model, x), a.steps, a.warmup, sampler)
            key = "eager_tf32" if tf32 else "eager_fp32"
            res[key] = dict(ms_per_call=round(ms, 3))
            if not tf32:
                ref = eager(model, x)
                for prec, o in outs.items():
                    res[prec]["codes_differing_from_eager_fp32"] = int((o[1] != ref[1]).sum())
                    res[prec]["max_abs_diff_outs_vs_eager_fp32"] = float((o[0] - ref[0]).abs().max())
                    res[prec]["max_abs_diff_spk_vs_eager_fp32"] = float((o[4] - ref[3]).abs().max())
                res["eager_fp32"]["peak_outs"] = float(ref[0].abs().max())
                res["eager_fp32"]["peak_spk"] = float(ref[3].abs().max())
                del ref
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
        # the README round trip at tc_f16: wav -> encoder -> forward(vq=True) -> vq2emb -> inference
        torch.manual_seed(0)
        enc = FACodecEncoder(**ENC).eval().cuda()
        enc.precision = model.precision = "tc_f16"
        wav = torch.randn(a.batch, 1, a.frames * 200, device="cuda", generator=g) * 0.3

        def round_trip():
            h = enc(wav)
            _, qs, _, _, spk = model(h, vq=True)
            return model.inference(model.vq2emb(qs), spk)

        ms = time_steps(round_trip, a.steps, a.warmup, sampler)
        res["readme_round_trip_tc_f16"] = dict(ms_per_call=round(ms, 3), samples=a.frames * 200)
    res["median_sm_clock_mhz"] = sampler.median()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
