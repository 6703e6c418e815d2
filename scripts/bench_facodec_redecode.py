"""Time FACodecRedecoder (the README's zero-shot voice conversion) at the released geometry (1280 channels, up_ratios
(5, 5, 4, 2), 1 + 2 + 3 tables of 2^10) on cuda:0: vq2emb(vq, spk, use_residual=False) and inference for B = 16
utterances of 800 frames (10 s at 16 kHz), against the same computation restated eagerly in torch.nn.functional (fp32
with TF32 off and on), then the whole A -> B conversion at tc_f16 (the encoder and forward(vq=True) on both utterance
batches, vq2emb and inference); one JSON line.

    python scripts/bench_facodec_redecode.py [--batch 16] [--frames 800] [--steps 5] [--warmup 2]

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

from amphion_b200.vocoders import FACodecDecoder, FACodecEncoder, FACodecRedecoder  # noqa: E402
from bench_facodec import eager_inference  # noqa: E402
from bench_facodec_quantize import ENC, HP as DEC_HP, init as init_decoder  # noqa: E402
from bench_melgan import ClockSampler, card, time_steps  # noqa: E402


def init(m, seed):
    """Trained-like scales for the embedding tables and the prosody transformer (the reference draws the tables at std
    1e-5, starts every style Linear at gamma = 1, beta = 0 and the FFN at 0.02), and the reference's positional
    encoding.  The generator keeps its constructor's weights."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if not name.startswith(("prosody_embs.", "content_embs.", "residual_embs.", "timbre_cond_prosody_enc.")):
                continue
            fan_in = p.shape[1] * (p.shape[2] if p.dim() > 2 else 1) if p.dim() > 1 else 1
            if name.startswith(("prosody_embs.", "content_embs.", "residual_embs.")):
                p.copy_(torch.randn(p.shape, generator=g))
            elif name.endswith(".style.weight"):
                p.copy_(torch.randn(p.shape, generator=g) * (0.3 / math.sqrt(fan_in)))
            elif name.endswith(".style.bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
                p[:p.shape[0] // 2] += 1.0
            elif name.endswith("weight"):
                p.copy_(torch.randn(p.shape, generator=g) / math.sqrt(fan_in))
            else:
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
        pe = m.timbre_cond_prosody_enc.position_emb.pe
        pos = torch.arange(pe.shape[0]).unsqueeze(1)
        div = torch.exp(torch.arange(0, 256, 2) * (-math.log(10000.0) / 256))
        pe[:, 0, 0::2] = torch.sin(pos * div)
        pe[:, 0, 1::2] = torch.cos(pos * div)
    m.invalidate()


def saln(ln, h, spk):
    """StyleAdaptiveLayerNorm (transformer.py:22-32) with the condition spk expanded over time, as the reference."""
    cond = spk.unsqueeze(1).expand(-1, h.shape[1], -1).mean(dim=1, keepdim=True)
    gamma, beta = F.linear(cond, ln.style.weight, ln.style.bias).chunk(2, -1)
    return gamma * F.layer_norm(h, (h.shape[-1],), eps=1e-5) + beta


def eager_vq2emb(m, vq, spk, use_residual=False):
    """FACodecRedecoder.vq2emb (facodec.py:734-759) in eval."""
    enc = m.timbre_cond_prosody_enc
    x_t = 0
    for i, e in enumerate(m.prosody_embs):
        x_t = x_t + F.embedding(vq[i], e.weight)
        h = x_t + enc.position_emb.pe[:x_t.shape[0]]
        for layer in enc.layers:
            a = saln(layer.ln_1, h, spk)
            h = h + layer.self_attn(a, a, a, need_weights=False)[0]
            a = saln(layer.ln_2, h, spk)
            f = F.relu(F.conv1d(a.transpose(1, 2), layer.ffn.ffn_1.weight, layer.ffn.ffn_1.bias, padding=2))
            h = h + F.linear(f.transpose(1, 2), layer.ffn.ffn_2.weight, layer.ffn.ffn_2.bias)
        x_t = saln(enc.last_ln, h, spk)
    out = x_t
    p, c = len(m.prosody_embs), len(m.content_embs)
    for i, e in enumerate(m.content_embs):
        out = out + F.embedding(vq[p + i], e.weight)
    if use_residual:
        for i, e in enumerate(m.residual_embs):
            out = out + F.embedding(vq[p + c + i], e.weight)
    return out.transpose(1, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--frames", type=int, default=800)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_facodec_redecode: needs a CUDA device")
    torch.manual_seed(0)
    red = FACodecRedecoder().eval()
    init(red, 3)
    red.remove_weight_norm()
    red = red.cuda()
    B, T = a.batch, a.frames
    g = torch.Generator(device="cuda").manual_seed(1)
    vq = torch.randint(0, 1024, (6, B, T), device="cuda", generator=g)
    spk = torch.randn(B, 256, device="cuda", generator=g)
    sampler = ClockSampler()
    res = dict(workload="facodec_redecoder_released", batch=B, frames=T, steps=a.steps, warmup=a.warmup,
               samples=T * red.hop_length)
    res["card"], res["power_limit"] = card()

    def prof_dict(prof):
        return {k: dict(launches=v["launches"], ms=round(v["ms"], 3), gflop=round(v["flops"] / 1e9, 2),
                        gb=round(v["bytes"] / 1e9, 3)) for k, v in prof.items() if v["launches"]}

    outs = {}
    with torch.no_grad():
        for prec in ("tc_f16", "tc_bf16", "fp32"):
            red.precision = prec
            ms_e = time_steps(lambda: red.vq2emb(vq, spk, use_residual=False), a.steps, a.warmup, sampler)
            red.set_profiling(True)
            emb = red.vq2emb(vq, spk, use_residual=False)
            prof_e = red.get_profile()
            launches_e = red.last_launches
            red.set_profiling(False)
            ms_i = time_steps(lambda: red.inference(emb, spk), a.steps, a.warmup, sampler)
            red.set_profiling(True)
            wav = red.inference(emb, spk)
            prof_i = red.get_profile()
            red.set_profiling(False)
            outs[prec] = (emb, wav)
            res[prec] = dict(vq2emb=dict(ms_per_call=round(ms_e, 3), launches=launches_e, profile=prof_dict(prof_e)),
                             inference=dict(ms_per_call=round(ms_i, 3), launches=red.last_launches,
                                            profile=prof_dict(prof_i)))
        for tf32 in (False, True):
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32
            ms_e = time_steps(lambda: eager_vq2emb(red, vq, spk), a.steps, a.warmup, sampler)
            emb_ref = eager_vq2emb(red, vq, spk)
            ms_i = time_steps(lambda: eager_inference(red, emb_ref, spk), a.steps, a.warmup, sampler)
            key = "eager_tf32" if tf32 else "eager_fp32"
            res[key] = dict(vq2emb_ms_per_call=round(ms_e, 3), inference_ms_per_call=round(ms_i, 3))
            if not tf32:
                wav_ref = eager_inference(red, emb_ref, spk)
                for prec, (emb, wav) in outs.items():
                    res[prec]["max_abs_diff_emb_vs_eager_fp32"] = float((emb - emb_ref).abs().max())
                    res[prec]["max_abs_diff_wav_vs_eager_fp32"] = float((wav - wav_ref).abs().max())
                res["eager_fp32"]["peak_emb"] = float(emb_ref.abs().max())
                res["eager_fp32"]["peak_wav"] = float(wav_ref.abs().max())
                del wav_ref
            del emb_ref
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
        del outs
        # the README conversion A -> B at tc_f16: encode both batches, quantize both, redecode A's codes in B's voice
        torch.manual_seed(0)
        enc = FACodecEncoder(**ENC).eval().cuda()
        dec = FACodecDecoder(**DEC_HP).eval()
        init_decoder(dec, 4)
        dec = dec.cuda()
        enc.precision = dec.precision = red.precision = "tc_f16"
        wav_a = torch.randn(B, 1, T * 200, device="cuda", generator=g) * 0.3
        wav_b = torch.randn(B, 1, T * 200, device="cuda", generator=g) * 0.3

        def convert():
            _, vq_a, _, _, _ = dec(enc(wav_a), eval_vq=False, vq=True)
            _, _, _, _, spk_b = dec(enc(wav_b), eval_vq=False, vq=True)
            return red.inference(red.vq2emb(vq_a, spk_b, use_residual=False), spk_b)

        ms = time_steps(convert, a.steps, a.warmup, sampler)
        res["conversion_a_to_b_tc_f16"] = dict(ms_per_call=round(ms, 3), samples=T * 200)
    res["median_sm_clock_mhz"] = sampler.median()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
