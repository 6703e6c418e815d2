"""Time FACodecEncoder.forward at the README geometry (models/codec/ns3_codec/README.md: ngf 32, up_ratios [2, 4, 5, 5],
out_channels 256) on cuda:0, B = 16 waveforms of 160 000 samples (10 s at 16 kHz), against the encoder's op sequence
restated eagerly in torch.nn.functional (cuDNN, fp32 with TF32 off and on), and print one JSON line.

    python scripts/bench_facodec_encode.py [--batch 16] [--samples 160000] [--steps 5] [--warmup 2]

ms per step come from CUDA events around `steps` forward calls after `warmup` untimed ones; the per-class profile of the
C ABI from one extra profiled call.  The card's name, power limit and the median SM clock over the timed windows come
from read-only nvidia-smi queries.  Quantization and the timbre encoder (the rest of the README's encode step) are not
served natively and are not timed."""
import argparse
import json
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from amphion_b200.vocoders import FACodecEncoder  # noqa: E402
from bench_facodec import eager_act  # noqa: E402
from bench_melgan import ClockSampler, card, time_steps  # noqa: E402

HP = dict(ngf=32, up_ratios=[2, 4, 5, 5], out_channels=256)


def eager_encode(m, x):
    """FACodecEncoder.forward (facodec.py:121-194) after remove_weight_norm."""
    seq = m.block
    x = F.conv1d(x, seq[0].weight, seq[0].bias, padding=3)
    for i, s in enumerate(m.up_ratios):
        blk = seq[1 + i].block
        for ru in blk[:3]:
            b = ru.block
            h = F.conv1d(eager_act(b[0], x), b[1].weight, b[1].bias, dilation=b[1].dilation, padding=b[1].padding)
            x = x + F.conv1d(eager_act(b[2], h), b[3].weight, b[3].bias)
        x = F.conv1d(eager_act(blk[3], x), blk[4].weight, blk[4].bias, stride=s, padding=s // 2 + s % 2)
    n = len(m.up_ratios)
    return F.conv1d(eager_act(seq[1 + n], x), seq[2 + n].weight, seq[2 + n].bias, padding=1)


def flops(hp, n):
    """2 x MACs of every convolution for one waveform of n samples."""
    c, t = hp["ngf"], n
    macs = t * c * 7
    for s in hp["up_ratios"]:
        macs += t * 3 * (c * c * 7 + c * c)
        t = (t + 2 * (s // 2 + s % 2) - 2 * s) // s + 1
        macs += t * c * 2 * c * 2 * s
        c *= 2
    macs += t * c * hp["out_channels"] * 3
    return 2.0 * macs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--samples", type=int, default=160000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_facodec_encode: needs a CUDA device")
    torch.manual_seed(0)
    model = FACodecEncoder(**HP).eval()
    model.remove_weight_norm()
    with torch.no_grad():   # the reference initialises the biases to 0 and SnakeBeta at alpha = beta = 0 (log scale)
        g = torch.Generator().manual_seed(2)
        for name, p in model.named_parameters():
            if name.endswith(("bias", ".alpha", ".beta")):
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
    model = model.cuda()
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(a.batch, 1, a.samples, device="cuda", generator=g) * 0.3
    samples = a.batch * a.samples
    flop = flops(HP, a.samples) * a.batch
    sampler = ClockSampler()
    res = dict(workload="facodec_encoder_readme", batch=a.batch, samples=a.samples, frames=model.frames(a.samples),
               steps=a.steps, warmup=a.warmup, tflop_per_step=round(flop / 1e12, 3))
    res["card"], res["power_limit"] = card()
    outs = {}
    with torch.no_grad():
        for prec in ("tc_f16", "tc_bf16", "fp32"):
            model.precision = prec
            ms = time_steps(lambda: model(x), a.steps, a.warmup, sampler)
            model.set_profiling(True)
            outs[prec] = model(x)
            prof = model.get_profile()
            model.set_profiling(False)
            res[prec] = dict(ms_per_step=round(ms, 3), samples_per_s=round(samples / ms * 1e3),
                             tflop_per_s=round(flop / ms / 1e9, 1), launches=model.last_launches,
                             profile={k: dict(launches=v["launches"], ms=round(v["ms"], 3),
                                              tflop=round(v["flops"] / 1e12, 3), gb=round(v["bytes"] / 1e9, 3))
                                      for k, v in prof.items() if v["launches"]})
        for tf32 in (False, True):
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32
            ms = time_steps(lambda: eager_encode(model, x), a.steps, a.warmup, sampler)
            key = "eager_tf32" if tf32 else "eager_fp32"
            res[key] = dict(ms_per_step=round(ms, 3), samples_per_s=round(samples / ms * 1e3))
            if not tf32:
                ref = eager_encode(model, x)
                for prec, o in outs.items():
                    res[prec]["max_abs_diff_vs_eager_fp32"] = float((o - ref).abs().max())
                res["eager_fp32"]["peak"] = float(ref.abs().max())
                del ref
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    res["median_sm_clock_mhz"] = sampler.median()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
