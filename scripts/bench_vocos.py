"""Time Vocos.forward at the recipe geometry of Vevo's vocoder (models/vc/vevo/config/Vocoder.json: 128 mels, dim
1024, intermediate 4096, 30 ConvNeXt layers, n_fft 1920, hop 480) on cuda:0, against the reference's op sequence in
eager torch (cuBLAS / cuDNN, fp32 with TF32 off and on, and the backbone under autocast fp16 with the head in fp32 —
cuFFT's half precision does not serve n_fft 1920), and print one JSON line.

    python scripts/bench_vocos.py [--batch 64] [--frames 1024] [--steps 5] [--warmup 2]

ms per step come from CUDA events around `steps` forwards after `warmup` untimed ones; the per-class profile of the
C ABI (and the pointwise GEMMs' achieved TFLOP/s) from one extra profiled forward.  The card's name, power limit and
the median SM clock over the timed windows come from read-only nvidia-smi queries."""
import argparse
import json
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from amphion_b200.vocoders import Vocos  # noqa: E402
from bench_melgan import ClockSampler, card, time_steps  # noqa: E402

HP = dict(input_channels=128, dim=1024, intermediate_dim=4096, num_layers=30, n_fft=1920, hop_size=480)


def eager_backbone(m, x):
    """VocosBackbone.forward (vocos.py:762-783) as the reference's torch calls on the module's parameters."""
    bb = m.backbone
    x = F.conv1d(x, bb.embed.weight, bb.embed.bias, padding=3)
    x = F.layer_norm(x.transpose(1, 2), (m.dim,), bb.norm.weight, bb.norm.bias, 1e-6).transpose(1, 2)
    for blk in bb.convnext:
        h = F.conv1d(x, blk.dwconv.weight, blk.dwconv.bias, padding=3, groups=m.dim).transpose(1, 2)
        h = F.layer_norm(h, (m.dim,), blk.norm.weight, blk.norm.bias, 1e-6)
        h = F.linear(F.gelu(F.linear(h, blk.pwconv1.weight, blk.pwconv1.bias)), blk.pwconv2.weight, blk.pwconv2.bias)
        x = x + (blk.gamma * h).transpose(1, 2)
    return F.layer_norm(x.transpose(1, 2), (m.dim,), bb.final_layer_norm.weight, bb.final_layer_norm.bias, 1e-6)


def eager_head(m, x):
    """ISTFTHead + ISTFT "same" (vocos.py:129-167, :343-361)."""
    x = F.linear(x.float(), m.head.out.weight, m.head.out.bias).transpose(1, 2)
    mag, p = x.chunk(2, dim=1)
    S = torch.clip(torch.exp(mag), max=1e2) * (torch.cos(p) + 1j * torch.sin(p))
    n_fft, hop, window = m.n_fft, m.hop_length, m.head.istft.window
    pad = (n_fft - hop) // 2
    T = S.shape[-1]
    ifft = torch.fft.irfft(S, n_fft, dim=1, norm="backward") * window[None, :, None]
    size = (T - 1) * hop + n_fft
    y = F.fold(ifft, output_size=(1, size), kernel_size=(1, n_fft), stride=(1, hop))[:, 0, 0, pad:-pad]
    env = F.fold(window.square().expand(1, T, -1).transpose(1, 2), output_size=(1, size), kernel_size=(1, n_fft),
                 stride=(1, hop)).squeeze()[pad:-pad]
    return (y / env)[:, None, :]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--frames", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vocos: needs a CUDA device")
    torch.manual_seed(0)
    model = Vocos(**HP).eval().cuda()
    g = torch.Generator(device="cuda").manual_seed(1)
    # Vevo calls vocoder_model(mel.transpose(1, 2)): a transposed view of [B, L, n_mels]
    mel = (torch.rand(a.batch, a.frames, HP["input_channels"], device="cuda", generator=g) * 13.5 - 11.5).transpose(1, 2)
    samples = a.batch * a.frames * HP["hop_size"]
    flop = 2.0 * a.batch * a.frames * HP["dim"] * (7 * HP["input_channels"] + 2 * HP["num_layers"] * HP["intermediate_dim"]
                                                   + HP["n_fft"] + 2)
    sampler = ClockSampler()
    res = dict(workload="vocos_recipe", batch=a.batch, frames=a.frames, steps=a.steps, warmup=a.warmup,
               tflop_per_step=round(flop / 1e12, 2))
    res["card"], res["power_limit"] = card()
    outs = {}
    with torch.no_grad():
        for prec in ("tc_f16", "tc_bf16", "fp32"):
            model.precision = prec
            ms = time_steps(lambda: model(mel), a.steps, a.warmup, sampler)
            model.set_profiling(True)
            outs[prec] = model(mel)
            prof = model.get_profile()
            model.set_profiling(False)
            res[prec] = dict(ms_per_step=round(ms, 3), samples_per_s=round(samples / ms * 1e3),
                             launches=model.last_launches,
                             profile={k: dict(launches=v["launches"], ms=round(v["ms"], 3),
                                              tflop=round(v["flops"] / 1e12, 3), gb=round(v["bytes"] / 1e9, 3))
                                      for k, v in prof.items() if v["launches"]})
            pw = prof.get("tc_pointwise", {})
            if pw.get("launches"):
                res[prec]["pointwise_tflop_per_s"] = round(pw["flops"] / pw["ms"] / 1e9, 1)
        for tf32 in (False, True):
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32
            ms = time_steps(lambda: eager_head(model, eager_backbone(model, mel)), a.steps, a.warmup, sampler)
            key = "eager_tf32" if tf32 else "eager_fp32"
            res[key] = dict(ms_per_step=round(ms, 3), samples_per_s=round(samples / ms * 1e3))
            if not tf32:
                ref = eager_head(model, eager_backbone(model, mel))
                for prec, o in outs.items():
                    res[prec]["max_abs_diff_vs_eager_fp32"] = float((o - ref).abs().max())
                res["eager_fp32"]["peak"] = float(ref.abs().max())
                del ref
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False

        def autocast_step():
            with torch.autocast("cuda", dtype=torch.float16):
                feat = eager_backbone(model, mel)
            return eager_head(model, feat)

        ms = time_steps(autocast_step, a.steps, a.warmup, sampler)
        res["eager_autocast_f16_backbone"] = dict(ms_per_step=round(ms, 3), samples_per_s=round(samples / ms * 1e3))
    res["median_sm_clock_mhz"] = sampler.median()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
