"""Time FACodecDecoder.inference at the README geometry (models/codec/ns3_codec/README.md: in_channels 256,
upsample_initial_channel 1024, up_ratios [5, 5, 4, 2]) on cuda:0, B = 16 latents of 800 frames (10 s of 16 kHz audio
each), against the decoder's op sequence restated eagerly in torch.nn.functional (cuDNN, fp32 with TF32 off and on),
and print one JSON line.

    python scripts/bench_facodec.py [--batch 16] [--frames 800] [--steps 5] [--warmup 2]

ms per step come from CUDA events around `steps` inference calls after `warmup` untimed ones; the per-class profile of
the C ABI from one extra profiled call.  The card's name, power limit and the median SM clock over the timed windows come
from read-only nvidia-smi queries."""
import argparse
import json
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from amphion_b200.vocoders import FACodecDecoder  # noqa: E402
from bench_melgan import ClockSampler, card, time_steps  # noqa: E402

HP = dict(in_channels=256, upsample_initial_channel=1024, ngf=32, up_ratios=[5, 5, 4, 2], vq_num_q_c=2, vq_num_q_p=1,
          vq_num_q_r=3, vq_dim=256, codebook_dim=8, codebook_size_prosody=10, codebook_size_content=10,
          codebook_size_residual=10, use_gr_x_timbre=True, use_gr_residual_f0=True, use_gr_residual_phone=True)


def eager_act(a, x):
    """Activation1d(SnakeBeta(alpha_logscale=True)) (alias_free_torch/act.py, resample.py, filter.py)."""
    c = x.shape[1]
    fu = a.upsample.filter.expand(c, -1, -1)
    fd = a.downsample.lowpass.filter.expand(c, -1, -1)
    x = 2 * F.conv_transpose1d(F.pad(x, (5, 5), mode="replicate"), fu, stride=2, groups=c)[..., 15:-15]
    al = torch.exp(a.act.alpha)[None, :, None]
    be = torch.exp(a.act.beta)[None, :, None]
    x = x + (1.0 / (be + 1e-9)) * torch.pow(torch.sin(x * al), 2)
    return F.conv1d(F.pad(x, (5, 6), mode="replicate"), fd, stride=2, groups=c)


def eager_inference(m, x, spk):
    """FACodecDecoder.inference (facodec.py:568-576) after remove_weight_norm."""
    style = F.linear(spk, m.timbre_linear.weight, m.timbre_linear.bias).unsqueeze(2)
    gamma, beta = style.chunk(2, 1)
    x = F.layer_norm(x.transpose(1, 2), (m.in_channels,), eps=1e-5).transpose(1, 2) * gamma + beta
    seq = m.model
    x = F.conv1d(x, seq[0].weight, seq[0].bias, padding=3)
    for i, u in enumerate(m.up_ratios):
        blk = seq[1 + i].block
        ct = blk[1]
        x = F.conv_transpose1d(eager_act(blk[0], x), ct.weight, ct.bias, stride=u, padding=u // 2 + u % 2,
                               output_padding=u % 2)
        for ru in blk[2:]:
            b = ru.block
            h = F.conv1d(eager_act(b[0], x), b[1].weight, b[1].bias, dilation=b[1].dilation, padding=b[1].padding)
            x = x + F.conv1d(eager_act(b[2], h), b[3].weight, b[3].bias)
    n = len(m.up_ratios)
    return torch.tanh(F.conv1d(eager_act(seq[1 + n], x), seq[2 + n].weight, seq[2 + n].bias, padding=3))


def flops_per_frame(hp):
    """2 x MACs of every convolution, per latent frame."""
    c, t, macs = hp["upsample_initial_channel"], 1, hp["in_channels"] * hp["upsample_initial_channel"] * 7
    for u in hp["up_ratios"]:
        co = c // 2
        macs += t * u * c * co * 2      # ConvTranspose1d(k = 2u, stride u): 2 taps per output sample
        t *= u
        macs += t * 3 * (co * co * 7 + co * co)
        c = co
    macs += t * c * 7
    return 2.0 * macs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--frames", type=int, default=800)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_facodec: needs a CUDA device")
    torch.manual_seed(0)
    model = FACodecDecoder(**HP).eval()
    model.remove_weight_norm()
    model = model.cuda()
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(a.batch, HP["in_channels"], a.frames, device="cuda", generator=g)
    spk = torch.randn(a.batch, HP["in_channels"], device="cuda", generator=g)
    samples = a.batch * a.frames * model.hop_length
    flop = flops_per_frame(HP) * a.batch * a.frames
    sampler = ClockSampler()
    res = dict(workload="facodec_readme", batch=a.batch, frames=a.frames, steps=a.steps, warmup=a.warmup,
               gflop_per_frame=round(flops_per_frame(HP) / 1e9, 3), tflop_per_step=round(flop / 1e12, 2))
    res["card"], res["power_limit"] = card()
    outs = {}
    with torch.no_grad():
        for prec in ("tc_f16", "tc_bf16", "fp32"):
            model.precision = prec
            ms = time_steps(lambda: model.inference(x, spk), a.steps, a.warmup, sampler)
            model.set_profiling(True)
            outs[prec] = model.inference(x, spk)
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
            ms = time_steps(lambda: eager_inference(model, x, spk), a.steps, a.warmup, sampler)
            key = "eager_tf32" if tf32 else "eager_fp32"
            res[key] = dict(ms_per_step=round(ms, 3), samples_per_s=round(samples / ms * 1e3))
            if not tf32:
                ref = eager_inference(model, x, spk)
                for prec, o in outs.items():
                    res[prec]["max_abs_diff_vs_eager_fp32"] = float((o - ref).abs().max())
                res["eager_fp32"]["peak"] = float(ref.abs().max())
                del ref
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    res["median_sm_clock_mhz"] = sampler.median()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
