"""Time DiffWave at the recipe geometry (egs/vocoder/diffusion/diffwave: 64 residual channels, 30 layers, dilation cycle
10, upsample factors [16, 16], 100 mels, 24 kHz) for one 10 s utterance (938 frames, L = 240,128 samples) and for B = 8:
  - native fp32, tc_f16 and tc_bf16,
  - a reference-equivalent eager PyTorch model of diffwave.py on the same GPU, fp32 with TF32 off and under autocast fp16.
Per configuration: ms per denoising step (one network pass plus the sampler update), the totals for the 6-step
fast_inference schedule and the 50-step schedule (the native conditioning is added once per call), per-kernel-class time
from the profile hook, and the share of the per-step lower bound computed from shapes: max(FLOPs / peak, HBM bytes /
3.35 TB/s) with the peak 67 TFLOP/s (fp32) or 989 TFLOP/s (fp16 / bf16 tensor cores, tc_* and autocast rows), naming
which bound applies (H100 SXM data-sheet rates).  Prints the card and its power limit.

    python scripts/bench_diffwave.py [--batches 1,8] [--seconds 10] [--iters 3]"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from diffwave_oracle import HP_DIFFWAVE_RECIPE, diffwave_cfg  # noqa: E402

N_MEL, HOP, SR = 100, 256, 24000
PEAK_FP32, PEAK_TC, PEAK_BW = 67e12, 989e12, 3.35e12   # dense fp32 / fp16-bf16 tensor FLOP/s, HBM3 B/s


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"{torch.cuda.get_device_name()} (nvidia-smi failed: {e})"
    return q


def build_model():
    from amphion_b200.vocoders import DiffWave
    torch.manual_seed(0)
    m = DiffWave(diffwave_cfg(HP_DIFFWAVE_RECIPE, N_MEL))
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for name, p in m.named_parameters():
            p.copy_(torch.randn(p.shape, generator=g) * (0.1 if name.endswith("bias") else 1.0 / p[0].numel() ** 0.5))
    return m.cuda().eval()


def step_cost(B, L):
    """FLOPs and compulsory HBM bytes of one network pass + update, from shapes (fp32 activations)."""
    C, nl, nm = 64, HP_DIFFWAVE_RECIPE["residual_layers"], N_MEL
    el = B * L
    flops = el * (2 * C + nl * 2 * 2 * C * (3 * C + nm + C) + 2 * (C * C + C))
    # per layer: x read + write, skip read + write (stored by layer 0), upsampled mel read; input / tail passes
    bytes_ = 4 * el * (nl * (4 * C + nm) - C + (1 + C) + (C + 3))
    return flops, bytes_


def eager_forward(m, audio, step, cond, emb_table):
    """diffwave.py's forward with the module's parameters, eager PyTorch ops (the reference's arithmetic)."""
    x = F.relu(F.conv1d(audio.unsqueeze(1), m.input_projection.weight, m.input_projection.bias))
    lo, hi = torch.floor(step).long(), torch.ceil(step).long()
    e = emb_table[lo] + (emb_table[hi] - emb_table[lo]) * (step - lo)
    de = m.diffusion_embedding
    h = F.silu(F.linear(F.silu(F.linear(e, de.projection1.weight, de.projection1.bias)), de.projection2.weight, de.projection2.bias))
    skip = None
    for layer in m.residual_layers:
        d = F.linear(h, layer.diffusion_projection.weight, layer.diffusion_projection.bias).unsqueeze(-1)
        dil = layer.dilated_conv.dilation[0]
        y = F.conv1d(x + d, layer.dilated_conv.weight, layer.dilated_conv.bias, padding=dil, dilation=dil)
        y = y + F.conv1d(cond, layer.conditioner_projection.weight, layer.conditioner_projection.bias)
        gate, filt = torch.chunk(y, 2, dim=1)
        y = F.conv1d(torch.sigmoid(gate) * torch.tanh(filt), layer.output_projection.weight, layer.output_projection.bias)
        res, s = torch.chunk(y, 2, dim=1)
        x = (x + res) / math.sqrt(2.0)
        skip = s if skip is None else s + skip
    x = F.relu(F.conv1d(skip / math.sqrt(len(m.residual_layers)), m.skip_projection.weight, m.skip_projection.bias))
    return F.conv1d(x, m.output_projection.weight, m.output_projection.bias)


def eager_upsample(m, mel):
    up = m.spectrogram_upsampler
    x = F.leaky_relu(F.conv_transpose2d(mel.unsqueeze(1), up.conv1.weight, up.conv1.bias, stride=up.conv1.stride,
                                        padding=up.conv1.padding), 0.4)
    return F.leaky_relu(F.conv_transpose2d(x, up.conv2.weight, up.conv2.bias, stride=up.conv2.stride,
                                           padding=up.conv2.padding), 0.4).squeeze(1)


def time_cuda(fn, iters):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def bench_native(m, B, frames, iters):
    from amphion_b200.vocoders.diffusion_vocoder_inference import noise_schedule
    L = frames * HOP
    mel = torch.randn(B, N_MEL, frames, device="cuda")
    audio = torch.randn(B, L, device="cuda").clamp_(-1, 1)
    noise = torch.randn(B, L, device="cuda")
    T = noise_schedule(m.cfg, True)[0]
    ws, need = m._condition(mel, T)
    step_ms = time_cuda(lambda: m._step(audio, 3, 1.01, 0.2, 0.1, noise, ws, need), iters)
    cond_ms = {}
    for n, fast in ((6, True), (50, False)):
        Tn = noise_schedule(m.cfg, fast)[0]
        cond_ms[n] = time_cuda(lambda: m._condition(mel, Tn), iters)
    m.set_profiling(True)
    m._step(audio, 3, 1.01, 0.2, 0.1, noise, *m._condition(mel, T))
    prof = {k: round(v["ms"], 3) for k, v in m.get_profile().items() if v["launches"]}
    m.set_profiling(False)
    return step_ms, cond_ms, prof


def bench_eager(m, B, frames, iters, autocast):
    L = frames * HOP
    mel = torch.randn(B, N_MEL, frames, device="cuda")
    audio = torch.randn(B, L, device="cuda").clamp_(-1, 1)
    noise = torch.randn(B, L, device="cuda")
    table = m.diffusion_embedding.embedding.cuda()
    step = torch.tensor([3.3], device="cuda")

    def one():
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16, enabled=autocast):
            # the reference recomputes the upsampler inside every network pass
            eps = eager_forward(m, audio, step, eager_upsample(m, mel), table).squeeze(1)
            a = 1.01 * (audio - 0.2 * eps.float())
            a += 0.1 * noise
            return torch.clamp(a, -1.0, 1.0)
    return time_cuda(one, iters)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,8")
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--iters", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_diffwave.py needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    frames = int(round(args.seconds * SR / HOP))
    m = build_model()
    print(json.dumps({"card": card(), "frames": frames, "samples": frames * HOP}))
    for B in (int(b) for b in args.batches.split(",")):
        flops, bytes_ = step_cost(B, frames * HOP)
        rows = []
        for prec in ("fp32", "tc_f16", "tc_bf16"):
            m.precision = prec
            step_ms, cond_ms, prof = bench_native(m, B, frames, args.iters)
            rows.append(dict(config=f"native {prec}", ms_per_step=step_ms, total_6=6 * step_ms + cond_ms[6],
                             total_50=50 * step_ms + cond_ms[50], profile_ms=prof))
        for ac, name in ((False, "eager fp32 (TF32 off)"), (True, "eager autocast fp16")):
            t = bench_eager(m, B, frames, args.iters, ac)
            rows.append(dict(config=name, ms_per_step=t, total_6=6 * t, total_50=50 * t))
        for r in rows:
            tc = "tc_" in r["config"] or "fp16" in r["config"]
            peak = PEAK_TC if tc else PEAK_FP32
            bound_s = max(flops / peak, bytes_ / PEAK_BW)
            bound = ("fp16 tensor" if tc else "fp32") + " compute" if flops / peak >= bytes_ / PEAK_BW else "HBM bandwidth"
            r.update(B=B, step_gflop=flops / 1e9, step_gbytes=bytes_ / 1e9, lower_bound_ms=bound_s * 1e3, bound=bound)
            if r["ms_per_step"]:
                r["share_of_lower_bound"] = bound_s * 1e3 / r["ms_per_step"]
            print(json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in r.items()}))
            sys.stdout.flush()


if __name__ == "__main__":
    t0 = time.time()
    main()
    print(f"# wall {time.time() - t0:.1f} s")
