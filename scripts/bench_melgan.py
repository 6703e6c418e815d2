"""Time MelGAN.forward at the recipe geometry (egs/vocoder/gan/melgan/exp_config.json: ratios [8, 8, 2, 2], ngf 32,
3 residual layers; 100 mels) on cuda:0, against the same op sequence in eager torch.nn.functional (cuDNN), and print
one JSON line.

    python scripts/bench_melgan.py [--batch 64] [--frames 1024] [--steps 20] [--warmup 3]

ms per step come from CUDA events around `steps` forwards after `warmup` untimed ones; the per-class profile of the
C ABI from one extra profiled forward.  The card's name, power limit and the median SM clock over the timed windows
come from read-only nvidia-smi queries."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
from types import SimpleNamespace as NS

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from amphion_b200.vocoders import MelGAN  # noqa: E402

HP = dict(ratios=[8, 8, 2, 2], ngf=32, n_residual_layers=3)
N_MEL = 100


def eager_forward(w, mel):
    """The generator as eager torch.nn.functional calls on folded weights (the rival)."""
    R, n = HP["n_residual_layers"], len(HP["ratios"])
    x = F.conv1d(F.pad(mel, (3, 3), mode="reflect"), *w[1])
    for i, r in enumerate(HP["ratios"]):
        base = 2 + i * (2 + R)
        x = F.conv_transpose1d(F.leaky_relu(x, 0.2), *w[base + 1], stride=r, padding=r // 2 + r % 2,
                               output_padding=r % 2)
        for j in range(R):
            d, blk = 3 ** j, base + 2 + j
            h = F.conv1d(F.pad(F.leaky_relu(x, 0.2), (d, d), mode="reflect"), *w[f"{blk}.block.2"], dilation=d)
            h = F.conv1d(F.leaky_relu(h, 0.2), *w[f"{blk}.block.4"])
            x = F.conv1d(x, *w[f"{blk}.shortcut"]) + h
    x = F.pad(F.leaky_relu(x, 0.2), (3, 3), mode="reflect")
    return torch.tanh(F.conv1d(x, *w[2 + n * (2 + R) + 2]))


def folded_weights(model):
    w = {}
    for name, m in model.model.named_modules():
        if hasattr(m, "weight_v"):
            key = int(name) if name.isdigit() else name
            w[key] = (torch._weight_norm(m.weight_v, m.weight_g, 0).detach(), m.bias.detach())
    return w


class ClockSampler:
    """nvidia-smi's SM clock every 100 ms while timing (read-only query); the process ends with stop()."""

    def __init__(self):
        self.f = tempfile.NamedTemporaryFile("w+", suffix=".csv", delete=False)
        self.proc = None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", "0", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits",
                                          "-lms", "100"], stdout=self.f, stderr=subprocess.DEVNULL)
        except OSError:
            self.proc = None

    def stop(self):
        if self.proc is not None:
            self.proc.terminate()
            self.proc.wait()
            self.proc = None

    def median(self):
        self.f.seek(0)
        vals = sorted(int(v) for v in self.f.read().split() if v.strip().isdigit())
        os.unlink(self.f.name)
        return vals[len(vals) // 2] if vals else None


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "not measured"


def time_steps(fn, steps, warmup, sampler):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    sampler.start()
    try:
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
    finally:   # the sampling process never outlives the timed window, also when fn() raises
        sampler.stop()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--frames", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_melgan: needs a CUDA device")
    torch.manual_seed(0)
    cfg = NS(preprocess=NS(n_mel=N_MEL, hop_size=256), model=NS(generator="melgan", melgan=NS(**HP)))
    model = MelGAN(cfg).eval().cuda()
    g = torch.Generator(device="cuda").manual_seed(1)
    mel = torch.rand(a.batch, N_MEL, a.frames, device="cuda", generator=g) * 13.5 - 11.5
    samples = a.batch * a.frames * 256
    sampler = ClockSampler()
    res = dict(workload="melgan_recipe", batch=a.batch, frames=a.frames, steps=a.steps, warmup=a.warmup)
    res["card"], res["power_limit"] = card()
    outs = {}
    with torch.no_grad():
        for prec in ("tc_f16", "fp32"):
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
        w = folded_weights(model)
        for tf32 in (False, True):
            torch.backends.cudnn.allow_tf32 = tf32
            torch.backends.cuda.matmul.allow_tf32 = tf32
            ms = time_steps(lambda: eager_forward(w, mel), a.steps, a.warmup, sampler)
            ref = eager_forward(w, mel)
            key = "eager_cudnn_tf32" if tf32 else "eager_cudnn_fp32"
            res[key] = dict(ms_per_step=round(ms, 3), samples_per_s=round(samples / ms * 1e3))
            if not tf32:
                for prec, o in outs.items():
                    res[prec]["max_abs_diff_vs_eager_fp32"] = float((o - ref).abs().max())
    res["median_sm_clock_mhz"] = sampler.median()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
