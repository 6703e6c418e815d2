#!/usr/bin/env python
"""Per-stage device-time split of one HiFi-GAN V1 generator step (bench.py config 2 by default) from a torch.profiler
trace with CUDA activities.

    python scripts/profile_stages.py [--batch 64] [--frames 1024] [--fusion 2] [--out DIR]

The tensor-core launches of `forward_impl` come in a fixed order: conv_pre, then per stage one ConvTranspose and per
ResBlock either one block-mode launch (`hchain_kernel`) or one `hpair_kernel` launch per dilation pair; conv_pre and
the ConvTranspose layers run on `hconv_kernel`.  The script
walks that order, attributes each tensor-core launch to (stage, plan) and prints time, share of the step, achieved
TFLOP/s and algorithmic GB/s per row.  Algorithmic bytes per ResBlock launch: the 16-bit operand image and the fp32
residual read, the fp32 output and its operand image written, the running branch sum read when it is accumulated, and
the weights once; ConvTranspose: fp32 in, fp32 out and its image; conv_pre: mel in, fp32 out.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from collections import OrderedDict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import HOP, WORKLOADS, make_cfg  # noqa: E402


def plan_rows(hp, n_mel, B, T):
    """(stage, plan, flops, bytes) of each tensor-core launch group, in launch order, with a callback deciding
    block versus pair per ResBlock from the trace."""
    C0 = hp["upsample_initial_channel"]
    rows = [("conv_pre", "conv", 2.0 * B * T * C0 * n_mel * 7, 4.0 * B * T * (n_mel + C0))]
    cin, Tn = C0, T
    for i, (u, k) in enumerate(zip(hp["upsample_rates"], hp["upsample_kernel_sizes"])):
        cout = cin // 2
        rows.append((f"stage {i}", "convT", 2.0 * B * cout * Tn * u * cin * k / u,
                     4.0 * B * cin * Tn + 10.0 * B * cout * Tn * u + 2.0 * cin * cout * k))
        Tn *= u
        el = float(B) * cout * Tn
        for j, (kk, dil) in enumerate(zip(hp["resblock_kernel_sizes"], hp["resblock_dilation_sizes"])):
            acc = 4.0 * el if j > 0 else 0.0
            per_pair = [(2.0 * el * cout * kk * 2, 12.0 * el + acc * (q == len(dil) - 1) + 2.0 * 2 * cout * cout * kk)
                        for q in range(len(dil))]
            block = (sum(f for f, _ in per_pair), 12.0 * el + acc + 2.0 * 2 * len(dil) * cout * cout * kk)
            rows.append((f"stage {i}", ("resblock", kk, per_pair, block), None, None))
        cin = cout
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--frames", type=int, default=1024)
    ap.add_argument("--fusion", type=int, default=2, help="resblock_fusion option of the generator")
    ap.add_argument("--precision", default="tc_f16")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default="", help="directory for the JSON table (and nothing else)")
    ap.add_argument("--time-fusions", default="", metavar="M,M,...",
                    help="instead of profiling, time these resblock_fusion settings alternately")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from amphion_b200.vocoders import _vocoders

    w = WORKLOADS["hifigan_v1"]
    dev = torch.device("cuda", 0)
    torch.manual_seed(1234)
    model = _vocoders[w["kind"]](make_cfg("hifigan_v1")).to(dev).eval()
    model.precision = args.precision
    model.set_option("resblock_fusion", args.fusion)
    B, T = args.batch, args.frames
    mel = torch.randn(B, w["n_mel"], T, generator=torch.Generator().manual_seed(0)).to(dev)
    if args.time_fusions:
        # profiler off: ms per step of each resblock_fusion setting, alternated over three rounds
        modes = [int(m) for m in args.time_fusions.split(",")]
        res = {m: [] for m in modes}
        with torch.no_grad():
            for _ in range(3):
                for m in modes:
                    model.set_option("resblock_fusion", m)
                    model(mel)
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(5):
                        model(mel)
                    e1.record()
                    torch.cuda.synchronize()
                    res[m].append(e0.elapsed_time(e1) / 5)
        for m in modes:
            print(f"resblock_fusion {m}: ms per step " + " ".join(f"{v:.1f}" for v in res[m]))
        return
    with torch.no_grad():
        for _ in range(args.warmup):
            model(mel)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            model(mel)
            torch.cuda.synchronize()
    kern = sorted((e for e in prof.events() if e.device_type.name == "CUDA" and "memcpy" not in e.name.lower()
                   and "memset" not in e.name.lower()), key=lambda e: e.time_range.start)
    step_us = kern[-1].time_range.end - kern[0].time_range.start
    tc = ("hconv_kernel", "hchain_kernel", "hpair_kernel")
    hc = [e for e in kern if any(n in e.name for n in tc)]
    other_us = sum(e.time_range.elapsed_us() for e in kern if not any(n in e.name for n in tc))

    def is_block(e):
        return "hchain_kernel" in e.name

    table = OrderedDict()

    def add(stage, plan, us, flops, nbytes):
        r = table.setdefault((stage, plan), dict(launches=0, us=0.0, flops=0.0, bytes=0.0))
        r["launches"] += 1; r["us"] += us; r["flops"] += flops; r["bytes"] += nbytes

    pos = 0
    for stage, plan, flops, nbytes in plan_rows(w["hp"], w["n_mel"], B, T):
        if isinstance(plan, tuple):
            _, kk, per_pair, block = plan
            if is_block(hc[pos]):
                add(stage, f"k={kk} block", hc[pos].time_range.elapsed_us(), *block)
                pos += 1
            else:
                for f, nb in per_pair:
                    add(stage, f"k={kk} pairs", hc[pos].time_range.elapsed_us(), f, nb)
                    pos += 1
        else:
            add(stage, plan, hc[pos].time_range.elapsed_us(), flops, nbytes)
            pos += 1
    if pos != len(hc):
        raise SystemExit(f"launch walk matched {pos} of {len(hc)} tensor-core launches: plan and trace disagree")

    props = torch.cuda.get_device_properties(dev)
    print(f"# {props.name}, HiFi-GAN V1 B={B} 80x{T} {args.precision}, resblock_fusion {args.fusion}: "
          f"step {step_us / 1e3:.1f} ms (first kernel start to last kernel end, profiler on)")
    print(f"{'stage':<9} {'plan':<13} {'n':>3} {'ms':>8} {'share':>6} {'TFLOP/s':>8} {'GB/s':>7}")
    out = []
    by_stage = OrderedDict()
    for (stage, plan), r in table.items():
        ms = r["us"] / 1e3
        row = dict(stage=stage, plan=plan, launches=r["launches"], ms=ms, share=r["us"] / step_us,
                   tflops=r["flops"] / (r["us"] * 1e-6) / 1e12, gbs=r["bytes"] / (r["us"] * 1e-6) / 1e9,
                   tflop=r["flops"] / 1e12, gb=r["bytes"] / 1e9)
        out.append(row)
        s = by_stage.setdefault(stage, [0.0, 0.0, 0.0])
        s[0] += r["us"]; s[1] += r["flops"]; s[2] += r["bytes"]
        print(f"{stage:<9} {plan:<13} {r['launches']:>3} {ms:>8.2f} {row['share']:>6.1%} {row['tflops']:>8.1f} {row['gbs']:>7.0f}")
    print(f"{'other':<9} {'non-hconv':<13} {'':>3} {other_us / 1e3:>8.2f} {other_us / step_us:>6.1%}")
    print("# per stage")
    for stage, (us, fl, nb) in by_stage.items():
        print(f"{stage:<9} {us / 1e3:>8.2f} ms {us / step_us:>6.1%} {fl / us / 1e6:>8.1f} TFLOP/s {nb / us / 1e3:>7.0f} GB/s")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, f"profile_fusion{args.fusion}.json"), "w") as f:
            json.dump(dict(gpu=props.name, batch=B, frames=T, fusion=args.fusion, step_ms=step_us / 1e3,
                           other_ms=other_us / 1e3, rows=out), f, indent=1)


if __name__ == "__main__":
    main()
