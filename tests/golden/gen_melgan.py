"""Generate tests/golden/melgan.npz by RUNNING THE REFERENCE's MelGAN (models/vocoders/gan/generator/melgan.py)
on the CPU in fp32.  Needs a checkout of the reference (open-mmlab/Amphion) at $AMPHION_REFERENCE:
    AMPHION_REFERENCE=/path/to/Amphion python tests/golden/gen_melgan.py

Two seeded variants, keys prefixed "a:" / "b:" (hyper-parameters: tests/melgan_oracle.py GOLDEN_MELGAN):
  a: ratios [4, 2], ngf 16, 3 residual layers, 20 mels, B = 2, T = 24, mel ~ N(0, 1), with per-stage outputs
  b: ratios [3, 5] (odd: output_padding 1), ngf 8, 2 residual layers, 12 mels, B = 1, T = 7, mel in the log-mel range
Writes this one file only; the other fixtures come from gen_golden.py."""
import os
import sys
from types import SimpleNamespace as NS

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("AMPHION_REFERENCE", "../Amphion")
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, REF)

from melgan_oracle import GOLDEN_MELGAN  # noqa: E402
from models.vocoders.gan.generator.melgan import MelGAN  # noqa: E402

SEEDS = {"a": 41, "b": 43}


def gen(tag, out):
    hp, n_mel, B, T = GOLDEN_MELGAN[tag]
    cfg = NS(preprocess=NS(n_mel=n_mel), model=NS(melgan=NS(**hp)))
    torch.manual_seed(SEEDS[tag])
    model = MelGAN(cfg).eval()
    g = torch.Generator().manual_seed(SEEDS[tag] + 1)
    if tag == "a":
        mel = torch.randn(B, n_mel, T, generator=g)
    else:  # log-mel range (utils/mel.py:11)
        mel = torch.rand(B, n_mel, T, generator=g) * 13.5 - 11.5
    R = hp["n_residual_layers"]
    stages, hooks = {}, []
    for i in range(len(hp["ratios"])):
        last = model.model[2 + i * (2 + R) + 2 + R - 1]
        hooks.append(last.register_forward_hook(lambda m, a, o, i=i: stages.__setitem__(i, o.detach().clone())))
    with torch.no_grad():
        wav = model(mel)
    for h in hooks:
        h.remove()
    out[f"{tag}:seed"] = np.array(SEEDS[tag])
    out[f"{tag}:mel"] = mel.numpy()
    out[f"{tag}:wav"] = wav.numpy()
    if tag == "a":
        for i in sorted(stages):
            out[f"{tag}:stage{i}"] = stages[i].numpy()
    for k, v in model.state_dict().items():
        out[f"{tag}:sd:{k}"] = v.detach().numpy()
    print(tag, "wav", tuple(wav.shape), "absmax", float(wav.abs().max()), "tensors", len(model.state_dict()))


if __name__ == "__main__":
    out = {}
    for tag in GOLDEN_MELGAN:
        gen(tag, out)
    path = os.path.join(HERE, "melgan.npz")
    np.savez(path, **out)
    print(path, os.path.getsize(path), "bytes")
