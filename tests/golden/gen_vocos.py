"""Generate tests/golden/vocos.npz by RUNNING THE REFERENCE's Vocos (models/codec/amphion_codec/vocos.py) on the CPU in
fp32.  Needs a checkout of the reference (open-mmlab/Amphion) at $AMPHION_REFERENCE:
    AMPHION_REFERENCE=/path/to/Amphion python tests/golden/gen_vocos.py

Two seeded variants, keys prefixed "a:" / "b:" (hyper-parameters: tests/vocos_oracle.py GOLDEN_VOCOS):
  a: 20 mels, dim 48, intermediate 144, 3 layers, n_fft 64, hop 16, B = 2, L = 24, mel ~ N(0, 1); also the initial
     state dict ("init:") and every block's and the backbone's output
  b: 12 mels, dim 40 (not a multiple of 16), intermediate 120, 2 layers, n_fft 48 (not a power of two), hop 12, B = 1,
     L = 7, mel in the log-mel range
After construction the parameters are moved to trained-like scales (gamma ~ U(0.2, 1), LayerNorm weights ~ N(1, 0.2)
with non-zero biases, larger depthwise / pointwise weights) so that every layer moves the output; the state dict that
ran is stored ("sd:").  The reference module imports librosa at module level without using it on this path: a stub
stands in for it.  Writes this one file only."""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("AMPHION_REFERENCE", "../Amphion")
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, REF)
sys.modules.setdefault("librosa", types.ModuleType("librosa"))

from vocos_oracle import GOLDEN_VOCOS  # noqa: E402
from models.codec.amphion_codec.vocos import Vocos  # noqa: E402

SEEDS = {"a": 51, "b": 53}


def trained_like(model, seed):
    """Parameters at trained-like scales, drawn in state-dict order."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if name.endswith("gamma"):
                p.copy_(torch.rand(p.shape, generator=g) * 0.8 + 0.2)
            elif "norm" in name and name.endswith("weight"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.2 + 1.0)
            elif name.endswith("bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
            elif "dwconv" in name:
                p.copy_(torch.randn(p.shape, generator=g) * 0.3)
            elif name.startswith("head.out"):
                p.copy_(torch.randn(p.shape, generator=g) * (0.5 / p.shape[1] ** 0.5))
            else:   # embed, pwconv1, pwconv2: unit-gain fan-in scaling
                fan_in = p[0].numel()
                p.copy_(torch.randn(p.shape, generator=g) / fan_in ** 0.5)


def gen(tag, out):
    hp, B, L = GOLDEN_VOCOS[tag]
    torch.manual_seed(SEEDS[tag])
    model = Vocos(**hp).eval()
    if tag == "a":
        for k, v in model.state_dict().items():
            out[f"{tag}:init:{k}"] = v.detach().numpy().copy()
    trained_like(model, SEEDS[tag] + 100)
    g = torch.Generator().manual_seed(SEEDS[tag] + 1)
    if tag == "a":
        mel = torch.randn(B, hp["input_channels"], L, generator=g)
    else:   # log-mel range
        mel = torch.rand(B, hp["input_channels"], L, generator=g) * 13.5 - 11.5
    blocks, hooks = {}, []
    for i, blk in enumerate(model.backbone.convnext):
        hooks.append(blk.register_forward_hook(lambda m, a, o, i=i: blocks.__setitem__(i, o.detach().clone())))
    hooks.append(model.backbone.register_forward_hook(lambda m, a, o: blocks.__setitem__("backbone", o.detach().clone())))
    with torch.no_grad():
        wav = model(mel)
    for h in hooks:
        h.remove()
    out[f"{tag}:seed"] = np.array(SEEDS[tag])
    out[f"{tag}:mel"] = mel.numpy()
    out[f"{tag}:wav"] = wav.numpy()
    if tag == "a":
        for i in range(hp["num_layers"]):
            out[f"{tag}:block{i}"] = blocks[i].numpy()
        out[f"{tag}:backbone"] = blocks["backbone"].numpy()
    for k, v in model.state_dict().items():
        out[f"{tag}:sd:{k}"] = v.detach().numpy()
    print(tag, "wav", tuple(wav.shape), "absmax", float(wav.abs().max()), "tensors", len(model.state_dict()))


if __name__ == "__main__":
    out = {}
    for tag in GOLDEN_VOCOS:
        gen(tag, out)
    path = os.path.join(HERE, "vocos.npz")
    np.savez(path, **out)
    print(path, os.path.getsize(path), "bytes")
