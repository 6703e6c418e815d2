"""Generate tests/golden/diffwave.npz by RUNNING THE REFERENCE's DiffWave (models/vocoders/diffusion/diffwave/diffwave.py)
and its sampler (models/vocoders/diffusion/diffusion_vocoder_inference.py) on the CPU in fp32.  Needs a checkout of the
reference (open-mmlab/Amphion) at $AMPHION_REFERENCE:
    AMPHION_REFERENCE=/path/to/Amphion python tests/golden/gen_diffwave.py

Geometry: tests/diffwave_oracle.py GOLDEN_DIFFWAVE (64 channels, 6 layers, dilation cycle 3, factors [4, 4]), 10 mels,
B = 2, 6 frames (96 samples).  Stored:
  seed, init:*   SHA-256 of every tensor of the seeded initial state dict (dtype, shape and bytes), in state-dict order
  table          the fp32 step-embedding table (a non-persistent buffer, not in the state dict)
  sd:*           the state dict that ran: after construction the parameters are moved to trained-like scales (unit-gain
                 fan-in weights, 0.1 biases, upsampler taps ~ N(0, 0.3), a non-zero output_projection.weight) so that
                 every layer moves the output
  mel, audio     inputs
  eps_float      forward with the float step [2.37] (lerp between table rows)
  x{i}, skip{i}  layer i's output x and running skip sum in that forward, utterance 0
  steps_int      int64 [B] steps; eps_int the forward with them
  sampler_*      vocoder_inference(fast_inference=True) on mel, with torch.randn / torch.randn_like intercepted to return
                 the stored sampler_noise0 (initial audio) and sampler_noise{n} (n = 5 .. 1, in draw order); sampler_audio
                 is its output
Writes diffwave.npz and diffwave.part<N>.npz (each under 1 MB; conftest.load_golden merges them)."""
import hashlib
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
# utils.util (imported by the sampler module for its padding helpers) pulls config libraries this path never uses
for name in ("json5", "ruamel", "ruamel.yaml", "ruamel_yaml"):
    sys.modules.setdefault(name, types.ModuleType(name))
sys.modules["ruamel.yaml"].YAML = sys.modules["ruamel_yaml"].YAML = object

from diffwave_oracle import GOLDEN_DIFFWAVE, GOLDEN_DIFFWAVE_BF, GOLDEN_DIFFWAVE_MEL, diffwave_cfg  # noqa: E402
from models.vocoders.diffusion.diffwave.diffwave import DiffWave  # noqa: E402
from models.vocoders.diffusion import diffusion_vocoder_inference as dvi  # noqa: E402

SEED = 61


def tensor_digest(a):
    return hashlib.sha256(f"{a.dtype.str}{a.shape}".encode() + np.ascontiguousarray(a).tobytes()).hexdigest()


def trained_like(model, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if name.endswith("bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
            elif name.startswith("spectrogram_upsampler"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.3)
            else:   # unit-gain fan-in scaling, output_projection.weight included
                p.copy_(torch.randn(p.shape, generator=g) / p[0].numel() ** 0.5)


def main():
    hp, n_mel = GOLDEN_DIFFWAVE, GOLDEN_DIFFWAVE_MEL
    B, F = GOLDEN_DIFFWAVE_BF
    out = {}
    torch.manual_seed(SEED)
    model = DiffWave(diffwave_cfg(hp, n_mel)).eval()
    out["seed"] = np.array(SEED)
    for k, v in model.state_dict().items():
        out[f"init:{k}"] = np.array(tensor_digest(v.numpy()))
    out["table"] = model.diffusion_embedding.embedding.numpy().copy()
    trained_like(model, SEED + 100)
    g = torch.Generator().manual_seed(SEED + 1)
    L = F * hp["upsample_factors"][0] * hp["upsample_factors"][1]
    mel = torch.randn(B, n_mel, F, generator=g)
    audio = torch.randn(B, L, generator=g) * 0.5
    layers = {}
    hooks = [blk.register_forward_hook(lambda m, a, o, i=i: layers.__setitem__(i, (o[0].clone(), o[1].clone())))
             for i, blk in enumerate(model.residual_layers)]
    with torch.no_grad():
        eps_f = model(audio, torch.tensor([2.37]), mel)
        for h in hooks:
            h.remove()
        steps_int = torch.tensor([1, 3])
        eps_i = model(audio, steps_int, mel)
    skip = None
    for i in range(len(model.residual_layers)):
        x, s = layers[i]
        skip = s if skip is None else s + skip
        out[f"x{i}"], out[f"skip{i}"] = x[:1].numpy(), skip[:1].numpy()
    out.update(mel=mel.numpy(), audio=audio.numpy(), eps_float=eps_f.numpy(), steps_int=steps_int.numpy(),
               eps_int=eps_i.numpy())

    # the sampler, with its noise draws replaced by stored values
    draws = []
    ng = torch.Generator().manual_seed(SEED + 2)
    real_randn, real_randn_like = torch.randn, torch.randn_like

    def randn(*shape, **kw):
        kw.pop("device", None)
        t = real_randn(*shape, generator=ng)
        draws.append(t.numpy().copy())
        return t

    def randn_like(t):
        return randn(*t.shape)

    dvi.torch.randn, dvi.torch.randn_like = randn, randn_like
    try:
        cfg = diffwave_cfg(hp, n_mel)
        cfg.model.diffwave.noise_schedule = model.cfg.model.diffwave.noise_schedule
        wav = dvi.vocoder_inference(cfg, model, mel[:1].clone(), device="cpu", fast_inference=True)
    finally:
        dvi.torch.randn, dvi.torch.randn_like = real_randn, real_randn_like
    out["sampler_mel"] = mel[:1].numpy()
    out["sampler_noise0"] = draws[0]
    n_steps = len(hp["inference_noise_schedule"])
    for j, n in enumerate(range(n_steps - 1, 0, -1)):
        out[f"sampler_noise{n}"] = draws[1 + j]
    assert len(draws) == n_steps
    out["sampler_audio"] = wav.numpy()
    print("eps absmax", float(eps_f.abs().max()), "sampler absmax", float(wav.abs().max()))
    for k, v in model.state_dict().items():
        out[f"sd:{k}"] = v.numpy()
    # greedy split in insertion order, each file's arrays under 900 KB
    files, cur, size = [], {}, 0
    for k, v in out.items():
        if cur and size + v.nbytes > 900_000:
            files.append(cur)
            cur, size = {}, 0
        cur[k], size = v, size + v.nbytes
    files.append(cur)
    for i, f in enumerate(files):
        path = os.path.join(HERE, "diffwave.npz" if i == 0 else f"diffwave.part{i + 1}.npz")
        np.savez_compressed(path, **f)
        print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
