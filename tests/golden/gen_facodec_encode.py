"""Generate tests/golden/fac_encoder*.npz by RUNNING THE REFERENCE's FACodecEncoder (models/codec/ns3_codec/facodec.py)
on the CPU in fp32.  Needs a checkout of the reference (open-mmlab/Amphion) at $AMPHION_REFERENCE:
    AMPHION_REFERENCE=/path/to/Amphion python tests/golden/gen_facodec_encode.py

Two seeded variants, keys prefixed "a:" / "b:" (constructor arguments, B and N: tests/facodec_encode_oracle.py
GOLDEN_FACODEC_ENCODE): the waveform ("wav"), each EncoderBlock's output ("stage{i}") and the encoder's output ("enc").
The reference zeroes every conv bias and starts SnakeBeta at alpha = beta = 0 (log scale), so after construction every
parameter is redrawn from a seeded generator (unit-gain weight-norm magnitudes, nonzero biases, alpha / beta) and
stored ("sd:"), with the reference's key -> shape list of the README geometry ("readme_keys" / "readme_shapes", shapes
padded with -1) so that strict loading is checked without the reference.  The arrays are split into files of under
1 MB: fac_encoder.npz, fac_encoder.part2.npz, ... (not "facodec*": that prefix is the decoder fixture's).

facodec.py imports .melspec, which needs pyworld, soundfile, librosa and torchaudio; the encoder never uses them, so
stubs stand in for them."""
import os
import re
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("AMPHION_REFERENCE", "../Amphion")
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, REF)


class _Stub(types.ModuleType):
    """Module whose every attribute is a dummy class (never executed)."""
    __path__ = []

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return type(name, (), {})


for _m in ["pyworld", "soundfile", "librosa", "librosa.filters", "torchaudio", "torchaudio.functional"]:
    sys.modules.setdefault(_m, _Stub(_m))

from facodec_encode_oracle import GOLDEN_FACODEC_ENCODE, README_FACODEC_ENCODER  # noqa: E402
from models.codec.ns3_codec.facodec import FACodecEncoder  # noqa: E402

SEEDS = {"a": 81, "b": 83}
PART_BYTES = 1000 * 1000


def perturb(model, seed):
    """Every parameter at trained-like scales, drawn in state-dict order."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if name.endswith("weight_g"):
                # a ResidualUnit's k = 1 conv small, as trained residual branches are
                scale = 0.25 if re.fullmatch(r"block\.\d+\.block\.[012]\.block\.3\.weight_g", name) else 1.0
                p.copy_((torch.rand(p.shape, generator=g) * 0.6 + 0.6) * scale)
            elif name.endswith("weight_v"):
                p.copy_(torch.randn(p.shape, generator=g))
            elif name.endswith(".alpha") or name.endswith(".beta"):   # log scale
                p.copy_(torch.randn(p.shape, generator=g) * 0.3)
            elif name.endswith("bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
            else:
                raise AssertionError(f"unexpected parameter {name}")


def gen(tag, out):
    hp, B, N = GOLDEN_FACODEC_ENCODE[tag]
    torch.manual_seed(SEEDS[tag])
    model = FACodecEncoder(**hp).eval()
    perturb(model, SEEDS[tag] + 100)
    g = torch.Generator().manual_seed(SEEDS[tag] + 1)
    wav = torch.randn(B, 1, N, generator=g) * 0.3
    seen = {}
    hooks = [model.block[1 + i].register_forward_hook(lambda m, a, o, i=i: seen.__setitem__(f"stage{i}", o.detach().clone()))
             for i in range(len(hp["up_ratios"]))]
    with torch.no_grad():
        enc = model(wav)
    for h in hooks:
        h.remove()
    out[f"{tag}:wav"] = wav.numpy()
    out[f"{tag}:enc"] = enc.numpy()
    for k, v in seen.items():
        out[f"{tag}:{k}"] = v.numpy()
    for k, v in model.state_dict().items():
        out[f"{tag}:sd:{k}"] = v.detach().numpy()
    print(tag, "enc", tuple(enc.shape), "absmax", float(enc.abs().max()))


def readme_keys(out):
    sd = FACodecEncoder(**README_FACODEC_ENCODER).state_dict()
    out["readme_keys"] = np.array(list(sd.keys()))
    shapes = np.full((len(sd), 4), -1, dtype=np.int64)
    for i, v in enumerate(sd.values()):
        shapes[i, :v.dim()] = v.shape
    out["readme_shapes"] = shapes
    print("readme", len(sd), "tensors")


if __name__ == "__main__":
    out = {}
    for tag in GOLDEN_FACODEC_ENCODE:
        gen(tag, out)
    readme_keys(out)
    parts, cur, size = [], {}, 0
    for k, v in out.items():
        if cur and size + v.nbytes > PART_BYTES * 0.95:
            parts.append(cur)
            cur, size = {}, 0
        cur[k] = v
        size += v.nbytes
    parts.append(cur)
    for i, p in enumerate(parts):
        path = os.path.join(HERE, "fac_encoder.npz" if i == 0 else f"fac_encoder.part{i + 1}.npz")
        np.savez(path, **p)
        print(path, os.path.getsize(path), "bytes")
