"""Generate tests/golden/facodec*.npz by RUNNING THE REFERENCE's FACodecDecoder (models/codec/ns3_codec/facodec.py) on the
CPU in fp32.  Needs a checkout of the reference (open-mmlab/Amphion) at $AMPHION_REFERENCE:
    AMPHION_REFERENCE=/path/to/Amphion python tests/golden/gen_facodec.py

Two seeded variants, keys prefixed "a:" / "b:" (constructor arguments: tests/facodec_oracle.py GOLDEN_FACODEC):
  a: in_channels 32, upsample_initial_channel 128, up_ratios [5, 4, 2], the reference's codebooks (1 + 2 + 3 layers of
     2^10 x 8), B = 2, T = 12: codes -> vq2emb -> inference; stores the codes, the speaker embedding, vq2emb's output
     ("emb"), the FiLM output ("film"), each DecoderBlock's output ("stage{i}") and the audio
  b: in_channels 16, up_ratios [3, 2] (odd ratio: output_padding 1), B = 1, T = 5: a float latent fed to inference
The reference zeroes every conv bias and starts SnakeBeta at alpha = beta = 0 (log scale), so after construction every
parameter the decode path reads is redrawn from a seeded generator: unit-gain weight-norm magnitudes, nonzero biases,
alpha / beta, timbre_linear and the codebooks.  Only those tensors are stored ("sd:"), with the reference's key -> shape
list of the README geometry ("readme_keys" / "readme_shapes", shapes padded with -1) so that strict loading is checked
without the reference.  The arrays are split into files of under 1 MB: facodec.npz, facodec.part2.npz, ...

facodec.py imports .melspec, which needs pyworld, soundfile, librosa and torchaudio; the decoder never uses them, so
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

from facodec_oracle import GOLDEN_FACODEC, README_FACODEC  # noqa: E402
from models.codec.ns3_codec.facodec import FACodecDecoder  # noqa: E402

SEEDS = {"a": 71, "b": 73}
PART_BYTES = 1000 * 1000


def decode_path(name):
    """Whether the waveform path (vq2emb, inference) reads this state-dict entry."""
    return (name.startswith("model.") or name.startswith("timbre_linear.") or
            (name.startswith("quantizer.") and (".out_proj." in name or "._codebook." in name)))


def perturb(model, seed):
    """Decode-path parameters at trained-like scales, drawn in state-dict order."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if not decode_path(name):
                continue
            if name.endswith("weight_g"):            # row norms of the folded weights
                # conv_post small enough that tanh stays near its linear range; a ResidualUnit's k = 1 conv small, as
                # trained residual branches are
                scale = 1.0
                if name.startswith(f"model.{len(model.up_ratios) + 2}."):
                    scale = 0.1
                elif re.fullmatch(r"model\.\d+\.block\.[234]\.block\.3\.weight_g", name):
                    scale = 0.25
                p.copy_((torch.rand(p.shape, generator=g) * 0.6 + 0.6) * scale)
            elif name.endswith("weight_v"):
                p.copy_(torch.randn(p.shape, generator=g))
            elif name.endswith(".alpha") or name.endswith(".beta"):   # log scale
                p.copy_(torch.randn(p.shape, generator=g) * 0.3)
            elif name == "timbre_linear.weight":
                p.copy_(torch.randn(p.shape, generator=g) * (0.3 / p.shape[1] ** 0.5))
            elif name == "timbre_linear.bias":
                c = p.shape[0] // 2
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
                p[:c] += 1.0
            elif name.endswith("_codebook.weight"):
                p.copy_(torch.randn(p.shape, generator=g))
            elif name.endswith("bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
            else:
                raise AssertionError(f"unexpected decode-path parameter {name}")


def gen(tag, out):
    hp, B, T = GOLDEN_FACODEC[tag]
    torch.manual_seed(SEEDS[tag])
    model = FACodecDecoder(**hp).eval()
    perturb(model, SEEDS[tag] + 100)
    g = torch.Generator().manual_seed(SEEDS[tag] + 1)
    C = hp["in_channels"]
    spk = torch.randn(B, C, generator=g)
    seen = {}
    hooks = [model.model.register_forward_pre_hook(lambda m, a: seen.__setitem__("film", a[0].detach().clone()))]
    for i in range(len(hp["up_ratios"])):
        hooks.append(model.model[1 + i].register_forward_hook(
            lambda m, a, o, i=i: seen.__setitem__(f"stage{i}", o.detach().clone())))
    with torch.no_grad():
        if tag == "a":
            n_q = model.vq_num_q_p + model.vq_num_q_c + model.vq_num_q_r
            codes = torch.randint(0, 2 ** 10, (n_q, B, T), generator=g)
            x = model.vq2emb(codes)
            out[f"{tag}:codes"] = codes.numpy()
            out[f"{tag}:emb"] = x.numpy()
            out[f"{tag}:emb_nores"] = model.vq2emb(codes, use_residual_code=False).numpy()
        else:
            x = torch.randn(B, C, T, generator=g) * 2.0 + 0.5
            out[f"{tag}:x"] = x.numpy()
        wav = model.inference(x, spk)
    for h in hooks:
        h.remove()
    out[f"{tag}:spk"] = spk.numpy()
    out[f"{tag}:wav"] = wav.numpy()
    for k, v in seen.items():
        out[f"{tag}:{k}"] = v.numpy()
    for k, v in model.state_dict().items():
        if decode_path(k):
            out[f"{tag}:sd:{k}"] = v.detach().numpy()
    print(tag, "wav", tuple(wav.shape), "absmax", float(wav.abs().max()))


def readme_keys(out):
    sd = FACodecDecoder(**README_FACODEC).state_dict()
    out["readme_keys"] = np.array(list(sd.keys()))
    shapes = np.full((len(sd), 4), -1, dtype=np.int64)
    for i, v in enumerate(sd.values()):
        shapes[i, :v.dim()] = v.shape
    out["readme_shapes"] = shapes
    print("readme", len(sd), "tensors")


if __name__ == "__main__":
    out = {}
    for tag in GOLDEN_FACODEC:
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
        path = os.path.join(HERE, "facodec.npz" if i == 0 else f"facodec.part{i + 1}.npz")
        np.savez(path, **p)
        print(path, os.path.getsize(path), "bytes")
