"""Generate tests/golden/fac_redecoder*.npz by RUNNING THE REFERENCE's FACodecRedecoder (models/codec/ns3_codec/
facodec.py:602-769) on the CPU in fp32 and eval mode.  Needs a checkout of the reference (open-mmlab/Amphion) at
$AMPHION_REFERENCE:
    AMPHION_REFERENCE=/path/to/Amphion python tests/golden/gen_facodec_redecode.py

Two seeded variants, keys prefixed "a:" / "b:" (constructor arguments, B and T: tests/facodec_redecode_oracle.py
GOLDEN_FACODEC_REDECODE): the codes, the speaker embedding ("spk"), vq2emb with use_residual False ("emb") and True
("emb_res"), each prosody-transformer layer's output of each transformer run ("layers" [runs, 4, B, T, 256]) and
inference(emb, spk) ("wav").  The transformer alone has about 6.5 M parameters, so no weight is stored: every parameter
is redrawn by facodec_redecode_oracle.perturb (seeded, sorted-name order) and the SHA-256 digest of every state-dict
entry is stored ("digest_names" / "digests"); the tests redraw them and check the digests.  "pe" and the anti-aliasing
filters are the reference's own buffers.  The arrays are split into files of under 1 MB: fac_redecoder.npz,
fac_redecoder.part2.npz, ... (not "facodec*", "fac_quantize*" or "fac_encoder*": other fixtures use those prefixes).

facodec.py imports .melspec, which needs pyworld, soundfile, librosa and torchaudio; the redecoder never uses them, so
stubs stand in for them."""
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


class _Stub(types.ModuleType):
    """Module whose every attribute is a dummy class (never executed)."""
    __path__ = []

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return type(name, (), {})


for _m in ["pyworld", "soundfile", "librosa", "librosa.filters", "torchaudio", "torchaudio.functional"]:
    sys.modules.setdefault(_m, _Stub(_m))

import facodec_redecode_oracle as fro  # noqa: E402
from models.codec.ns3_codec.facodec import FACodecRedecoder  # noqa: E402

SEEDS = {"a": 111, "b": 113}
PART_BYTES = 1000 * 1000


def gen(tag, out):
    hp, B, T = fro.GOLDEN_FACODEC_REDECODE[tag]
    torch.manual_seed(SEEDS[tag])
    model = FACodecRedecoder(**hp).eval()
    fro.perturb(model.named_parameters(), SEEDS[tag] + 100, len(hp["up_ratios"]))
    assert torch.equal(model.timbre_cond_prosody_enc.position_emb.pe, fro.positional_encoding())
    g = torch.Generator().manual_seed(SEEDS[tag] + 1)
    p, c, r = fro.n_tables(hp)
    rows = []
    for q, (k, n) in enumerate(zip(("prosody", "content", "residual"), (p, c, r))):
        rows += [torch.randint(0, 2 ** hp[f"codebook_size_{k}"], (1, B, T), generator=g) for _ in range(n)]
    codes = torch.cat(rows)
    spk = torch.randn(B, 256, generator=g)
    seen = []
    hooks = [layer.register_forward_hook(lambda m, a, o, i=i: seen.append((i, o.detach().clone())))
             for i, layer in enumerate(model.timbre_cond_prosody_enc.layers)]
    with torch.no_grad():
        emb = model.vq2emb(codes, spk, use_residual=False)
        n_seen = len(seen)
        emb_res = model.vq2emb(codes, spk, use_residual=True)
        wav = model.inference(emb, spk)
    for h in hooks:
        h.remove()
    assert n_seen == 4 * p and [i for i, _ in seen[:n_seen]] == list(range(4)) * p
    out[f"{tag}:codes"] = codes.numpy()
    out[f"{tag}:spk"] = spk.numpy()
    out[f"{tag}:emb"] = emb.numpy()
    out[f"{tag}:emb_res"] = emb_res.numpy()
    out[f"{tag}:layers"] = torch.stack([o for _, o in seen[:n_seen]]).reshape(p, 4, B, T, 256).numpy()
    out[f"{tag}:wav"] = wav.numpy()
    dg = fro.digests({k: v.detach().numpy() for k, v in model.state_dict().items()})
    out[f"{tag}:digest_names"] = np.array(list(dg.keys()))
    out[f"{tag}:digests"] = np.array(list(dg.values()))
    print(tag, "emb absmax", float(emb.abs().max()), "wav", tuple(wav.shape), "absmax", float(wav.abs().max()))


def released_keys(out):
    sd = FACodecRedecoder(**fro.RELEASED).state_dict()
    out["released_keys"] = np.array(list(sd.keys()))
    shapes = np.full((len(sd), 4), -1, dtype=np.int64)
    for i, v in enumerate(sd.values()):
        shapes[i, :v.dim()] = v.shape
    out["released_shapes"] = shapes
    print("released", len(sd), "tensors,", sum(v.numel() for v in sd.values()), "elements")


if __name__ == "__main__":
    out = {}
    for tag in fro.GOLDEN_FACODEC_REDECODE:
        gen(tag, out)
    released_keys(out)
    parts, cur, size = [], {}, 0
    for k, v in out.items():
        if cur and size + v.nbytes > PART_BYTES * 0.95:
            parts.append(cur)
            cur, size = {}, 0
        cur[k] = v
        size += v.nbytes
    parts.append(cur)
    for i, p in enumerate(parts):
        path = os.path.join(HERE, "fac_redecoder.npz" if i == 0 else f"fac_redecoder.part{i + 1}.npz")
        np.savez(path, **p)
        print(path, os.path.getsize(path), "bytes")
