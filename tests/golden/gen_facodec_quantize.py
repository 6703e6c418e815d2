"""Generate tests/golden/fac_quantize*.npz by RUNNING THE REFERENCE's FACodecDecoder.forward(vq=True)
(models/codec/ns3_codec/facodec.py:408-471) on the CPU in fp32 and eval mode.  Needs a checkout of the reference
(open-mmlab/Amphion) at $AMPHION_REFERENCE:
    AMPHION_REFERENCE=/path/to/Amphion python tests/golden/gen_facodec_quantize.py

Two seeded variants, keys prefixed "a:" / "b:" (constructor arguments, B, T and n_quantizers:
tests/facodec_quantize_oracle.py GOLDEN_FACODEC_QUANTIZE): the latent ("x"), the codes ("qs"), "outs", the groups' sums
("buf0".."buf2"), "spk_embs" and each timbre-encoder layer's output ("layer0".."layer3", [B, T, 256]).  The timbre
encoder alone has about 6.5 M parameters, so the weights are not stored: the quantizers' and the timbre encoder's
parameters are redrawn by facodec_quantize_oracle.perturb (seeded, state-dict order) and their SHA-256 digests stored
("digest_names" / "digests"); the tests redraw them and check the digests.  "pe" is the reference's own buffer.
The arrays are split into files of under 1 MB: fac_quantize.npz, fac_quantize.part2.npz, ... (not "facodec*": that
prefix is the decoder fixture's).

facodec.py imports .melspec, which needs pyworld, soundfile, librosa and torchaudio; forward(vq=True) never uses them,
so stubs stand in for them."""
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

import facodec_quantize_oracle as fqo  # noqa: E402
from models.codec.ns3_codec.facodec import FACodecDecoder  # noqa: E402

SEEDS = {"a": 91, "b": 93}
PART_BYTES = 1000 * 1000


def gen(tag, out):
    hp, B, T, nq = fqo.GOLDEN_FACODEC_QUANTIZE[tag]
    torch.manual_seed(SEEDS[tag])
    model = FACodecDecoder(**hp).eval()
    fqo.perturb(model.named_parameters(), SEEDS[tag] + 100)
    assert torch.equal(model.timbre_encoder.position_emb.pe, fqo.positional_encoding())
    g = torch.Generator().manual_seed(SEEDS[tag] + 1)
    x = torch.randn(B, hp["in_channels"], T, generator=g)
    seen = {}
    hooks = [layer.register_forward_hook(lambda m, a, o, i=i: seen.__setitem__(f"layer{i}", o.detach().clone()))
             for i, layer in enumerate(model.timbre_encoder.layers)]
    with torch.no_grad():
        outs, qs, commit, bufs, spk = model(x, vq=True, eval_vq=True, n_quantizers=nq)
    for h in hooks:
        h.remove()
    out[f"{tag}:x"] = x.numpy()
    out[f"{tag}:qs"] = qs.numpy()
    out[f"{tag}:outs"] = outs.numpy()
    for i, b in enumerate(bufs):
        out[f"{tag}:buf{i}"] = b.numpy()
    out[f"{tag}:spk_embs"] = spk.numpy()
    for k, v in seen.items():
        out[f"{tag}:{k}"] = v.numpy()
    dg = fqo.digests({k: v.detach().numpy() for k, v in model.state_dict().items()})
    out[f"{tag}:digest_names"] = np.array(list(dg.keys()))
    out[f"{tag}:digests"] = np.array(list(dg.values()))
    assert commit.abs().max() == 0
    print(tag, "qs", tuple(qs.shape), "outs absmax", float(outs.abs().max()), "spk absmax", float(spk.abs().max()))


if __name__ == "__main__":
    out = {}
    for tag in fqo.GOLDEN_FACODEC_QUANTIZE:
        gen(tag, out)
    parts, cur, size = [], {}, 0
    for k, v in out.items():
        if cur and size + v.nbytes > PART_BYTES * 0.95:
            parts.append(cur)
            cur, size = {}, 0
        cur[k] = v
        size += v.nbytes
    parts.append(cur)
    for i, p in enumerate(parts):
        path = os.path.join(HERE, "fac_quantize.npz" if i == 0 else f"fac_quantize.part{i + 1}.npz")
        np.savez(path, **p)
        print(path, os.path.getsize(path), "bytes")
