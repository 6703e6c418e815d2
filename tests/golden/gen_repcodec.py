"""Generate tests/golden/repcodec*.npz by RUNNING THE REFERENCE's RepCodec (models/codec/kmeans/repcodec_model.py,
kmeans/vocos.py, amphion_codec/quantize) on the CPU in fp32 and eval mode, as MaskGCT runs it
(models/tts/maskgct/maskgct_utils.py:111-121).  Needs a checkout of the reference (open-mmlab/Amphion) at
$AMPHION_REFERENCE:
    AMPHION_REFERENCE=/path/to/Amphion python tests/golden/gen_repcodec.py

Two seeded variants, keys prefixed "a:" / "b:" (constructor arguments, B and T: tests/repcodec_oracle.py
GOLDEN_REPCODEC): the features ("x" [B, T, hidden]), the encoder's output ("enc" [B, T, hidden]), quantize(x)'s codes
("codes") and quantized view (stored contiguous, "quantized"), and forward(x)'s x_rec ("x_rec").  The weights are not
stored: the codec is built under torch.manual_seed(seed), every bias, LayerNorm affine and layer scale is then redrawn
by repcodec_oracle.perturb, and the SHA-256 digests of the resulting state dict are stored ("digest_names",
"digests"); the tests rebuild it with the native class and check the digests.

"maskgct:*" holds the key list and shapes of RepCodec(cfg=semantic_codec) at models/tts/maskgct/config/maskgct.json,
for the strict-load test.

vocos.py imports torchaudio and librosa, which the codec never calls; stubs stand in for them."""
import json
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
    """Module whose every attribute is a dummy (never executed)."""
    __path__ = []

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return type(name, (), {})


for _m in ["librosa", "librosa.filters", "torchaudio", "torchaudio.functional", "torchaudio.functional.functional"]:
    sys.modules.setdefault(_m, _Stub(_m))

import repcodec_oracle as rco  # noqa: E402
from models.codec.kmeans.repcodec_model import RepCodec  # noqa: E402

PART_BYTES = 1000 * 1000


def build(tag):
    hp, B, T = rco.GOLDEN_REPCODEC[tag]
    torch.manual_seed(rco.SEEDS[tag])
    m = RepCodec(**hp).eval()
    rco.perturb(m.named_parameters(), rco.SEEDS[tag] + 100)
    return m


def gen(tag, out):
    hp, B, T = rco.GOLDEN_REPCODEC[tag]
    m = build(tag)
    g = torch.Generator().manual_seed(rco.SEEDS[tag] + 1)
    x = torch.randn(B, T, hp["hidden_size"], generator=g)
    with torch.no_grad():
        enc = m.encoder(x.transpose(1, 2))
        codes, quantized = m.quantize(x)
        x_rec, loss, all_indices = m(x)
    assert float(loss) == 0.0 and loss.dim() == 0
    assert torch.equal(all_indices.reshape(codes.shape), codes)
    out[f"{tag}:x"] = x.numpy()
    out[f"{tag}:enc"] = enc.numpy()
    out[f"{tag}:codes"] = codes.numpy()
    out[f"{tag}:quantized"] = quantized.contiguous().numpy()
    out[f"{tag}:x_rec"] = x_rec.numpy()
    dg = rco.digests({k: v.detach().numpy() for k, v in m.state_dict().items()})
    out[f"{tag}:digest_names"] = np.array(list(dg.keys()))
    out[f"{tag}:digests"] = np.array(list(dg.values()))
    print(tag, "enc", tuple(enc.shape), "codes", tuple(codes.shape), "x_rec absmax", float(x_rec.abs().max()))


def maskgct_keys(out):
    cfg = json.load(open(os.path.join(REF, "models/tts/maskgct/config/maskgct.json")))["model"]["semantic_codec"]
    sd = RepCodec(cfg=types.SimpleNamespace(**cfg)).state_dict()
    out["maskgct:names"] = np.array(list(sd.keys()))
    out["maskgct:ndim"] = np.array([v.dim() for v in sd.values()], np.int64)
    out["maskgct:shapes"] = np.concatenate([np.array(v.shape, np.int64) for v in sd.values()])


if __name__ == "__main__":
    out = {}
    for tag in rco.GOLDEN_REPCODEC:
        gen(tag, out)
    maskgct_keys(out)
    parts, cur, size = [], {}, 0
    for k, v in out.items():
        if cur and size + v.nbytes > PART_BYTES * 0.95:
            parts.append(cur)
            cur, size = {}, 0
        cur[k] = v
        size += v.nbytes
    parts.append(cur)
    for i, p in enumerate(parts):
        path = os.path.join(HERE, "repcodec.npz" if i == 0 else f"repcodec.part{i + 1}.npz")
        np.savez(path, **p)
        print(path, os.path.getsize(path), "bytes")
