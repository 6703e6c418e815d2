"""Generate tests/golden/amphion_codec*.npz by RUNNING THE REFERENCE's CodecEncoder and CodecDecoder
(models/codec/amphion_codec/codec.py, quantize/residual_vq.py, quantize/factorized_vector_quantize.py, vocos.py) on the
CPU in fp32 and eval mode, as MaskGCT runs them (models/tts/maskgct/maskgct_utils.py:124-127, :223-230).  Needs a
checkout of the reference (open-mmlab/Amphion) at $AMPHION_REFERENCE:
    AMPHION_REFERENCE=/path/to/Amphion python tests/golden/gen_amphion_codec.py

Two seeded variants, keys prefixed "a:" / "b:" (constructor arguments, B, N and n_quantizers:
tests/amphion_codec_oracle.py GOLDEN_CODEC): the waveform ("wav"), each EncoderBlock's output ("stage0".."stageN-1"),
the encoder output ("enc"), quantizer(enc, n_quantizers)'s codes ("codes"), "quantized_out" and "all_quantized",
vq2emb(codes) ("vq2emb") and the decoder's waveform of it ("out").  The weights are not stored: both modules are built
under torch.manual_seed(seed), every bias and Snake1d alpha is then redrawn by amphion_codec_oracle.perturb, and the
SHA-256 digests of the resulting state dicts are stored ("enc_digest_*", "dec_digest_*"); the tests rebuild them with the
native classes and check the digests.

"maskgct:*" holds the key lists and shapes of CodecEncoder(cfg.encoder) and CodecDecoder(cfg.decoder) at
models/tts/maskgct/config/maskgct.json, for the strict-load test.

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

import amphion_codec_oracle as aco  # noqa: E402
from models.codec.amphion_codec.codec import CodecDecoder, CodecEncoder  # noqa: E402

PART_BYTES = 1000 * 1000


def build(tag):
    enc_hp, dec_hp, B, N, nq = aco.GOLDEN_CODEC[tag]
    torch.manual_seed(aco.SEEDS[tag])
    enc = CodecEncoder(**enc_hp).eval()
    dec = CodecDecoder(**dec_hp).eval()
    aco.perturb(enc.named_parameters(), aco.SEEDS[tag] + 100)
    aco.perturb(dec.named_parameters(), aco.SEEDS[tag] + 200)
    return enc, dec


def gen(tag, out):
    enc_hp, dec_hp, B, N, nq = aco.GOLDEN_CODEC[tag]
    enc, dec = build(tag)
    g = torch.Generator().manual_seed(aco.SEEDS[tag] + 1)
    wav = torch.randn(B, 1, N, generator=g) * 0.3
    stages = []
    hooks = [enc.block[1 + i].register_forward_hook(lambda m, a, o: stages.append(o.detach().clone()))
             for i in range(len(enc_hp["up_ratios"]))]
    with torch.no_grad():
        z = enc(wav)
        qo, codes, commit, cbl, allq = dec(z, vq=True, eval_vq=True, n_quantizers=nq)
        emb = dec.vq2emb(codes, n_quantizers=nq)
        y = dec(emb)
    for h in hooks:
        h.remove()
    assert commit.abs().max() == 0 and cbl.abs().max() == 0 and tuple(commit.shape) == (nq,)
    out[f"{tag}:wav"] = wav.numpy()
    for i, s in enumerate(stages):
        out[f"{tag}:stage{i}"] = s.numpy()
    out[f"{tag}:enc"] = z.numpy()
    out[f"{tag}:codes"] = codes.numpy()
    out[f"{tag}:quantized_out"] = qo.numpy()
    out[f"{tag}:all_quantized"] = allq.numpy()
    out[f"{tag}:vq2emb"] = emb.numpy()
    out[f"{tag}:out"] = y.numpy()
    for who, m in (("enc", enc), ("dec", dec)):
        dg = aco.digests({k: v.detach().numpy() for k, v in m.state_dict().items()})
        out[f"{tag}:{who}_digest_names"] = np.array(list(dg.keys()))
        out[f"{tag}:{who}_digests"] = np.array(list(dg.values()))
    print(tag, "enc", tuple(z.shape), "codes", tuple(codes.shape), "out", tuple(y.shape), "absmax", float(y.abs().max()))


def maskgct_keys(out):
    cfg = json.load(open(os.path.join(REF, "models/tts/maskgct/config/maskgct.json")))["model"]["acoustic_codec"]
    ns = lambda d: types.SimpleNamespace(**d)   # noqa: E731
    for who, m in (("enc", CodecEncoder(cfg=ns(cfg["encoder"]))), ("dec", CodecDecoder(cfg=ns(cfg["decoder"])))):
        sd = m.state_dict()
        out[f"maskgct:{who}_names"] = np.array(list(sd.keys()))
        out[f"maskgct:{who}_ndim"] = np.array([v.dim() for v in sd.values()], np.int64)
        out[f"maskgct:{who}_shapes"] = np.concatenate([np.array(v.shape, np.int64) for v in sd.values()])


if __name__ == "__main__":
    out = {}
    for tag in aco.GOLDEN_CODEC:
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
        path = os.path.join(HERE, "amphion_codec.npz" if i == 0 else f"amphion_codec.part{i + 1}.npz")
        np.savez(path, **p)
        print(path, os.path.getsize(path), "bytes")
