"""Generate tests/golden/fac_v2*.npz by RUNNING THE REFERENCE's FACodecEncoderV2 and FACodecDecoderV2
(models/codec/ns3_codec/facodec.py:772-1199) on the CPU in fp32 and eval mode.  Needs a checkout of the reference
(open-mmlab/Amphion) at $AMPHION_REFERENCE:
    AMPHION_REFERENCE=/path/to/Amphion python tests/golden/gen_facodec_v2.py

Two seeded variants, keys prefixed "a:" / "b:" (constructor arguments, B, samples and n_quantizers:
tests/facodec_v2_oracle.py GOLDEN_FACODEC_V2): the waveforms "wav" / "wav_b", the encoder output "enc", the prosody
feature "pf", each melspec_encoder layer's output ("player0".."player3", [B, T, 256]), the forward(vq=True) tuple
("qs", "outs", "buf0".."buf2", "spk_embs"), vq2emb with and without the residual codes ("emb_res", "emb_nores"),
inference(outs, spk_embs) ("wav_out") and the README's A -> B conversion ("vc": inference(vq2emb(codes of A,
use_residual=False), spk_embs of B)).  The weights are not stored: the quantizers', both transformers' and
melspec_linear's are redrawn by facodec_v2_oracle.perturb (seeded, state-dict order), the rest come from the seeds,
and SHA-256 digests are stored ("digest_names" / "digests").  The mel filterbank the encoder built is stored
("mel_basis"), and the reference modules' state-dict keys and shapes ("enc_keys" / "enc_shapes", "dec_keys" /
"dec_shapes").  Files of under 1 MB: fac_v2.npz, fac_v2.part2.npz, ...

facodec.py imports .melspec, which imports pyworld, soundfile, librosa and torchaudio.  The V2 encoder builds a mel
filterbank with librosa.filters.mel, so that one is the Slaney restatement in oracle/mel.py; the others are stubs that
are never executed."""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("AMPHION_REFERENCE", "../Amphion")
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
sys.path.insert(0, REF)


class _Stub(types.ModuleType):
    """Module whose every attribute is a dummy class (never executed)."""
    __path__ = []

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return type(name, (), {})


from oracle.mel import slaney_mel_filterbank  # noqa: E402

for _m in ["pyworld", "soundfile", "librosa", "torchaudio", "torchaudio.functional"]:
    sys.modules.setdefault(_m, _Stub(_m))
_filters = types.ModuleType("librosa.filters")
_filters.mel = lambda sr, n_fft, n_mels, fmin, fmax: slaney_mel_filterbank(sr, n_fft, n_mels, fmin, fmax)
sys.modules["librosa.filters"] = _filters

import facodec_v2_oracle as fvo  # noqa: E402
from models.codec.ns3_codec.facodec import FACodecDecoderV2, FACodecEncoderV2  # noqa: E402

SEEDS = {"a": 191, "b": 193}
PART_BYTES = 1000 * 1000


def gen(tag, out):
    enc_hp, dec_hp, B, N, nq = fvo.GOLDEN_FACODEC_V2[tag]
    torch.manual_seed(SEEDS[tag])
    enc = FACodecEncoderV2(**enc_hp).eval()
    dec = FACodecDecoderV2(**dec_hp).eval()
    fvo.perturb(dec.named_parameters(), SEEDS[tag] + 100)
    g = torch.Generator().manual_seed(SEEDS[tag] + 1)
    wav = torch.randn(B, 1, N, generator=g) * 0.3
    wav_b = torch.randn(B, 1, N, generator=g) * 0.3
    seen = {}
    hooks = [layer.register_forward_hook(lambda m, a, o, i=i: seen.__setitem__(f"player{i}", o.detach().clone()))
             for i, layer in enumerate(dec.melspec_encoder.layers)]
    with torch.no_grad():
        h = enc(wav)
        pf = enc.get_prosody_feature(wav)
        outs, qs, commit, bufs, spk = dec(h, pf, vq=True, eval_vq=True, n_quantizers=nq)
        for hk in hooks:
            hk.remove()
        stages = dict(wav=wav, enc=h, pf=pf, qs=qs, outs=outs, spk_embs=spk, **seen)
        if nq is None:   # vq2emb reads every code row: the variants that keep all layers
            stages["emb_nores"] = dec.vq2emb(qs, use_residual=False)
            if dec_hp["vq_num_q_r"] > 0:
                stages["emb_res"] = dec.vq2emb(qs, use_residual=True)
            stages["wav_out"] = dec.inference(outs, spk)
            # README (models/codec/ns3_codec/README.md): A's prosody and content codes with B's speaker embedding
            h_b = enc(wav_b)
            pf_b = enc.get_prosody_feature(wav_b)
            _, qs_b, _, _, spk_b = dec(h_b, pf_b, vq=True, eval_vq=True, n_quantizers=nq)
            stages.update(wav_b=wav_b, enc_b=h_b, pf_b=pf_b, qs_b=qs_b, spk_b=spk_b,
                          vc=dec.inference(dec.vq2emb(qs, use_residual=False), spk_b))
    for k, v in stages.items():
        out[f"{tag}:{k}"] = v.numpy()
    for i, b in enumerate(bufs):
        out[f"{tag}:buf{i}"] = b.numpy()
    out[f"{tag}:mel_basis"] = enc.mel_transform.mel_basis.numpy()
    sd = {k: v.detach().numpy() for k, v in list(enc.state_dict().items()) + list(dec.state_dict().items())}
    dg = fvo.digests(sd)
    dg.update(fvo.fqo.digests({"timbre_encoder.enc." + k: v for k, v in enc.state_dict().items()}))
    dg.update(fvo.fqo.digests({"timbre_encoder.dec." + k: v for k, v in dec.state_dict().items()
                               if k.startswith(("model.", "timbre_linear."))}))
    out[f"{tag}:digest_names"] = np.array(list(dg.keys()))
    out[f"{tag}:digests"] = np.array(list(dg.values()))
    for name, m in (("enc", enc), ("dec", dec)):
        sdm = m.state_dict()
        out[f"{tag}:{name}_keys"] = np.array(list(sdm.keys()))
        out[f"{tag}:{name}_shapes"] = np.array([",".join(map(str, v.shape)) for v in sdm.values()])
    assert commit.abs().max() == 0
    print(tag, "qs", tuple(qs.shape), "outs absmax", float(outs.abs().max()), "spk absmax", float(spk.abs().max()))


if __name__ == "__main__":
    out = {}
    for tag in fvo.GOLDEN_FACODEC_V2:
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
        path = os.path.join(HERE, "fac_v2.npz" if i == 0 else f"fac_v2.part{i + 1}.npz")
        np.savez(path, **p)
        print(path, os.path.getsize(path), "bytes")
